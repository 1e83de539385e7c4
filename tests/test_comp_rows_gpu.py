"""GPU: the term batch's rows in compressible memory, scanned in query groups.  Every group width G in {1, 3, 8, all}
ranks term-only, term + phrase and slop-2 batches as the CPU oracle does, in one term launch per chunk, and gives the
same bits as SA_DENSE_PLAIN=1 (every row in plain memory), each arm in its own process (tests/_comp_rows_worker.py).
Compressible rows start on a granule of their own (2 MiB on H100); they grow and are freed with the index."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KNOBS = ("SA_DENSE_PLAIN", "SA_COMP_ROW_GROUP", "SA_TERM_QUERY_MAJOR")


def run_worker(plain):
    env = {k: v for k, v in os.environ.items() if k not in KNOBS}
    if plain:
        env["SA_DENSE_PLAIN"] = "1"
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_comp_rows_worker.py")
    r = subprocess.run([sys.executable, worker], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_groups_give_the_oracle_and_plain_bits():
    comp = run_worker(plain=False)
    plain = run_worker(plain=True)
    assert comp["compressible"] == 1     # H100 supports generic compression
    assert plain["compressible"] == 0
    want = plain["digest"]["0"]
    assert set(plain["digest"].values()) == {want}
    assert set(comp["digest"].values()) == {want}, comp["digest"]
    assert comp["launches"] == plain["launches"]       # one term launch per chunk (and per exact re-run) either way
    # the width reaches the kernel: ceil(rows / G) groups for the batch's launch, one for each single-query re-run
    n = comp["n_terms"]
    for g, width in (("1", 1), ("3", 3), ("8", 8), ("0", n)):
        redo = comp["launches"][g] - 1
        assert comp["groups"][g] == (n + width - 1) // width + redo, (g, comp["groups"], comp["launches"])
        assert plain["groups"][g] == plain["launches"][g]   # plain rows: every launch walks its queries as one group


def live():
    from searcharray_b200 import _lib
    n, b = ctypes.c_uint64(), ctypes.c_uint64()
    _lib.check(_lib.lib().sa_device_allocations(ctypes.byref(n), ctypes.byref(b)))
    return n.value, b.value


def _oracle_order(dense, k=10):
    nz = np.flatnonzero(dense > 0)
    return nz[np.lexsort((nz, -dense[nz].astype(np.float64)))][:k]


@pytest.mark.parametrize("n_docs", [300_000, 4_300_000])
def test_compressible_rows_grow_and_are_freed(monkeypatch, n_docs):
    """A row of >= 8 granules (4.3M docs: 17.2 MB) starts on a granule of its own; a shorter one (300k docs: 1.2 MB)
    stays packed, since padding it would cost 70 % more memory."""
    import gc
    from oracle import search as osearch
    from searcharray_b200 import SearchArray, synth
    monkeypatch.delenv("SA_DENSE_PLAIN", raising=False)
    monkeypatch.setenv("SA_COMP_ROW_GROUP", "3")
    before = live()
    spec = synth.SynthSpec(n_docs)
    host, _, _ = synth.generate_shard(spec)
    arr = SearchArray.from_host_index(host)
    oidx = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                               avg_doc_length=host.avg_doc_length, corpus_size=host.n_docs, cache=False)
    names = [nm for bi in range(len(synth.DF_BUCKETS)) for nm in spec.bucket_terms[bi][:8]]
    arr.score(names[0])                                 # the index's norms and one plain row
    base = live()[1]
    row = (host.n_docs + 8191) // 8192 * 8192 * 4
    padded = (row + (2 << 20) - 1) // (2 << 20) * (2 << 20)
    pad = padded - row <= row // 8
    assert pad == (n_docs > 1_000_000)
    for n in (2, 12, len(names)):                       # the compressible rows grow twice
        q = names[:n]
        docs, scores = arr.search_topk(q, k=10)
        if n == len(names):
            grown = live()[1] - base
            assert grown >= n * (padded if pad else row)
            if not pad:
                assert grown < n * padded
        for i, nm in enumerate(q):
            dense = oidx.score(spec.term_index[nm], k1=1.2, b=0.75)
            order = _oracle_order(dense)
            assert np.array_equal(docs[i][:len(order)], order), nm
            assert np.array_equal(scores[i][:len(order)].view(np.uint32), dense[order].view(np.uint32)), nm
    m = ctypes.c_int(-1)
    from searcharray_b200 import _lib
    _lib.check(_lib.lib().sa_index_dense_compressible(arr._device().handle, ctypes.byref(m)))
    assert m.value == 1
    arr._shared["dev"].close()
    del arr
    gc.collect()
    assert live() == before


def test_many_term_queries_on_a_one_tile_index():
    """40,000 term queries on an 8,192-doc index (one tile, 32 KB rows) in one chunk: packed compressible rows, so the
    batch takes about the memory its plain rows would, and ranks as the oracle does."""
    import gc
    from oracle import search as osearch
    from searcharray_b200 import SearchArray
    rng = np.random.default_rng(5)
    vocab = [f"w{i}" for i in range(64)]
    p = 1.0 / np.arange(1, 65)
    p /= p.sum()
    docs = [" ".join(rng.choice(vocab, size=int(rng.integers(1, 40)), p=p)) for _ in range(8192)]
    before = live()
    arr = SearchArray.index(docs)
    host = arr.host
    oidx = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                               avg_doc_length=host.avg_doc_length)
    tid = host.term_dict.term_to_ids
    arr.score(vocab[0])
    base = live()[1]
    Q = 40_000
    queries = [vocab[i % len(vocab)] for i in range(Q)]
    got_docs, got_scores = arr.search_topk(queries, k=10)
    row, cand = 8192 * 4, 128 * 8 + 8                  # one tile per row; 128 candidate slots + count + max at k = 10
    assert live()[1] - base <= 1.25 * Q * (row + cand) + (32 << 20)
    want = {}
    for w in vocab:
        dense = oidx.score(tid[w])
        order = _oracle_order(dense)
        want[w] = (order.astype(np.uint32), dense[order].view(np.uint32))
    for i, w in enumerate(queries):
        order, bits = want[w]
        assert np.array_equal(got_docs[i][:len(order)], order), (i, w)
        assert np.array_equal(got_scores[i][:len(order)].view(np.uint32), bits), (i, w)
        assert np.all(got_docs[i][len(order):] == 0xFFFFFFFF), (i, w)
    arr._shared["dev"].close()
    del arr
    gc.collect()
    assert live() == before
