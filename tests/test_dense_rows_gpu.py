"""GPU: the term batch writes rare terms' rows to compressible device memory (sa_index_dense_compressible), and
SA_DENSE_PLAIN=1 keeps every row in plain cudaMalloc memory.  Both give the same bits: term, phrase, slop-2 and mixed
batches and .score() vectors of every df bucket, each arm in its own process (tests/_dense_rows_worker.py)."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def run_worker(plain):
    env = dict(os.environ)
    env.pop("SA_DENSE_PLAIN", None)
    if plain:
        env["SA_DENSE_PLAIN"] = "1"
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_dense_rows_worker.py")
    r = subprocess.run([sys.executable, worker], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    return json.loads(r.stdout.strip().splitlines()[-1])


def test_compressible_and_plain_rows_give_the_same_bits():
    comp = run_worker(plain=False)
    plain = run_worker(plain=True)
    assert comp["compressible"] == 1     # H100 supports generic compression
    assert plain["compressible"] == 0
    assert comp["digest"] == plain["digest"]


def live():
    from searcharray_b200 import _lib
    n, b = ctypes.c_uint64(), ctypes.c_uint64()
    _lib.check(_lib.lib().sa_device_allocations(ctypes.byref(n), ctypes.byref(b)))
    return n.value, b.value


def test_rare_rows_grow_and_are_freed():
    import gc
    from oracle import search as osearch
    from searcharray_b200 import SearchArray, synth
    before = live()
    spec = synth.SynthSpec(300_000)
    host, _, _ = synth.generate_shard(spec)
    arr = SearchArray.from_host_index(host)
    oidx = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                               avg_doc_length=host.avg_doc_length, corpus_size=host.n_docs, cache=False)
    rare = list(spec.bucket_terms[5]) + list(spec.bucket_terms[4])
    for n in (2, 12, len(rare)):                       # the rare rows grow twice
        q = rare[:n] + list(spec.bucket_terms[0][:3])
        docs, scores = arr.search_topk(q, k=10)
        for i, nm in enumerate(q):
            dense = oidx.score(spec.term_index[nm], k1=1.2, b=0.75)
            nz = np.flatnonzero(dense > 0)
            order = nz[np.lexsort((nz, -dense[nz].astype(np.float64)))][:10]
            assert np.array_equal(docs[i][:len(order)], order), nm
            assert np.array_equal(scores[i][:len(order)].view(np.uint32), dense[order].view(np.uint32)), nm
    arr._shared["dev"].close()
    del arr
    gc.collect()
    assert live() == before
