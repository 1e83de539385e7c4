"""Worker for tests/test_comp_rows_gpu.py: term-only, term + phrase and slop-2 batches on the 300k-doc synthetic corpus
under several query-group widths of the term scan over compressible rows (SA_COMP_ROW_GROUP, read per launch), in a
process whose SA_DENSE_PLAIN setting (read once per process) decides whether the term rows are compressible.  Every
result is checked against the CPU oracle here; prints one JSON line with a digest of each width's results and the
term launches and query groups of its term-only batch."""
import ctypes
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

import numpy as np  # noqa: E402

K = 10
GROUPS = ("1", "3", "8", "0")       # the 31 and 11 term rows below leave a partial last group at G = 3 and at G = 8


def oracle_check(oidx, ops, spec, q, slop, docs, scores):
    toks = [q] if isinstance(q, str) else q
    ids = [spec.term_index[t] for t in toks]
    s = oidx.score(ids[0]) if len(ids) == 1 else oidx.score(ids, slop=slop)
    if len(ids) > 1 and ops.last_span_undefined:
        return
    nz = np.flatnonzero(s > 0)
    order = nz[np.lexsort((nz, -s[nz].astype(np.float64)))][:K]
    assert np.array_equal(docs[:len(order)], order.astype(np.uint32)), (q, slop)
    assert np.all(docs[len(order):] == 0xFFFFFFFF), (q, slop)
    if len(ids) == 1:              # term rows: the oracle's bits
        assert np.array_equal(scores[:len(order)].view(np.uint32), s[order].view(np.uint32)), q
    else:
        np.testing.assert_allclose(scores[:len(order)], s[order], rtol=1e-5, atol=0)


def main():
    from oracle import ops, search as osearch
    from searcharray_b200 import SearchArray, _lib, synth
    spec = synth.SynthSpec(300_000)
    host, _, _ = synth.generate_shard(spec)
    arr = SearchArray.from_host_index(host)
    oidx = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                               avg_doc_length=host.avg_doc_length, corpus_size=host.n_docs, cache=False)
    terms = [nm for bi in range(len(synth.DF_BUCKETS)) for nm in spec.bucket_terms[bi][:5]]
    terms.append(spec.bucket_terms[0][5])                                                      # 31 rows, then 16, 11
    phrases = [ph["terms"] for ph in spec.phrases[:6]]
    batches = [(terms, 0), (terms[::2] + phrases, 0), (terms[::3] + phrases, 2)]
    L, h = _lib.lib(), arr._device().handle
    st = _lib.SaStats()
    out = {"digest": {}, "launches": {}, "groups": {}, "n_terms": len(terms)}
    for g in GROUPS:
        os.environ["SA_COMP_ROW_GROUP"] = g
        dig = hashlib.sha256()
        for bi, (qs, slop) in enumerate(batches):
            _lib.check(L.sa_stats_reset(h))
            docs, scores = arr.search_topk(qs, k=K, slop=slop)
            if bi == 0:
                _lib.check(L.sa_stats_get(h, ctypes.byref(st)))
                out["launches"][g] = st.term_kernel_launches
                out["groups"][g] = st.term_kernel_groups
            for i, q in enumerate(qs):
                oracle_check(oidx, ops, spec, q, slop, docs[i], scores[i])
            dig.update(np.ascontiguousarray(docs).tobytes())
            dig.update(np.ascontiguousarray(scores).tobytes())
        out["digest"][g] = dig.hexdigest()
    m = ctypes.c_int(-1)
    _lib.check(L.sa_index_dense_compressible(h, ctypes.byref(m)))
    out["compressible"] = m.value
    print(json.dumps(out))


if __name__ == "__main__":
    main()
