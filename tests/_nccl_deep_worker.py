"""Worker for tests/test_nccl_deep_gpu.py: one process per GPU, doc-range shards of one synthetic corpus, and
sa_score_batch_topk_allgather at deep k (the per-shard deep collector, ncclAllGather and the device merge); rank 0
compares the merged global top k (doc ids and score bits) with the CPU oracle on the full corpus."""
import ctypes
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from searcharray_b200 import _lib, synth  # noqa: E402
from searcharray_b200.postings import DeviceIndex  # noqa: E402
from searcharray_b200.similarity import compute_idf  # noqa: E402

K1, B = 1.2, 0.75


def main():
    rank, world, key = int(sys.argv[1]), int(sys.argv[2]), sys.argv[3]
    os.environ.setdefault("NCCL_SOCKET_IFNAME", "lo")
    os.environ.setdefault("NCCL_IB_DISABLE", "1")
    n_docs = 400_000
    L = _lib.lib()
    spec = synth.SynthSpec(n_docs, terms_per_bucket=3, n_phrases=12, n_bigrams=2)
    host, lo, hi = synth.generate_shard(spec, rank, world, n_threads=4)
    avgdl = synth.global_avg_doc_length(spec)
    dev = DeviceIndex(host, device=rank, doc_base=lo)
    h = dev.handle
    uid = (ctypes.c_char * 128)()
    if rank == 0:
        _lib.check(L.sa_comm_unique_id(uid))
        with open(key + ".tmp", "wb") as f:
            f.write(bytes(uid))
        os.replace(key + ".tmp", key)
    else:
        t0 = time.time()
        while not os.path.exists(key):
            assert time.time() - t0 < 300
            time.sleep(0.05)
        with open(key, "rb") as f:
            uid = (ctypes.c_char * 128).from_buffer_copy(f.read(128))
    _lib.check(L.sa_comm_init(h, uid, rank, world))
    df = np.zeros(host.n_terms, dtype=np.uint64)
    tmp = ctypes.c_uint64(0)
    for t in range(host.n_terms):
        _lib.check(L.sa_docfreq(h, t, ctypes.byref(tmp)))
        df[t] = tmp.value
    _lib.check(L.sa_comm_allreduce_sum_u64(h, _lib.p_u64(df), len(df)))
    queries = [[t] for t in range(host.n_terms)]
    terms = np.asarray([q[0] for q in queries], dtype=np.uint32)
    starts = np.arange(len(queries) + 1, dtype=np.uint32)
    idf = np.asarray([compute_idf(n_docs, df[np.asarray(q)]) for q in queries], dtype=np.float32)
    results = {}
    for k in (100, 1024):
        docs = np.empty((len(queries), k), dtype=np.uint32)
        scores = np.empty((len(queries), k), dtype=np.float32)
        _lib.check(L.sa_score_batch_topk_allgather(h, _lib.p_u32(terms), _lib.p_u32(starts), _lib.p_f32(idf),
                                                   len(queries), 0, float(avgdl), K1, B, k, _lib.p_u32(docs),
                                                   _lib.p_f32(scores)))
        results[k] = (docs, scores)
    if rank == 0:
        from oracle import search as osearch
        full, _, _ = synth.generate_shard(spec, 0, 1, n_threads=4)
        oidx = osearch.OracleIndex({t: full.term_words(t) for t in range(full.n_terms)}, full.doc_lens,
                                   avg_doc_length=avgdl, corpus_size=n_docs)
        n_checked = 0
        for k, (docs, scores) in results.items():
            for i, q in enumerate(queries):
                dense = oidx.score(q[0], k1=K1, b=B)
                nz = np.flatnonzero(dense > 0)
                order = nz[np.lexsort((nz, -dense[nz].astype(np.float64)))][:k]
                assert np.array_equal(docs[i][:len(order)], order.astype(np.uint32)), (k, q)
                assert np.all(docs[i][len(order):] == 0xFFFFFFFF), (k, q)
                assert np.array_equal(scores[i][:len(order)].view(np.uint32), dense[order].view(np.uint32)), (k, q)
                n_checked += 1
        print("NCCL_DEEP_OK", world, n_checked, flush=True)
    _lib.check(L.sa_comm_barrier(h))
    dev.close()


if __name__ == "__main__":
    main()
