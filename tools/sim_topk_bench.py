#!/usr/bin/env python
"""search_topk under bm25_impact, bm25_legacy_similarity and classic_similarity on the bench corpus, against the
alternative it replaces and against BM25 search_topk on the same array.

    python tools/sim_topk_bench.py [--docs 10000000] [--queries 1024] [--k 10] [--reps 5]

Corpus and queries are bench.py's: the seeded 10M-doc synthetic corpus and its 1,024 stratified single-term
queries.  Arrays: the unsliced array and a 10 % random mask.  Per (array, similarity), after a sample of the results
has been checked against .score(q, similarity=sim) (ids, score bits, dtype):
  qps            search_topk over the whole batch, host clock around the synchronous call, after warm-up;
  bm25_qps       the same batch with the default bm25_similarity;
  bytes / gbs    algorithmic bytes per term query and the rate they are moved at over the whole call:
                 P + 4*N (the tf scan and its doc-space count row), then per position 4 (count) + 8 (row index, views
                 only), and 4 per position with a count > 0 (doc length);
                 P = 4*df for terms with a tf table, 8*W for the others;
  score_argpartition_qps   the alternative: .score(q, similarity=sim) + np.argpartition, for 32 queries.
The card name and power limit come from a read-only nvidia-smi query in the same run.  Prints one JSON line.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from view_topk_bench import card  # noqa: E402


def expected_topk(dense, k):
    nz = np.flatnonzero(dense > 0)
    order = nz[np.lexsort((nz, -dense[nz].astype(np.float64)))][:k]
    docs = np.full(k, 0xFFFFFFFF, dtype=np.uint32)
    scores = np.zeros(k, dtype=dense.dtype)
    docs[:len(order)] = order
    scores[:len(order)] = dense[order]
    return docs, scores


def timed(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t0)
    return float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--verify", type=int, default=16, help="queries per (array, similarity) checked against .score")
    ap.add_argument("--baseline-queries", type=int, default=32)
    args = ap.parse_args()

    from searcharray_b200 import (SearchArray, bm25_impact, bm25_legacy_similarity, bm25_similarity,
                                  classic_similarity, synth)
    info = card()
    spec = synth.SynthSpec(args.docs)
    host, _, _ = synth.generate_shard(spec)
    avgdl = synth.global_avg_doc_length(spec)
    host.avg_doc_length = avgdl
    arr = SearchArray.from_host_index(host, avg_doc_length=avgdl)
    names = synth.stratified_term_queries(spec, args.queries)
    tids = np.asarray([spec.term_index[n] for n in names], dtype=np.uint32)
    n = host.n_docs

    n_tiles = (n + 8191) // 8192
    dir_min = max(1024, n_tiles // 2)
    lens = np.asarray(host.term_lengths, dtype=np.int64)[tids]
    df = np.asarray([int(arr.docfreq(nm)) for nm in names], dtype=np.int64)
    P = np.where((lens >= dir_min) & (lens < 0xFFFFFFFF), 4 * df, 8 * lens)

    rng = np.random.default_rng(20261015)
    arrays = {"unsliced": arr, "mask_10pct": arr[rng.random(n) < 0.10]}
    sims = {"bm25_impact": bm25_impact(), "bm25_legacy": bm25_legacy_similarity(), "classic": classic_similarity()}
    out = {"card": info, "docs": n, "queries": len(names), "k": args.k, "reps": args.reps, "arrays": {}}
    for label, view in arrays.items():
        sliced = view.rows is not None
        frac = len(view) / n
        bm25_t = timed(lambda: view.search_topk(names, k=args.k, similarity=bm25_similarity()), args.warmup, args.reps)
        recs = {"rows": len(view), "bm25_qps": len(names) / bm25_t}
        for sname, sim in sims.items():
            sample = names[::max(1, len(names) // args.verify)][:args.verify]
            d, s = view.search_topk(sample, k=args.k, similarity=sim)
            for i, q in enumerate(sample):
                wd, ws = expected_topk(view.score(q, similarity=sim), args.k)
                if not (s.dtype == ws.dtype and np.array_equal(d[i], wd) and
                        np.array_equal(s[i].view(np.uint8), ws.view(np.uint8))):
                    raise SystemExit(f"{label}/{sname}: search_topk differs from .score's top k for {q!r}")
            t_med = timed(lambda: view.search_topk(names, k=args.k, similarity=sim), args.warmup, args.reps)
            per_pos = 4 + (8 if sliced else 0)
            per_query = P + 4 * n + per_pos * len(view) + 4 * df * frac
            bq = names[:args.baseline_queries]
            t0 = time.perf_counter()
            for q in bq:
                sc = view.score(q, similarity=sim)
                top = np.argpartition(-sc, args.k)[:args.k] if len(sc) > args.k else np.arange(len(sc))
                top[np.argsort(-sc[top], kind="stable")]
            recs[sname] = {"verified_queries": len(sample), "qps_median": len(names) / t_med,
                           "ms_per_batch_median": 1e3 * t_med, "bytes_per_query_mean": float(per_query.mean()),
                           "gbs_median": float(per_query.sum()) / t_med / 1e9,
                           "score_argpartition_qps": len(bq) / (time.perf_counter() - t0)}
            print(f"[sim_topk_bench] {label}/{sname}: {json.dumps(recs[sname])}", file=sys.stderr, flush=True)
        out["arrays"][label] = recs
    print(json.dumps(out))


if __name__ == "__main__":
    main()
