#!/usr/bin/env python
"""Boolean queries in search_topk (sa_score_batch_topk_bool) on the bench corpus, against the composition they
replace.

    python tools/bool_topk_bench.py [--docs 10000000] [--queries 1024] [--phrase-queries 64] [--k 10] [--reps 5]

Corpus and terms are bench.py's: the seeded 10M-doc synthetic corpus and its 1,024 stratified single-term queries,
so the clauses of one query are drawn across the df buckets.  Workloads: OR of 2, 3 and 4 terms, AND of 2 and 3
terms, OR of two terms and one two-term phrase (its own, smaller batch: each phrase row is built synchronously).
Per workload, after a sample has been checked against the composition of .score (ids and score bits):
  qps            the whole batch through search_topk, host clock around the synchronous call, after warm-up;
  bytes / gbs    algorithmic bytes per query (DESIGN.md 3.9): sum over term clauses of P_c + 4*df_c
                 (P_c = 4*df_c with a tf table, 8*W_c without), plus per phrase clause 8*(W_a + W_b) + 8*N
                 (its lists, its row written and read), and the rate they are moved at over the whole call;
  n_redone       queries of the timed batch re-run exactly (candidate overflow);
  compose_qps    the composition: one .score per clause, the float32 sum and mm mask in numpy, argpartition,
                 for --baseline-queries queries.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from view_topk_bench import card  # noqa: E402
from _bool_compose import compose, topk  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--phrase-queries", type=int, default=64)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--verify", type=int, default=8)
    ap.add_argument("--baseline-queries", type=int, default=32)
    args = ap.parse_args()

    from searcharray_b200 import And, Or, SearchArray, bm25_similarity, synth
    info = card()
    spec = synth.SynthSpec(args.docs)
    host, _, _ = synth.generate_shard(spec)
    avgdl = synth.global_avg_doc_length(spec)
    host.avg_doc_length = avgdl
    arr = SearchArray.from_host_index(host, avg_doc_length=avgdl)
    names = synth.stratified_term_queries(spec, args.queries)
    n = host.n_docs
    n_tiles = (n + 8191) // 8192
    dir_min = max(1024, n_tiles // 2)
    lens = np.asarray(host.term_lengths, dtype=np.int64)

    def term_bytes(t):
        tid = spec.term_index[t]
        df = int(arr.docfreq(t))
        P = 4 * df if dir_min <= lens[tid] < 0xFFFFFFFF else 8 * int(lens[tid])
        return P + 4 * df

    def clause_bytes(c):
        if isinstance(c, str):
            return term_bytes(c)
        return 8 * sum(int(lens[spec.term_index[t]]) for t in c) + 8 * n

    rng = np.random.default_rng(20261016)
    perm = [rng.permutation(len(names)) for _ in range(4)]

    def terms(i, m):
        return [names[p[i]] for p in perm[:m]]

    nq, npq = len(names), min(args.phrase_queries, len(names))
    workloads = {
        "or2": [Or(terms(i, 2)) for i in range(nq)],
        "or3": [Or(terms(i, 3)) for i in range(nq)],
        "or4": [Or(terms(i, 4)) for i in range(nq)],
        "and2": [And(terms(i, 2)) for i in range(nq)],
        "and3": [And(terms(i, 3)) for i in range(nq)],
        "or2_phrase": [Or(terms(i, 2) + [terms(i + 1, 4)[2:]]) for i in range(npq)],
    }
    sim = bm25_similarity()
    out = {"card": info, "docs": n, "k": args.k, "reps": args.reps, "workloads": {}}
    for label, queries in workloads.items():
        sample = queries[::max(1, len(queries) // args.verify)][:args.verify]
        d, s, _ = arr._search_topk_bool(sample, args.k, sim, 0)
        for i, q in enumerate(sample):
            v, _ = compose(lambda c: arr.score(c), q.clauses, q.mm)
            wd, ws = topk(v, args.k)
            if not (np.array_equal(d[i], wd) and np.array_equal(s[i].view(np.uint32), ws.view(np.uint32))):
                raise SystemExit(f"{label}: search_topk differs from the composition for {q!r}")
        for _ in range(args.warmup):
            arr._search_topk_bool(queries, args.k, sim, 0)
        times, redone = [], []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            _, _, r = arr._search_topk_bool(queries, args.k, sim, 0)
            times.append(time.perf_counter() - t0)
            redone.append(r)
        t_med = float(np.median(times))
        per_query = np.asarray([sum(clause_bytes(c) for c in q.clauses) for q in queries], dtype=np.float64)
        rec = {"queries": len(queries), "verified_queries": len(sample), "qps_median": len(queries) / t_med,
               "qps_best": len(queries) / min(times), "ms_per_batch_median": 1e3 * t_med,
               "bytes_per_query_mean": float(per_query.mean()), "gbs_median": float(per_query.sum()) / t_med / 1e9,
               "n_redone": redone}
        bq = queries[:args.baseline_queries]
        t0 = time.perf_counter()
        for q in bq:
            scores = [arr.score(c) for c in q.clauses]
            v = scores[0]
            for x in scores[1:]:
                v = v + x
            ok = np.sum(np.array(scores) > 0, axis=0) >= q.mm
            np.argpartition(np.where(ok, v, 0), -args.k)[-args.k:]
        rec["compose_qps"] = len(bq) / (time.perf_counter() - t0)
        out["workloads"][label] = rec
        print(f"[bool_topk_bench] {label}: {json.dumps(rec)}", file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
