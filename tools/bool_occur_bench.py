#!/usr/bin/env python
"""Bool queries (must / should / filter / must_not) and boosted Or in search_topk (sa_score_batch_topk_bool) on
the bench corpus, next to the plain Or / And they extend, measured in the same run.

    python tools/bool_occur_bench.py [--docs 10000000] [--queries 1024] [--phrase-queries 64] [--k 10] [--reps 5]

Corpus and terms are bench.py's: the seeded 10M-doc synthetic corpus and its 1,024 stratified single-term queries.
Clause terms are drawn from those; the `+rare common` pair takes its terms from the rarest df bucket (1e-4: about
one doc per 8192-doc tile, so about half of the tiles hold none) and the most common one (0.3).  Workloads (a, b, c:
random stratified terms):
  must_a_b_c        Bool(must=[a], should=[b, c])         `+a b c`
  a_b_not_c         Bool(should=[a, b], must_not=[c])     `a b -c`
  must_a_must_b     Bool(must=[a, b])                     `+a +b`, next to and2 = And([a, b])
  filter_a_b_c      Bool(filter=[a], should=[b, c])
  or3_boosted       Or([a^2, b^0.5, c^3]), next to or3 = Or([a, b, c])
  must_rare_common  Bool(must=[rare], should=[common]), next to or_rare_common = Or([rare, common])
  a_b_not_phrase    Bool(should=[a, b], must_not=[phrase of two terms]) in its own, smaller batch (each phrase row is
                    built synchronously)
Per workload, after a sample has been checked against the composition of .score (ids and score bits):
  qps            the whole batch through search_topk, host clock around the synchronous call, median of --reps
                 after --warmup warm-ups;
  bytes / gbs    algorithmic bytes per query (DESIGN.md 3.10): over every clause, whatever its role, P_c + 4*df_c for
                 a term (P_c = 4*df_c with a tf table, 8*W_c without), 8*(W_a + W_b) + 8*N for a phrase (its lists,
                 its row written and read), and the rate they are moved at over the whole call;
  n_redone       queries of the timed batch re-run exactly (candidate overflow);
  host_prep_ms   the Python part of one call (flattening, per-clause idf), timed alone;
  c_call_qps     the C entry point alone on arrays prepared once (planning, uploads, kernels, the result copy),
                 median of --reps after --warmup, its result checked equal to search_topk's.
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
from _bool_compose import topk  # noqa: E402
from _bool_occur_compose import compose_occur, parts  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--phrase-queries", type=int, default=64)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--verify", type=int, default=8)
    args = ap.parse_args()

    from searcharray_b200 import And, Bool, Boost, Or, SearchArray, bm25_similarity, synth
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
    dfs = {t: int(arr.docfreq(t)) for t in names}

    def term_bytes(t):
        P = 4 * dfs[t] if dir_min <= lens[spec.term_index[t]] < 0xFFFFFFFF else 8 * int(lens[spec.term_index[t]])
        return P + 4 * dfs[t]

    def clause_bytes(c):
        if isinstance(c, str):
            return term_bytes(c)
        return 8 * sum(int(lens[spec.term_index[t]]) for t in c) + 8 * n

    def query_bytes(q):
        must, _, should, _, filt, must_not, _ = parts(q)
        return sum(clause_bytes(c) for c in must + should + filt + must_not)

    rng = np.random.default_rng(20261016)
    perm = [rng.permutation(len(names)) for _ in range(4)]
    by_df = sorted(names, key=lambda t: dfs[t])
    sixth = max(1, len(by_df) // len(synth.DF_BUCKETS))
    rare, common = by_df[:sixth], by_df[-sixth:]                  # the rarest and the most common df bucket
    rare_perm, common_perm = rng.permutation(len(rare)), rng.permutation(len(common))

    def t(i, j):
        return names[perm[j][i % len(names)]]

    nq, npq = len(names), min(args.phrase_queries, len(names))
    workloads = {
        "must_a_b_c": [Bool(must=[t(i, 0)], should=[t(i, 1), t(i, 2)]) for i in range(nq)],
        "or3": [Or([t(i, 0), t(i, 1), t(i, 2)]) for i in range(nq)],
        "a_b_not_c": [Bool(should=[t(i, 0), t(i, 1)], must_not=[t(i, 2)]) for i in range(nq)],
        "must_a_must_b": [Bool(must=[t(i, 0), t(i, 1)]) for i in range(nq)],
        "and2": [And([t(i, 0), t(i, 1)]) for i in range(nq)],
        "filter_a_b_c": [Bool(filter=[t(i, 0)], should=[t(i, 1), t(i, 2)]) for i in range(nq)],
        "or3_boosted": [Or([Boost(t(i, 0), 2), Boost(t(i, 1), 0.5), Boost(t(i, 2), 3)]) for i in range(nq)],
        "must_rare_common": [Bool(must=[rare[rare_perm[i % len(rare)]]], should=[common[common_perm[i % len(common)]]])
                             for i in range(nq)],
        "or_rare_common": [Or([rare[rare_perm[i % len(rare)]], common[common_perm[i % len(common)]]])
                           for i in range(nq)],
        "a_b_not_phrase": [Bool(should=[t(i, 0), t(i, 1)], must_not=[[t(i, 2), t(i, 3)]]) for i in range(npq)],
    }
    sim = bm25_similarity()
    out = {"card": info, "docs": n, "k": args.k, "reps": args.reps, "warmup": args.warmup,
           "rare_df_mean": float(np.mean([dfs[x] for x in rare])), "common_df_mean": float(np.mean([dfs[x] for x in common])),
           "workloads": {}}
    for label, queries in workloads.items():
        sample = queries[::max(1, len(queries) // args.verify)][:args.verify]
        d, s, _ = arr._search_topk_bool(sample, args.k, sim, 0)
        for i, q in enumerate(sample):
            wd, ws = topk(compose_occur(lambda c: arr.score(c), q), args.k)
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
        per_query = np.asarray([query_bytes(q) for q in queries], dtype=np.float64)
        # the Python side of the call alone: flattening and the per-clause idf (part of every timed call)
        t0 = time.perf_counter()
        call = arr._prepare_bool(queries, sim)
        prep_ms = 1e3 * (time.perf_counter() - t0)
        # the C call alone on the prepared arrays: planning, uploads, kernels, the result copy
        for _ in range(args.warmup):
            call.run(args.k, 0)
        c_times = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            docs, scores, _ = call.run(args.k, 0)
            c_times.append(time.perf_counter() - t0)
        d_ref, s_ref, _ = arr._search_topk_bool(queries, args.k, sim, 0)
        if not (np.array_equal(docs, d_ref) and np.array_equal(scores.view(np.uint32), s_ref.view(np.uint32))):
            raise SystemExit(f"{label}: the C call on prepared arrays differs from search_topk")
        rec = {"queries": len(queries), "verified_queries": len(sample), "qps_median": len(queries) / t_med,
               "qps_best": len(queries) / min(times), "ms_per_batch_median": 1e3 * t_med,
               "host_prep_ms": prep_ms, "c_call_qps_median": len(queries) / float(np.median(c_times)),
               "c_call_ms_median": 1e3 * float(np.median(c_times)),
               "mb_per_query_mean": float(per_query.mean()) / 1e6, "gbs_median": float(per_query.sum()) / t_med / 1e9,
               "n_redone": redone}
        out["workloads"][label] = rec
        print(f"[bool_occur_bench] {label}: {json.dumps(rec)}", file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
