#!/usr/bin/env python
"""Disjunction-max clauses (query.DisMax) on the bench corpus: best_fields over two DataFrame fields through
solr.fields_topk (sa_multi_score_batch_topk_bool with groups), next to the same leaves as most_fields (an Or of the Field
clauses, sa_multi_score_batch_topk_bool) measured in the same run, and single-column synonyms through search_topk.

    python tools/dismax_topk_bench.py [--docs 10000000] [--queries 1024] [--k 10] [--reps 5] [--edismax-queries 4]

Corpus and terms are bench.py's: the seeded 10M-doc synthetic corpus and its 1,024 stratified single-term queries,
uploaded as TWO columns with identical data, f1 and f2 (as tools/fields_topk_bench.py).  Workloads (a, b, c: random
stratified terms; rare / common: the rarest and the most common df bucket):
  best2_tie0 / best2_tie03   Or([DisMax([f1:a^2, f2:a], tie), DisMax([f1:b^2, f2:b], tie)])       tie 0 / 0.3
  best3_tie0 / best3_tie03   the same over a, b, c
  must_rare_common           Bool(must=[DisMax([f1:rare, f2:rare])], should=[DisMax([f1:common, f2:common])])
  synonyms                   search_topk on f1 of DisMax([a, b], tie=0.1), against Or([a, b])
Its most_fields equivalent is the Or of the same leaves (with their boosts), every leaf one clause.  Per workload,
after a sample has been checked against the numpy composition of per-field .score (ids and score bits):
  qps              fields_topk (search_topk for synonyms), host clock around the synchronous call, median of --reps;
  c_call_qps       the C entry point alone on arrays prepared once;
  most_fields_c_call_qps, ratio_c_call   the same for the most_fields equivalent, and c_call_qps over it;
  n_redone         queries of the timed batch re-run exactly (candidate overflow);
  edismax_qps      for the best_fields workloads: the host-driven solr.edismax with qf=[f1^2, f2] alone (no pf) on
                   --edismax-queries of the same queries, for context.
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
from _bool_fields_compose import field_scorer  # noqa: E402
from _dismax_compose import compose_dismax  # noqa: E402


def median_time(fn, warmup, reps):
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
    ap.add_argument("--edismax-queries", type=int, default=4)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--verify", type=int, default=6)
    args = ap.parse_args()

    import pandas as pd
    from searcharray_b200 import Bool, Boost, DisMax, Field, Or, SearchArray, bm25_similarity, synth
    from searcharray_b200.postings import _PreparedBool
    from searcharray_b200.solr import _clause_slots, _fields_plan, _fields_topk, _multi_for
    from searcharray_b200 import solr
    info = card()
    spec = synth.SynthSpec(args.docs)
    host, _, _ = synth.generate_shard(spec)
    avgdl = synth.global_avg_doc_length(spec)
    host.avg_doc_length = avgdl
    frame = pd.DataFrame({"f1": SearchArray.from_host_index(host, avg_doc_length=avgdl),
                          "f2": SearchArray.from_host_index(host, avg_doc_length=avgdl)})
    f1 = frame["f1"].array
    names = synth.stratified_term_queries(spec, args.queries)
    dfs = {t: int(f1.docfreq(t)) for t in names}
    rng = np.random.default_rng(20261016)
    perm = [rng.permutation(len(names)) for _ in range(3)]
    by_df = sorted(names, key=lambda t: dfs[t])
    sixth = max(1, len(by_df) // len(synth.DF_BUCKETS))
    rare, common = by_df[:sixth], by_df[-sixth:]
    rare_perm, common_perm = rng.permutation(len(rare)), rng.permutation(len(common))

    def t(i, j):
        return names[perm[j][i % len(names)]]

    def rare_i(i):
        return rare[rare_perm[i % len(rare)]]

    def common_i(i):
        return common[common_perm[i % len(common)]]

    F = Field
    nq = len(names)

    def best(i, n_terms, tie):
        return Or([DisMax([Boost(F("f1", t(i, j)), 2), F("f2", t(i, j))], tie=tie) for j in range(n_terms)])

    def most(i, n_terms):
        return Or([x for j in range(n_terms) for x in (Boost(F("f1", t(i, j)), 2), F("f2", t(i, j)))])
    work = {
        "best2_tie0": (lambda i: best(i, 2, 0.0), lambda i: most(i, 2), 2),
        "best2_tie03": (lambda i: best(i, 2, 0.3), lambda i: most(i, 2), 2),
        "best3_tie0": (lambda i: best(i, 3, 0.0), lambda i: most(i, 3), 3),
        "best3_tie03": (lambda i: best(i, 3, 0.3), lambda i: most(i, 3), 3),
        "must_rare_common": (lambda i: Bool(must=[DisMax([F("f1", rare_i(i)), F("f2", rare_i(i))])],
                                            should=[DisMax([F("f1", common_i(i)), F("f2", common_i(i))])]),
                             lambda i: Or([F("f1", rare_i(i)), F("f2", rare_i(i)), F("f1", common_i(i)),
                                           F("f2", common_i(i))]), 0),
    }
    sim = bm25_similarity()
    score = field_scorer({f: (lambda c, f=f: frame[f].array.score(c)) for f in ("f1", "f2")})
    out = {"card": info, "docs": host.n_docs, "k": args.k, "reps": args.reps, "warmup": args.warmup,
           "rare_df_mean": float(np.mean([dfs[x] for x in rare])), "common_df_mean": float(np.mean([dfs[x] for x in common])),
           "workloads": {}}

    def c_time(queries):
        batch, slot_of, arrays, sims = _fields_plan(frame, queries, sim)
        call = _PreparedBool(arrays, sims, _clause_slots(batch, slot_of), queries, batch,
                             multi=_multi_for(arrays))
        return median_time(lambda: call.run(args.k, 0), args.warmup, args.reps)

    def verify(label, queries, run, scorer):
        sample = queries[::max(1, len(queries) // args.verify)][:args.verify]
        d, s = run(sample)
        for i, q in enumerate(sample):
            wd, ws = topk(compose_dismax(scorer, q), args.k)
            if not (np.array_equal(d[i], wd) and np.array_equal(s[i].view(np.uint32), ws.view(np.uint32))):
                raise SystemExit(f"{label}: differs from the composition for {q!r}")
        return len(sample)

    for label, (make, make_most, n_terms) in work.items():
        dq = [make(i) for i in range(nq)]
        mq = [make_most(i) for i in range(nq)]
        n_ver = verify(label, dq, lambda qs: _fields_topk(frame, qs, args.k, sim, 0)[:2], score)
        redone = []

        def run():
            redone.append(_fields_topk(frame, dq, args.k, sim, 0)[2])
        t_api = median_time(run, args.warmup, args.reps)
        t_c, t_most = c_time(dq), c_time(mq)
        rec = {"queries": nq, "verified_queries": n_ver, "qps": nq / t_api, "c_call_qps": nq / t_c,
               "most_fields_c_call_qps": nq / t_most, "ratio_c_call": t_most / t_c, "n_redone": redone[-args.reps:]}
        if n_terms and args.edismax_queries:
            tie = dq[0].clauses[0].tie
            ne = min(args.edismax_queries, nq)
            texts = [" ".join(t(i, j) for j in range(n_terms)) for i in range(ne)]
            try:
                solr.edismax(frame, texts[0], qf=["f1^2", "f2"], mm="1", tie=float(tie))     # warm
                t0 = time.perf_counter()
                for q in texts:
                    solr.edismax(frame, q, qf=["f1^2", "f2"], mm="1", tie=float(tie))
                rec["edismax_qps"] = ne / (time.perf_counter() - t0)
                rec["edismax_queries"] = ne
            except Exception as e:                  # noqa: BLE001 -- reported in the record
                rec["edismax_error"] = repr(e)
        out["workloads"][label] = rec
        print(f"[dismax_topk_bench] {label}: {json.dumps(rec)}", file=sys.stderr, flush=True)

    # single-column synonyms through search_topk, against Or of the same terms
    sq = [DisMax([t(i, 0), t(i, 1)], tie=0.1) for i in range(nq)]
    oq = [Or([t(i, 0), t(i, 1)]) for i in range(nq)]
    n_ver = verify("synonyms", sq, lambda qs: f1.search_topk(qs, k=args.k), f1.score)
    t_api = median_time(lambda: f1.search_topk(sq, k=args.k), args.warmup, args.reps)
    t_or_api = median_time(lambda: f1.search_topk(oq, k=args.k), args.warmup, args.reps)
    dismax_call, or_call = f1._prepare_bool(sq, sim), f1._prepare_bool(oq, sim)
    redone = []
    t_c = median_time(lambda: redone.append(dismax_call.run(args.k, 0)[2]), args.warmup, args.reps)
    t_or_c = median_time(lambda: or_call.run(args.k, 0), args.warmup, args.reps)
    rec = {"queries": nq, "verified_queries": n_ver, "qps": nq / t_api, "or_qps": nq / t_or_api, "c_call_qps": nq / t_c,
           "or_c_call_qps": nq / t_or_c, "ratio_c_call": t_or_c / t_c, "n_redone": redone[-args.reps:]}
    out["workloads"]["synonyms"] = rec
    print(f"[dismax_topk_bench] synonyms: {json.dumps(rec)}", file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
