#!/usr/bin/env python
"""Nested boolean queries (an Or / And / Bool as a clause of another) on the bench corpus, through solr.fields_topk
(sa_multi_score_batch_topk_bool) and SearchArray.search_topk (sa_score_batch_topk_bool), with clause_node.

    python tools/nested_topk_bench.py [--docs 10000000] [--queries 1024] [--k 10] [--reps 5]

Corpus and terms are bench.py's: the seeded 10M-doc synthetic corpus and its 1,024 stratified single-term queries,
uploaded as TWO columns with identical data, f1 and f2 (as tools/dismax_topk_bench.py).  Workloads (a, b, c, d:
random stratified terms):
  and_of_ors      And([Or([f1:a, f2:a]), Or([f1:b, f2:b])]), next to flat_or, the flat Or of the same four leaves
  or_of_ands      Or([And([a, b]), And([c, d])]) on f1 through search_topk
  must_not_conj   Bool(should=[f1:a], must_not=[And([f1:b, f2:c])])
  qf_pf           edismax's qf + pf shape: Bool(must=[Or([DisMax([f1:a^2, f2:a]), DisMax([f1:b^2, f2:b])], mm="75%")],
                  should=[Boost(f1:"a b", 3)])
Per workload, after a sample has been checked against the numpy composition of per-field .score (ids and score bits):
  qps            the public call, host clock around the synchronous call, median of --reps;
  c_call_qps     the C entry point alone on arrays prepared once;
  n_redone       queries of the timed batch re-run exactly (candidate overflow);
  nested_nodes   nested queries per query;
  leaf_df_mean   mean over queries of the summed document frequencies of its leaves (each posting is read once);
  row_bytes_max  per query, the most the nested rows can move: 4 bytes per doc written and read once per nested node
                 (a node writes only the tiles where it ranks, and its parent reads only those).
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
from _nested_compose import compose_nested  # noqa: E402


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
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--verify", type=int, default=6)
    args = ap.parse_args()

    import pandas as pd
    from searcharray_b200 import And, Bool, Boost, DisMax, Field, Or, SearchArray, bm25_similarity
    from searcharray_b200 import synth
    from searcharray_b200.postings import _PreparedBool
    from searcharray_b200.query import _leaves
    from searcharray_b200.solr import _clause_slots, _fields_plan, _fields_topk, _multi_for
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
    perm = [rng.permutation(len(names)) for _ in range(4)]
    nq = len(names)

    def t(i, j):
        return names[perm[j][i % len(names)]]
    F = Field
    work = {
        "and_of_ors": lambda i: And([Or([F("f1", t(i, 0)), F("f2", t(i, 0))]), Or([F("f1", t(i, 1)), F("f2", t(i, 1))])]),
        "flat_or": lambda i: Or([F("f1", t(i, 0)), F("f2", t(i, 0)), F("f1", t(i, 1)), F("f2", t(i, 1))]),
        "must_not_conj": lambda i: Bool(should=[F("f1", t(i, 0))], must_not=[And([F("f1", t(i, 1)), F("f2", t(i, 2))])]),
        "qf_pf": lambda i: Bool(must=[Or([DisMax([Boost(F("f1", t(i, j)), 2), F("f2", t(i, j))], tie=0.1)
                                          for j in range(2)], mm="75%")],
                                should=[Boost(F("f1", [t(i, 0), t(i, 1)]), 3)]),
    }
    sim = bm25_similarity()
    score = field_scorer({f: (lambda c, f=f: frame[f].array.score(c)) for f in ("f1", "f2")})
    out = {"card": info, "docs": host.n_docs, "k": args.k, "reps": args.reps, "warmup": args.warmup, "workloads": {}}

    def verify(label, queries, run, scorer):
        sample = queries[::max(1, len(queries) // args.verify)][:args.verify]
        d, s = run(sample)
        for i, q in enumerate(sample):
            wd, ws = topk(compose_nested(scorer, q), args.k)
            if not (np.array_equal(d[i], wd) and np.array_equal(s[i].view(np.uint32), ws.view(np.uint32))):
                raise SystemExit(f"{label}: differs from the composition for {q!r}")
        return len(sample)

    def shape(queries):
        n_nested = float(np.mean([getattr(q, "n_nested", 0) for q in queries]))
        def df(c):                      # a term leaf's df; phrases and DisMax clauses (their members are leaves) 0
            x = c.clause if isinstance(c, Field) else c
            return dfs.get(x, 0) if isinstance(x, str) else 0
        leaf_df = [sum(df(c) for c in _leaves(q)) for q in queries]
        return {"nested_nodes": n_nested, "leaf_df_mean": float(np.mean(leaf_df)),
                "row_bytes_max": 2 * 4 * host.n_docs * n_nested}

    for label, make in work.items():
        qs = [make(i) for i in range(nq)]
        n_ver = verify(label, qs, lambda x: _fields_topk(frame, x, args.k, sim, 0)[:2], score)
        redone = []

        def run():
            redone.append(_fields_topk(frame, qs, args.k, sim, 0)[2])
        t_api = median_time(run, args.warmup, args.reps)
        batch, slot_of, arrays, sims = _fields_plan(frame, qs, sim)
        call = _PreparedBool(arrays, sims, _clause_slots(batch, slot_of), qs, batch, multi=_multi_for(arrays))
        t_c = median_time(lambda: call.run(args.k, 0), args.warmup, args.reps)
        rec = dict({"queries": nq, "verified_queries": n_ver, "qps": nq / t_api, "c_call_qps": nq / t_c,
                    "n_redone": redone[-args.reps:]}, **shape(qs))
        out["workloads"][label] = rec
        print(f"[nested_topk_bench] {label}: {json.dumps(rec)}", file=sys.stderr, flush=True)

    # one column through search_topk
    qs = [Or([And([t(i, 0), t(i, 1)]), And([t(i, 2), t(i, 3)])]) for i in range(nq)]
    n_ver = verify("or_of_ands", qs, lambda x: f1.search_topk(x, k=args.k), f1.score)
    t_api = median_time(lambda: f1.search_topk(qs, k=args.k), args.warmup, args.reps)
    call = f1._prepare_bool(qs, sim)
    redone = []
    t_c = median_time(lambda: redone.append(call.run(args.k, 0)[2]), args.warmup, args.reps)
    rec = dict({"queries": nq, "verified_queries": n_ver, "qps": nq / t_api, "c_call_qps": nq / t_c,
                "n_redone": redone[-args.reps:]}, **shape(qs))
    out["workloads"]["or_of_ands"] = rec
    print(f"[nested_topk_bench] or_of_ands: {json.dumps(rec)}", file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
