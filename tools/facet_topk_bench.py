#!/usr/bin/env python
"""Hit and facet counts in batched top-k: search_topk with `facets=` on the bench corpus, against the same queries
without counts.

    python tools/facet_topk_bench.py [--docs 10000000] [--queries 1024] [--k 10] [--reps 5] [--verify 4]

Corpus and terms are bench.py's: the seeded 10M-doc synthetic corpus and its stratified single-term queries.  Facets
(seeded): `f20`, 20 buckets with ~5 % of docs without a value; `f1024`, 1,024 buckets.  Workloads (a, b: random
stratified terms), timed alternating in one run:
  or            Or([a, b])                      without facets
  or_total      Or([a, b]), facets=[]           totals only
  or_f20        Or([a, b]), facets=["f20"]
  or_f1024      Or([a, b]), facets=["f1024"]    (shared-atomic contention on broad queries would show here)
  term          a                               plain terms through the term scan
  term_total    a, facets=[]                    plain terms through the one-clause Or fold, totals only
Per workload: qps (the public call, host clock around the synchronous call, median of --reps), c_call_qps for the
Or workloads (sa_score_batch_topk_bool, with or without counts, on arrays prepared once), n_redone, and
verified: sampled queries whose total and facet rows equal numpy's count over the composed dense vector.  The card
name and power limit come from a read-only nvidia-smi query in the same run.  Prints one JSON line.
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
from _nested_compose import compose_nested  # noqa: E402


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--verify", type=int, default=4)
    args = ap.parse_args()

    from searcharray_b200 import Or, SearchArray, bm25_similarity
    from searcharray_b200 import synth
    info = card()
    spec = synth.SynthSpec(args.docs)
    host, _, _ = synth.generate_shard(spec)
    avgdl = synth.global_avg_doc_length(spec)
    host.avg_doc_length = avgdl
    arr = SearchArray.from_host_index(host, avg_doc_length=avgdl)
    n = len(arr)
    rng = np.random.default_rng(20261017)
    codes = {"f20": np.where(rng.random(n) < 0.05, -1, rng.integers(0, 20, n)), "f1024": rng.integers(0, 1024, n)}
    for name, c in codes.items():
        arr.set_facet(name, c)
    names = synth.stratified_term_queries(spec, args.queries)
    perm = [rng.permutation(len(names)) for _ in range(2)]
    nq = len(names)
    ors = [Or([names[perm[0][i]], names[perm[1][i]]]) for i in range(nq)]
    terms = [names[perm[0][i]] for i in range(nq)]
    sim = bm25_similarity()

    def c_call(facets):
        """The C call of search_topk(ors, facets=facets) on arrays prepared once: fn() -> n_redone."""
        call = arr._prepare_bool(ors, sim, facets=facets)
        return lambda: call.run(args.k, 0)[2]

    cells = {
        "or": (lambda: arr.search_topk(ors, k=args.k), c_call(None), ors, None),
        "or_total": (lambda: arr.search_topk(ors, k=args.k, facets=[]), c_call([]), ors, []),
        "or_f20": (lambda: arr.search_topk(ors, k=args.k, facets=["f20"]), c_call(["f20"]), ors, ["f20"]),
        "or_f1024": (lambda: arr.search_topk(ors, k=args.k, facets=["f1024"]), c_call(["f1024"]), ors, ["f1024"]),
        "term": (lambda: arr.search_topk(terms, k=args.k), None, terms, None),
        "term_total": (lambda: arr.search_topk(terms, k=args.k, facets=[]), None, terms, []),
    }
    for fn_pub, fn_c, _, _ in cells.values():            # warm every shape
        for _ in range(args.warmup):
            fn_pub()
            if fn_c:
                fn_c()
    times = {name: ([], [], []) for name in cells}
    for _ in range(args.reps):                           # alternating, so the cells see the same machine state
        for name, (fn_pub, fn_c, _, _) in cells.items():
            pub, cc, red = times[name]
            pub.append(timed(fn_pub))
            if fn_c:
                t0 = time.perf_counter()
                red.append(fn_c())
                cc.append(time.perf_counter() - t0)

    def verify(queries, hits, facets):
        ok = 0
        for i in range(min(args.verify, len(queries))):
            q = queries[i]
            dense = compose_nested(arr.score, q) if isinstance(q, Or) else arr.score(q)
            good = hits.total[i] == np.count_nonzero(dense)
            for f in facets:
                c = codes[f]
                good = good and np.array_equal(hits.facets[f][i], np.bincount(c[(dense > 0) & (c >= 0)],
                                                                              minlength=arr.host.facets[f][1]))
            ok += bool(good)
        return ok

    out = {"docs": n, "queries": nq, "k": args.k, "card": info, "workloads": {}}
    for name, (fn_pub, fn_c, queries, facets) in cells.items():
        pub, cc, red = times[name]
        rec = {"qps": round(nq / float(np.median(pub)), 1)}
        if fn_c:
            rec["c_call_qps"] = round(nq / float(np.median(cc)), 1)
            rec["n_redone"] = int(max(red))
        if facets is not None:
            _, _, hits = fn_pub()
            rec["verified"] = verify(queries, hits, facets)
            rec["sampled"] = min(args.verify, nq)
            rec["mean_total"] = round(float(hits.total.mean()), 1)
        out["workloads"][name] = rec
    w = out["workloads"]
    out["cost_c_call"] = {c: round(w["or"]["c_call_qps"] / w[c]["c_call_qps"], 3)
                          for c in ("or_total", "or_f20", "or_f1024")}
    out["term_total_cost"] = round(w["term"]["qps"] / w["term_total"]["qps"], 3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
