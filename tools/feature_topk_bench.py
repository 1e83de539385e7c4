#!/usr/bin/env python
"""Feature clauses in batched boolean queries: search_topk / fields_topk with a per-document feature column on the
bench corpus, against the same queries without the feature and against composing on the host.

    python tools/feature_topk_bench.py [--docs 10000000] [--queries 1024] [--k 10] [--reps 5] [--verify 4]

Corpus and terms are bench.py's: the seeded 10M-doc synthetic corpus and its stratified single-term queries.  The
feature `pop` is seeded: an integer in [1, 10000) at ~80 % of docs, 0 elsewhere.  Workloads (a, b: random
stratified terms):
  bool          Bool(must=[Or([a, b])])                                      (no feature: the OCCUR instance)
  bool_sat      Bool(must=[Or([a, b])], should=[Feature(pop, saturation)])   (timed alternating with `bool`)
  or_log        Or([a, Feature(pop, log)])                  (the feature is present in every tile: every tile folds)
  fields        fields_topk: Bool(must=[Field(body, a)], should=[Field(title, b), Field(body, Feature(pop, saturation))]),
                `title` a second name of the body column (one index)
  range10       bool_sat with where= a contiguous 10 % of the doc ids
Per workload: qps (the public call, host clock around the synchronous call, median of --reps), c_call_qps
(sa_score_batch_topk_bool / sa_multi_score_batch_topk_bool on arrays prepared once), n_redone (queries re-run exactly
in the timed C calls) and verified (queries of a sample whose ids and score bits equal the top k of the numpy
composition).  compose_qps: .score per clause + Feature.apply + the composition + argpartition on the host, over
--compose bool_sat queries.  The card name and power limit come from a read-only nvidia-smi query in the same run.
Prints one JSON line.
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
    ap.add_argument("--compose", type=int, default=32)
    args = ap.parse_args()

    import pandas as pd
    from searcharray_b200 import Bool, Feature, Field, Or, SearchArray, bm25_similarity, fields_topk
    from searcharray_b200 import synth
    from searcharray_b200.postings import _PreparedBool, pack_where
    from searcharray_b200.solr import _clause_slots, _fields_plan, _locked, _multi_for
    info = card()
    spec = synth.SynthSpec(args.docs)
    host, _, _ = synth.generate_shard(spec)
    avgdl = synth.global_avg_doc_length(spec)
    host.avg_doc_length = avgdl
    arr = SearchArray.from_host_index(host, avg_doc_length=avgdl)
    n = len(arr)
    rng = np.random.default_rng(20261017)
    pop = np.where(rng.random(n) < 0.8, rng.integers(1, 10_000, n), 0).astype(np.float32)
    arr.set_feature("pop", pop)
    names = synth.stratified_term_queries(spec, args.queries)
    perm = [rng.permutation(len(names)) for _ in range(2)]
    nq = len(names)
    sat, lg = Feature("pop", "saturation", pivot=500.0), Feature("pop", "log", scaling_factor=1.0)
    sim = bm25_similarity()

    def t(i, j):
        return names[perm[j][i % nq]]
    work = {
        "bool": [Bool(must=[Or([t(i, 0), t(i, 1)])]) for i in range(nq)],
        "bool_sat": [Bool(must=[Or([t(i, 0), t(i, 1)])], should=[sat]) for i in range(nq)],
        "or_log": [Or([t(i, 0), lg]) for i in range(nq)],
    }
    frame = pd.DataFrame({"body": arr})
    frame["title"] = frame["body"]
    fields_q = [Bool(must=[Field("body", t(i, 0))], should=[Field("title", t(i, 1)), Field("body", sat)])
                for i in range(nq)]
    range10 = np.zeros(n, dtype=bool)
    range10[n // 2: n // 2 + n // 10] = True
    score_cache = {}

    def score(c):
        key = repr(c)
        if key not in score_cache:
            inner = c.clause if isinstance(c, Field) else c
            score_cache[key] = inner.apply(pop) if isinstance(inner, Feature) else arr.score(inner)
        return score_cache[key]

    def prepared(queries, bits=None):
        """The C call of search_topk(queries) on arrays prepared once: fn() -> n_redone."""
        call = arr._prepare_bool(queries, sim, None if bits is None else pack_where(bits, n, len(queries)))
        return lambda: call.run(args.k, 0)[2]

    def verify(queries, docs, scores, where=None):
        ok = 0
        for i in range(min(args.verify, len(queries))):
            dense = compose_nested(score, queries[i])
            if where is not None:
                dense = np.where(where, dense, np.float32(0))
            wd, ws = topk(dense, args.k)
            ok += bool(np.array_equal(docs[i], wd) and np.array_equal(scores[i].view(np.uint32), ws.view(np.uint32)))
        return ok

    out = {"docs": n, "queries": nq, "k": args.k, "card": info, "workloads": {}}
    cells = {
        "bool": (lambda: arr.search_topk(work["bool"], k=args.k), prepared(work["bool"]), work["bool"], None),
        "bool_sat": (lambda: arr.search_topk(work["bool_sat"], k=args.k), prepared(work["bool_sat"]),
                     work["bool_sat"], None),
        "or_log": (lambda: arr.search_topk(work["or_log"], k=args.k), prepared(work["or_log"]), work["or_log"], None),
        "range10": (lambda: arr.search_topk(work["bool_sat"], k=args.k, where=range10),
                    prepared(work["bool_sat"], range10), work["bool_sat"], range10),
    }
    batch, slot_of, arrays, sims = _fields_plan(frame, fields_q, sim)
    multi = _multi_for(arrays)
    fields_call = _PreparedBool(arrays, sims, _clause_slots(batch, slot_of), fields_q, batch, multi=multi)

    def fields_c():
        with _locked(multi, arrays):
            return fields_call.run(args.k, 0)[2]
    cells["fields"] = (lambda: fields_topk(frame, fields_q, k=args.k), fields_c, fields_q, None)
    for fn_pub, fn_c, _, _ in cells.values():            # warm every shape
        for _ in range(args.warmup):
            fn_pub()
            fn_c()
    times = {name: ([], [], []) for name in cells}
    for _ in range(args.reps):                           # alternating, so the pairs see the same machine state
        for name, (fn_pub, fn_c, _, _) in cells.items():
            pub, cc, red = times[name]
            pub.append(timed(fn_pub))
            t0 = time.perf_counter()
            red.append(fn_c())
            cc.append(time.perf_counter() - t0)
    for name, (fn_pub, _, queries, where) in cells.items():
        pub, cc, red = times[name]
        docs, scores = fn_pub()
        out["workloads"][name] = {"qps": round(nq / float(np.median(pub)), 1),
                                  "c_call_qps": round(nq / float(np.median(cc)), 1),
                                  "n_redone": int(max(red)), "verified": verify(queries, docs, scores, where),
                                  "sampled": min(args.verify, nq)}
    w = out["workloads"]
    out["feature_cost_c_call"] = round(w["bool"]["c_call_qps"] / w["bool_sat"]["c_call_qps"], 3)
    qs = work["bool_sat"][:args.compose]
    score_cache.clear()
    t0 = time.perf_counter()
    for q in qs:
        d = compose_nested(score, q)
        top = np.argpartition(d, -args.k)[-args.k:]
        top[np.argsort(-d[top], kind="stable")]
        score_cache.clear()
    out["compose_qps"] = round(len(qs) / (time.perf_counter() - t0), 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
