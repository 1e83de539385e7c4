#!/usr/bin/env python
"""Scoring at given documents and window rescoring on the bench corpus: SearchArray.score_docs at the top 1,000 of a
first pass, search_topk(..., rescore=) end to end, and the host combine, against the first pass alone and the
reference's `.score(q)[docs[q]]` composition.

    python tools/rescore_bench.py [--docs 10000000] [--queries 1024] [--window 1000] [--k 10] [--reps 5]

Corpus and terms are bench.py's: the seeded 10M-doc synthetic corpus and its stratified single-term queries; a, b, c
are stratified terms drawn per query with a fixed seed, and `pop` a seeded feature column (an integer in [1, 10000) at
~80 % of docs).  Pass 1 is Or([a, b]) at k = --window.  Rescore workloads, scored at pass 1's docs:
  terms    Bool(should=[Or([a, b, c]), Feature(pop, saturation)])     terms and a feature: no dense row
  phrase   the phrase [a, b] at slop 2                                  pays for one count row per query
Arms, timed alternately (median of --reps after --warmup; the phrase workload, whose count rows make a call take
seconds, --phrase-reps after one warm-up; a host clock around each synchronous call): pass1
(search_topk at k = window), score_docs_c (sa_score_docs_bool on a call prepared once), score_docs (the public call),
rescore (search_topk(k, rescore=Rescore(window)) end to end) and combine (query.rescore_window alone).  dense_row:
the `.score()` composition gathered at the docs, over --dense queries.  Each arm verifies --verify queries against
the dense composition (ids and float32 bits).  The card name and power limit come from a read-only nvidia-smi query
in the same run.  Prints one JSON line.
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
    ap.add_argument("--window", type=int, default=1000)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--verify", type=int, default=4)
    ap.add_argument("--dense", type=int, default=32)
    ap.add_argument("--phrase-reps", type=int, default=1, help="reps (and 1 warm-up) of the phrase workload")
    args = ap.parse_args()

    def log(*a):
        print(f"[rescore_bench +{time.perf_counter() - t_start:.1f}s]", *a, file=sys.stderr, flush=True)
    t_start = time.perf_counter()

    from searcharray_b200 import Bool, Feature, Or, Rescore, SearchArray, bm25_similarity, synth
    from searcharray_b200.query import rescore_window
    info = card()
    spec = synth.SynthSpec(args.docs)
    host, _, _ = synth.generate_shard(spec)
    avgdl = synth.global_avg_doc_length(spec)
    host.avg_doc_length = avgdl
    arr = SearchArray.from_host_index(host, avg_doc_length=avgdl)
    n = len(arr)
    rng = np.random.default_rng(20261018)
    pop = np.where(rng.random(n) < 0.8, rng.integers(1, 10_000, n), 0).astype(np.float32)
    arr.set_feature("pop", pop)
    names = synth.stratified_term_queries(spec, args.queries)
    nq = len(names)
    perm = [rng.permutation(nq) for _ in range(3)]
    a, b, c = ([names[p[i]] for i in range(nq)] for p in perm)
    sat = Feature("pop", "saturation", pivot=500.0)
    sim = bm25_similarity()
    pass1 = [Or([a[i], b[i]]) for i in range(nq)]
    work = {"terms": ([Bool(should=[Or([a[i], b[i], c[i]]), sat]) for i in range(nq)], 0),
            "phrase": ([[a[i], b[i]] for i in range(nq)], 2)}
    W, k = args.window, args.k
    log("corpus ready")
    d1, s1 = arr.search_topk(pass1, k=W)
    score_cache = {}

    def score(cl, slop=0):
        key = (repr(cl), slop)
        if key not in score_cache:
            score_cache[key] = pop_value(cl) if isinstance(cl, Feature) else arr.score(cl, slop=slop)
        return score_cache[key]

    def pop_value(f):
        return f.apply(pop)

    def dense(q, slop=0):
        return compose_nested(lambda cl: score(cl, slop), q if isinstance(q, (Or, Bool)) else Or([q]))

    def verify_docs(queries, slop, got):
        ok = 0
        for i in range(min(args.verify, nq)):
            want = np.where(d1[i] == 0xFFFFFFFF, np.float32(0), dense(queries[i], slop)[np.minimum(d1[i], n - 1)])
            ok += bool(np.array_equal(got[i].view(np.uint32), want.view(np.uint32)))
        score_cache.clear()
        return ok

    def verify_pass1(docs, scores):
        ok = 0
        for i in range(min(args.verify, nq)):
            wd, ws = topk(dense(pass1[i]), W)
            ok += bool(np.array_equal(docs[i], wd) and np.array_equal(scores[i].view(np.uint32), ws.view(np.uint32)))
        score_cache.clear()
        return ok

    def verify_rescore(queries, slop, docs, scores):
        ok = 0
        for i in range(min(args.verify, nq)):
            s2 = np.where(d1[i] == 0xFFFFFFFF, np.float32(0), dense(queries[i], slop)[np.minimum(d1[i], n - 1)])
            wd, ws = rescore_window(d1[i:i + 1], s1[i:i + 1], s2[None], 1.0, 1.0, k)
            ok += bool(np.array_equal(docs[i], wd[0]) and np.array_equal(scores[i].view(np.uint32),
                                                                          ws[0].view(np.uint32)))
        score_cache.clear()
        return ok

    out = {"docs": n, "queries": nq, "window": W, "k": k, "card": info, "workloads": {}}
    for name, (rq, slop) in work.items():
        from searcharray_b200.query import is_boolean
        nodes = [q if is_boolean(q) else Or([q]) for q in rq]
        with arr._shared["lock"]:
            call = arr._prepare_bool(nodes, sim)
        s2 = arr.score_docs(rq, d1, slop=slop)
        log(name, "first score_docs done")
        r = Rescore(rq, window=W, slop=slop)

        def c_call():
            with arr._shared["lock"]:
                return call.score_docs(d1, slop)
        arms = {"pass1": lambda: arr.search_topk(pass1, k=W),
                "score_docs_c": c_call,
                "score_docs": lambda: arr.score_docs(rq, d1, slop=slop),
                "rescore": lambda: arr.search_topk(pass1, k=k, rescore=r),
                "combine": lambda: rescore_window(d1, s1, s2, 1.0, 1.0, k)}
        warmup, reps = (1, args.phrase_reps) if name == "phrase" else (args.warmup, args.reps)
        for fn in arms.values():
            for _ in range(warmup):
                fn()
        log(name, "warm")
        times = {a_: [] for a_ in arms}
        for _ in range(reps):                                # alternating, so the arms see the same machine state
            for a_, fn in arms.items():
                times[a_].append(timed(fn))
            log(name, "rep", {a_: round(t[-1] * 1e3, 2) for a_, t in times.items()})
        ms = {a_: round(1e3 * float(np.median(t)), 3) for a_, t in times.items()}
        res = {"reps": reps, "ms": ms, "qps": {a_: round(nq / (v / 1e3), 1) for a_, v in ms.items()}}
        res["score_docs_over_pass1"] = round(ms["score_docs_c"] / ms["pass1"], 4)
        res["combine_share_of_rescore"] = round(ms["combine"] / ms["rescore"], 4)
        res["verified"] = {"pass1": verify_pass1(*arr.search_topk(pass1, k=W)),
                           "score_docs_c": verify_docs(rq, slop, c_call()),
                           "score_docs": verify_docs(rq, slop, arr.score_docs(rq, d1, slop=slop)),
                           "rescore": verify_rescore(rq, slop, *arr.search_topk(pass1, k=k, rescore=r)),
                           "sampled": min(args.verify, nq)}
        # the reference's idiom: a dense float32[N] row per query, gathered at the docs
        score_cache.clear()
        m = min(args.dense, nq)
        t0 = time.perf_counter()
        for i in range(m):
            dense(rq[i], slop)[np.minimum(d1[i], n - 1)]
            score_cache.clear()
        res["dense_row_qps"] = round(m / (time.perf_counter() - t0), 2)
        out["workloads"][name] = res
        log(name, json.dumps(res))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
