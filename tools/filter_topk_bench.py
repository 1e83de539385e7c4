#!/usr/bin/env python
"""Range and In filter clauses against `where=` masks: SearchArray.search_topk of Bool(must=[Or([a, b])],
filter=[Range(...)] / [In(...)]) on the bench corpus, against Bool(must=[Or([a, b])]) with the same filter as a
document mask built and packed on the host, and against the unfiltered query.

    python tools/filter_topk_bench.py [--docs 10000000] [--queries 1024] [--perq-queries 64] [--k 10] [--reps 5]

Corpus and terms are bench.py's: the seeded 10M-doc synthetic corpus and its stratified single-term queries (a, b:
two random ones per query).  Seeded columns, each in two layouts -- shuffled (random over the docs) and clustered
(increasing with doc id, so whole 8,192-doc tiles fall outside a filter):
  year   a feature, 1900-2024 on 90 % of the docs (0 elsewhere: no value)
  lang   a facet of 32 codes on 90 % of the docs (-1 elsewhere)
Arms, timed alternately within each repetition (host clock around the synchronous public call, median of --reps):
  range_shared / mask_shared     Range(year, gte=1977, lt=1990) for every query / its mask, one for the batch
  range_perq / mask_perq         a different 13-year range per query / its (Q, N) mask, over --perq-queries queries
                                 (a mask of 10M docs is 1.25 MB packed per query; its packing and copy are timed)
  in_shared / isin_shared        In(lang, [0, 1]) / np.isin mask, one for the batch
  in_perq / isin_perq            two random codes per query / their masks, over --perq-queries queries
  none                           the unfiltered Bool(must=[Or([a, b])])
Per layout: filter_tiles, the (query, tile) pairs sa_stats counted as skipped by an absent range / In, in one
range_shared and one in_shared call.  Every filter arm is verified: a sample of its queries must give the ids and score
bits of its mask arm.  The card name and power limit come from a read-only nvidia-smi query in the same run.  Prints
one JSON line.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--perq-queries", type=int, default=64)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--verify", type=int, default=8)
    args = ap.parse_args()

    from searcharray_b200 import Bool, In, Or, Range, SearchArray, _lib
    from searcharray_b200 import synth
    info = card()
    spec = synth.SynthSpec(args.docs)
    host, _, _ = synth.generate_shard(spec)
    avgdl = synth.global_avg_doc_length(spec)
    host.avg_doc_length = avgdl
    arr = SearchArray.from_host_index(host, avg_doc_length=avgdl)
    n = len(arr)
    names = synth.stratified_term_queries(spec, args.queries)
    nq = len(names)
    rng = np.random.default_rng(20261018)
    pa, pb = rng.permutation(nq), rng.permutation(nq)
    base = [Or([names[pa[i]], names[pb[i]]]) for i in range(nq)]
    n_pq = min(args.perq_queries, nq)
    present = rng.random(n) < 0.9
    ids = np.arange(n)
    layouts = {
        "shuffled": (np.where(present, rng.integers(1900, 2025, n), 0).astype(np.float32),
                     np.where(present, rng.integers(0, 32, n), -1).astype(np.int32)),
        "clustered": (np.where(present, 1900 + ids * 125 // n, 0).astype(np.float32),
                      np.where(present, ids * 32 // n, -1).astype(np.int32)),
    }
    y0 = rng.integers(1900, 2012, n_pq)
    codes = [sorted(rng.choice(32, 2, replace=False).tolist()) for _ in range(n_pq)]
    h = arr._device().handle
    out = {"card": info, "docs": n, "k": args.k, "queries": nq, "perq_queries": n_pq, "reps": args.reps,
           "warmup": args.warmup, "layouts": {}}

    def filt(qs, cs):
        return [Bool(must=[q], filter=[c]) for q, c in zip(qs, cs)]
    plain = [Bool(must=[q]) for q in base]
    for lname, (year, lang) in layouts.items():
        arr.set_feature(f"year_{lname}", year)
        arr.set_facet(f"lang_{lname}", lang, 32)
        yr, lg = f"year_{lname}", f"lang_{lname}"
        shared_r = Range(yr, gte=1977, lt=1990)
        shared_i = In(lg, [0, 1])
        perq_r = [Range(yr, gte=int(y), lt=int(y) + 13) for y in y0]
        perq_i = [In(lg, c) for c in codes]
        arms = {
            "range_shared": lambda: arr.search_topk(filt(base, [shared_r] * nq), k=args.k),
            "mask_shared": lambda: arr.search_topk(plain, k=args.k, where=shared_r.match(year)),
            "range_perq": lambda: arr.search_topk(filt(base[:n_pq], perq_r), k=args.k),
            "mask_perq": lambda: arr.search_topk(plain[:n_pq], k=args.k,
                                                 where=np.stack([r.match(year) for r in perq_r])),
            "in_shared": lambda: arr.search_topk(filt(base, [shared_i] * nq), k=args.k),
            "isin_shared": lambda: arr.search_topk(plain, k=args.k, where=shared_i.match(lang)),
            "in_perq": lambda: arr.search_topk(filt(base[:n_pq], perq_i), k=args.k),
            "isin_perq": lambda: arr.search_topk(plain[:n_pq], k=args.k,
                                                 where=np.stack([c.match(lang) for c in perq_i])),
            "none": lambda: arr.search_topk(plain, k=args.k),
        }
        queries = {a: (nq if "shared" in a or a == "none" else n_pq) for a in arms}
        # verification: each filter arm's sample against its mask arm, bit for bit
        sample = list(range(0, n_pq, max(1, n_pq // args.verify)))[:args.verify]
        for c_of, m_of, what in ((lambda i: shared_r, lambda i: shared_r.match(year), "range_shared"),
                                 (lambda i: perq_r[i], lambda i: perq_r[i].match(year), "range_perq"),
                                 (lambda i: shared_i, lambda i: shared_i.match(lang), "in_shared"),
                                 (lambda i: perq_i[i], lambda i: perq_i[i].match(lang), "in_perq")):
            d1, s1 = arr.search_topk(filt([base[i] for i in sample], [c_of(i) for i in sample]), k=args.k)
            d2, s2 = arr.search_topk([plain[i] for i in sample], k=args.k,
                                     where=np.stack([m_of(i) for i in sample]))
            if not (np.array_equal(d1, d2) and np.array_equal(s1.view(np.uint32), s2.view(np.uint32))):
                raise SystemExit(f"{lname} / {what}: differs from its mask arm")
        skipped = {}
        for what, c in (("range_shared", shared_r), ("in_shared", shared_i)):
            _lib.check(_lib.lib().sa_stats_reset(h))
            arr.search_topk(filt(base, [c] * nq), k=args.k)
            st = _lib.SaStats()
            _lib.check(_lib.lib().sa_stats_get(h, st))
            skipped[what] = int(st.filter_tiles)
        for _ in range(args.warmup):
            for fn in arms.values():
                fn()
        times = {a: [] for a in arms}
        for _ in range(args.reps):
            for a, fn in arms.items():
                t0 = time.perf_counter()
                fn()
                times[a].append(time.perf_counter() - t0)
        cells = {}
        for a in arms:
            t = float(np.median(times[a]))
            cells[a] = {"queries": queries[a], "ms": 1e3 * t, "qps": queries[a] / t,
                        "verified": len(sample) if a not in ("none",) and not a.startswith(("mask", "isin")) else 0}
        out["layouts"][lname] = {"cells": cells, "filter_tiles": skipped, "n_tiles": (n + 8191) // 8192}
        print(f"[filter_topk_bench] {lname}: {json.dumps(out['layouts'][lname])}", file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
