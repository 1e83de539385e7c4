#!/usr/bin/env python
"""Batched top-k at depth: SearchArray.search_topk at k = 10, 100 and 1000 on the bench corpus.

    python tools/deep_topk_bench.py [--docs 10000000] [--queries 1024] [--ks 10,100,1000] [--reps 5]

Corpus and terms are bench.py's: the seeded 10M-doc synthetic corpus and its 1,024 stratified single-term queries.
Workloads: term (the stratified terms), or2 (Or([a, b]) of two stratified terms), view (the terms on arr[::2]).
Per (workload, k) cell:
  qps             queries / s of the public call, host clock around the synchronous call, median of --reps
  term_ms, topk_ms, phrase_ms   one profiled call's CUDA-event times from sa_stats: the term scan, the top-k
                  kernels (select, and the view path's sim tile kernels), the phrase kernels
  deep_tiles      (query, tile) pairs the deep collector took in that call
  cand_bytes_per_query   candidate bytes a query's tiles write: tiles * slots * 8 (slots = k above 32, else 128/256)
  verified        sampled queries whose ids and score bits equal the top k of .score (or the Or composition)
The card name and power limit come from a read-only nvidia-smi query in the same run.  Prints one JSON line.
"""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from view_topk_bench import card  # noqa: E402


def expected(dense, k):
    nz = np.flatnonzero(dense > 0)
    order = nz[np.lexsort((nz, -dense[nz].astype(np.float64)))][:k]
    return order.astype(np.uint32), dense[order]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--ks", default="10,100,1000")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--verify", type=int, default=4)
    args = ap.parse_args()

    from searcharray_b200 import Or, SearchArray, _lib, synth
    info = card()
    spec = synth.SynthSpec(args.docs)
    host, _, _ = synth.generate_shard(spec)
    avgdl = synth.global_avg_doc_length(spec)
    host.avg_doc_length = avgdl
    arr = SearchArray.from_host_index(host, avg_doc_length=avgdl)
    names = synth.stratified_term_queries(spec, args.queries)
    rng = np.random.default_rng(20261018)
    other = [names[i] for i in rng.permutation(len(names))]
    view = arr[::2]
    pairs = list(zip(names, other))
    work = {"term": (arr, list(names)), "or2": (arr, [Or([a, b]) for a, b in pairs]), "view": (view, list(names))}
    n_tiles = (len(arr) + 8191) // 8192
    out = {"card": info, "docs": len(arr), "queries": len(names), "reps": args.reps, "cells": {}}
    for label, (a, qs) in work.items():
        h = a._device().handle
        sample = list(range(0, len(qs), max(1, len(qs) // args.verify)))[:args.verify]
        dense = {i: (a.score(pairs[i][0]) + a.score(pairs[i][1])).astype(np.float32) if label == "or2"
                 else np.asarray(a.score(qs[i]), dtype=np.float32) for i in sample}
        tiles = (len(a) + 8191) // 8192
        for k in (int(x) for x in args.ks.split(",")):
            for _ in range(args.warmup):
                a.search_topk(qs, k=k)
            _lib.check(_lib.lib().sa_set_profiling(h, 1))
            _lib.check(_lib.lib().sa_stats_reset(h))
            a.search_topk(qs, k=k)
            st = _lib.SaStats()
            _lib.check(_lib.lib().sa_stats_get(h, ctypes.byref(st)))
            _lib.check(_lib.lib().sa_set_profiling(h, 0))
            times = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                docs, scores = a.search_topk(qs, k=k)
                times.append(time.perf_counter() - t0)
            ok = 0
            for i in sample:
                wd, ws = expected(dense[i], k)
                ok += bool(np.array_equal(docs[i][:len(wd)], wd) and
                           np.array_equal(scores[i][:len(ws)].view(np.uint32), ws.view(np.uint32)) and
                           np.all(docs[i][len(wd):] == 0xFFFFFFFF))
            slots = k if k > 32 else (128 if k <= 16 else 256)
            out["cells"][f"{label}@{k}"] = {
                "qps": len(qs) / float(np.median(times)),
                "term_ms": st.term_kernel_ms, "topk_ms": st.topk_kernel_ms, "phrase_ms": st.phrase_kernel_ms,
                "deep_tiles": st.deep_tiles,
                "cand_bytes_per_query": tiles * slots * 8,
                "verified": f"{ok}/{len(sample)}"}
    out["n_tiles"] = n_tiles
    print(json.dumps(out))


if __name__ == "__main__":
    main()
