#!/usr/bin/env python
"""Collapsed batched top-k: search_topk with `collapse=` on the bench corpus, against the same queries without it.

    python tools/collapse_topk_bench.py [--docs 10000000] [--queries 1024] [--reps 5] [--verify 4]

Corpus and terms are bench.py's: the seeded 10M-doc synthetic corpus and its stratified single-term queries, here
as 1,024 Or([a, b]) queries of two random stratified terms.  Group columns (seeded): `random`, N/8 groups drawn at
random; `clustered`, doc // 16 (runs of 16 neighbouring docs); `dominant`, one group holding half the docs, the others
in groups of their own.  Arms, timed alternating in one run at k = 10 and k = 100: `or` (no collapse) and one per
group column.  Per arm: ms per call and q/s (host clock around the synchronous public call, median of --reps),
device_ms (CUDA events on the library's stream around the prepared C call: the tile kernels and the select),
select_ms (the select kernel's CUDA-event time, sa_stats.topk_kernel_ms with profiling on), the collapse windows
past the first per call, and verified: sampled queries equal to the numpy collapse of the composed dense vector.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from view_topk_bench import card  # noqa: E402
from _nested_compose import compose_nested  # noqa: E402
from test_collapse_cpu import collapse_ref  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--verify", type=int, default=4)
    args = ap.parse_args()

    from searcharray_b200 import Or, SearchArray, _lib, bm25_similarity
    from searcharray_b200 import synth
    info = card()
    spec = synth.SynthSpec(args.docs)
    host, _, _ = synth.generate_shard(spec)
    avgdl = synth.global_avg_doc_length(spec)
    host.avg_doc_length = avgdl
    arr = SearchArray.from_host_index(host, avg_doc_length=avgdl)
    n = len(arr)
    rng = np.random.default_rng(20261019)
    codes = {"random": rng.integers(0, max(1, n // 8), n), "clustered": np.arange(n) // 16,
             "dominant": np.where(rng.random(n) < 0.5, 0, np.arange(n) + 1)}
    for name, c in codes.items():
        arr.set_group(name, c)
    names = synth.stratified_term_queries(spec, args.queries)
    perm = [rng.permutation(len(names)) for _ in range(2)]
    nq = len(names)
    ors = [Or([names[perm[0][i]], names[perm[1][i]]]) for i in range(nq)]
    sim = bm25_similarity()
    dev = arr._device()
    lib = _lib.lib()
    st = _lib.SaStats()

    def device_call(k, group):
        """The prepared C call of search_topk(ors, k, collapse=group): fn() -> (event ms, select ms, windows)."""
        call = arr._prepare_bool(ors, sim, collapse=group)

        def fn():
            ms = ctypes.c_double()
            _lib.check(lib.sa_stats_reset(dev.handle))
            _lib.check(lib.sa_timer_start(dev.handle))
            call.run(k, 0)
            _lib.check(lib.sa_timer_stop(dev.handle, ctypes.byref(ms)))
            _lib.check(lib.sa_stats_get(dev.handle, ctypes.byref(st)))
            return ms.value, st.topk_kernel_ms, st.collapse_windows
        return fn

    _lib.check(lib.sa_set_profiling(dev.handle, 1))
    arms = {}
    for k in (10, 100):
        for group in (None,) + tuple(codes):
            arms[(k, group)] = (lambda k=k, group=group: arr.search_topk(ors, k=k, collapse=group),
                                device_call(k, group))
    for pub, dc in arms.values():                        # warm every shape
        for _ in range(args.warmup):
            pub()
            dc()
    times = {a: ([], []) for a in arms}
    for _ in range(args.reps):                           # alternating, so the arms see the same machine state
        for a, (pub, dc) in arms.items():
            t0 = time.perf_counter()
            pub()
            times[a][0].append(time.perf_counter() - t0)
            times[a][1].append(dc())
    out = {"docs": n, "queries": nq, "card": info, "arms": {}}
    for (k, group), (pub, _) in arms.items():
        wall, dcs = times[(k, group)]
        rec = {"k": k, "collapse": group, "ms_per_call": round(1e3 * float(np.median(wall)), 2),
               "qps": round(nq / float(np.median(wall)), 1),
               "device_ms": round(float(np.median([d[0] for d in dcs])), 2),
               "select_ms": round(float(np.median([d[1] for d in dcs])), 2),
               "windows_past_first": int(max(d[2] for d in dcs))}
        if group is not None:
            docs, scores = pub()
            ok = 0
            for i in range(min(args.verify, nq)):
                wd, ws = collapse_ref(compose_nested(arr.score, ors[i]), codes[group], k)
                ok += bool(np.array_equal(docs[i], wd) and np.array_equal(scores[i].view(np.uint32), ws.view(np.uint32)))
            rec["verified"] = ok
            rec["sampled"] = min(args.verify, nq)
        out["arms"][f"k{k}_{group or 'none'}"] = rec
    for k in (10, 100):
        base = out["arms"][f"k{k}_none"]["device_ms"]
        out[f"device_cost_k{k}"] = {g: round(out["arms"][f"k{k}_{g}"]["device_ms"] / base, 3) for g in codes}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
