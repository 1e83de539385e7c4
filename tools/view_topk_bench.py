#!/usr/bin/env python
"""search_topk on views of the bench corpus, against the unsliced array and against today's alternative.

    python tools/view_topk_bench.py [--docs 10000000] [--queries 1024] [--k 10] [--reps 5]

Corpus and queries are bench.py's: the seeded 10M-doc synthetic corpus and its 1,024 stratified single-term
queries.  Arrays: the unsliced array, arr[:N//2], a 10 % and a 1 % random mask.  Per array, after a sample of its
results has been checked against view.score (positions and score bits):
  qps            search_topk over the whole batch, host clock around the synchronous call, after warm-up;
  docfreq_ms     one sa_docfreq_rows_batch over the batch's distinct terms (views only);
  bytes / gbs    algorithmic bytes per term query and the rate they are moved at over the whole call: views
                 P + 4*N + 12*len(view) + 4*df*len(view)/N (the tf scan in doc space, its row, then row index and
                 gathered count per position, and the doc length of each position with a count), the unsliced path
                 DESIGN.md 3.1's P + 4*df + 4*N; P = 4*df for terms with a tf table, 8*W for the others;
  score_argpartition_qps   the alternative a view had before: view.score(q) + np.argpartition, for 32 queries.
The card name and power limit come from a read-only nvidia-smi query in the same run.  Prints one JSON line.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=60).stdout.strip().splitlines()
        name, limit = (x.strip() for x in out[0].split(","))
        return {"name": name, "power_limit": limit}
    except Exception as e:                      # the numbers are still printed, without the card
        return {"name": None, "power_limit": None, "error": str(e)}


def expected_topk(dense, k):
    nz = np.flatnonzero(dense > 0)
    order = nz[np.lexsort((nz, -dense[nz].astype(np.float64)))][:k]
    docs = np.full(k, 0xFFFFFFFF, dtype=np.uint32)
    scores = np.zeros(k, dtype=np.float32)
    docs[:len(order)] = order
    scores[:len(order)] = dense[order]
    return docs, scores


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=10_000_000)
    ap.add_argument("--queries", type=int, default=1024)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--verify", type=int, default=16, help="queries per array checked against view.score")
    ap.add_argument("--baseline-queries", type=int, default=32)
    args = ap.parse_args()

    from searcharray_b200 import SearchArray, _lib, synth
    info = card()
    spec = synth.SynthSpec(args.docs)
    host, _, _ = synth.generate_shard(spec)
    avgdl = synth.global_avg_doc_length(spec)
    host.avg_doc_length = avgdl
    arr = SearchArray.from_host_index(host, avg_doc_length=avgdl)
    names = synth.stratified_term_queries(spec, args.queries)
    tids = np.asarray([spec.term_index[n] for n in names], dtype=np.uint32)
    n = host.n_docs

    # term-scan bytes P per query (DESIGN.md 3.1): the tf table exists for lists with a tile directory
    n_tiles = (n + 8191) // 8192
    dir_min = max(1024, n_tiles // 2)
    lens = np.asarray(host.term_lengths, dtype=np.int64)[tids]
    df = np.asarray([int(arr.docfreq(nm)) for nm in names], dtype=np.int64)
    P = np.where((lens >= dir_min) & (lens < 0xFFFFFFFF), 4 * df, 8 * lens)

    rng = np.random.default_rng(20261015)
    arrays = {"unsliced": arr, "first_half": arr[:n // 2], "mask_10pct": arr[rng.random(n) < 0.10],
              "mask_1pct": arr[rng.random(n) < 0.01]}
    out = {"card": info, "docs": n, "queries": len(names), "k": args.k, "reps": args.reps, "arrays": {}}
    for label, view in arrays.items():
        sliced = view.rows is not None
        sample = names[::max(1, len(names) // args.verify)][:args.verify]
        d, s = view.search_topk(sample, k=args.k)
        for i, q in enumerate(sample):
            wd, ws = expected_topk(view.score(q), args.k)
            if not (np.array_equal(d[i], wd) and np.array_equal(s[i].view(np.uint32), ws.view(np.uint32))):
                raise SystemExit(f"{label}: search_topk differs from view.score top-k for {q!r}")
        for _ in range(args.warmup):
            view.search_topk(names, k=args.k)
        times = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            view.search_topk(names, k=args.k)
            times.append(time.perf_counter() - t0)
        t_best, t_med = min(times), float(np.median(times))
        rec = {"rows": len(view), "verified_queries": len(sample), "qps_median": len(names) / t_med,
               "qps_best": len(names) / t_best, "ms_per_batch_median": 1e3 * t_med}
        if sliced:
            per_query = P + 4 * n + 12 * len(view) + 4 * df * len(view) / n
            dev = view._device()
            uniq = np.unique(tids)
            dfs = np.zeros(len(uniq), dtype=np.uint64)
            df_times = []
            with view._shared["lock"]:
                view._apply_rows(dev)
                for _ in range(args.warmup + args.reps):
                    t0 = time.perf_counter()
                    _lib.check(_lib.lib().sa_docfreq_rows_batch(dev.handle, _lib.p_u32(uniq), len(uniq),
                                                                _lib.p_u64(dfs)))
                    df_times.append(time.perf_counter() - t0)
            rec["docfreq_terms"] = len(uniq)
            rec["docfreq_ms_median"] = 1e3 * float(np.median(df_times[args.warmup:]))
        else:
            per_query = P + 4 * df + 4 * n
        rec["bytes_per_query_mean"] = float(per_query.mean())
        rec["gbs_median"] = float(per_query.sum()) / t_med / 1e9
        # today's alternative on a view: the dense score vector to the host, argpartition there
        bq = names[:args.baseline_queries]
        t0 = time.perf_counter()
        for q in bq:
            sc = view.score(q)
            top = np.argpartition(-sc, args.k)[:args.k] if len(sc) > args.k else np.arange(len(sc))
            top[np.argsort(-sc[top], kind="stable")]
        rec["score_argpartition_qps"] = len(bq) / (time.perf_counter() - t0)
        out["arrays"][label] = rec
        print(f"[view_topk_bench] {label}: {json.dumps(rec)}", file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
