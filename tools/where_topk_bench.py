#!/usr/bin/env python
"""Filtered batched top-k: SearchArray.search_topk(queries, where=mask) on the bench corpus, against the same batch
without a mask and against composing the filter on the host.

    python tools/where_topk_bench.py [--docs 10000000] [--queries 1024] [--k 10] [--reps 5] [--perq-queries 64]
                                     [--workloads term,or2,and2,bool,or_of_ands,phrase]

Corpus and terms are bench.py's: the seeded 10M-doc synthetic corpus and its 1,024 stratified single-term queries.
Workloads (a, b, c, d: random stratified terms):
  term          a                                    (plain; with a mask, a one-clause Or through the boolean fold)
  or2, and2     Or([a, b]), And([a, b])
  bool          Bool(must=[a], should=[b], must_not=[c])
  or_of_ands    Or([And([a, b]), And([c, d])])
  phrase        the phrase [a, b] (slop 0)
Masks: none (today's call, no `where`), all (all true), rand50 / rand10 / rand1 (random docs), range10 (a contiguous
10% of the doc ids), perq10 (a different random 10% per query, over the first --perq-queries queries: a (Q, N) mask
of 10M docs is 1.25 MB packed per query and N bytes per query as numpy bools).
Per (workload, mask) cell:
  qps           the public call, host clock around the synchronous call (packing the mask included), median of --reps
  c_call_qps    sa_score_batch_topk_bool on arrays and a mask packed once (the mask's upload included);
                for `none`: sa_score_batch_topk for term and phrase, and for the boolean workloads the same
                prepared call without a mask (the unmasked instances)
  n_redone      queries re-run exactly in the timed C calls (candidate overflow)
  verified      queries of a sample whose ids and score bits equal the top k of np.where(mask, S_q, 0)
Per workload, compose_qps: .score per clause + the boolean composition + np.where + np.argpartition on the host, over
32 queries under rand10.  The card name and power limit come from a read-only nvidia-smi query in the same run.
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
    ap.add_argument("--perq-queries", type=int, default=64)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--verify", type=int, default=4)
    ap.add_argument("--compose", type=int, default=32)
    ap.add_argument("--workloads", default="term,or2,and2,bool,or_of_ands,phrase")
    args = ap.parse_args()

    from searcharray_b200 import And, Bool, Or, SearchArray, _lib, bm25_similarity, compute_idf
    from searcharray_b200 import synth
    from searcharray_b200.postings import pack_where
    info = card()
    spec = synth.SynthSpec(args.docs)
    host, _, _ = synth.generate_shard(spec)
    avgdl = synth.global_avg_doc_length(spec)
    host.avg_doc_length = avgdl
    arr = SearchArray.from_host_index(host, avg_doc_length=avgdl)
    n = len(arr)
    names = synth.stratified_term_queries(spec, args.queries)
    rng = np.random.default_rng(20261017)
    perm = [rng.permutation(len(names)) for _ in range(4)]
    nq = len(names)

    def t(i, j):
        return names[perm[j][i % nq]]
    work = {
        "term": lambda i: t(i, 0),
        "or2": lambda i: Or([t(i, 0), t(i, 1)]),
        "and2": lambda i: And([t(i, 0), t(i, 1)]),
        "bool": lambda i: Bool(must=[t(i, 0)], should=[t(i, 1)], must_not=[t(i, 2)]),
        "or_of_ands": lambda i: Or([And([t(i, 0), t(i, 1)]), And([t(i, 2), t(i, 3)])]),
        "phrase": lambda i: [t(i, 0), t(i, 1)],
    }
    ids = np.arange(n)
    masks = {
        "none": None,
        "all": np.ones(n, dtype=bool),
        "rand50": rng.random(n) < 0.5,
        "rand10": rng.random(n) < 0.1,
        "rand1": rng.random(n) < 0.01,
        "range10": (ids >= int(n * 0.45)) & (ids < int(n * 0.55)),
    }
    n_pq = min(args.perq_queries, nq)
    sim = bm25_similarity()
    out = {"card": info, "docs": n, "k": args.k, "queries": nq, "perq_queries": n_pq, "reps": args.reps,
           "warmup": args.warmup, "workloads": {}}
    h = arr._device().handle

    for label in args.workloads.split(","):
        qs = [work[label](i) for i in range(nq)]
        sample_i = list(range(0, n_pq, max(1, n_pq // args.verify)))[:args.verify]
        dense = {i: compose_nested(arr.score, qs[i]) if not isinstance(qs[i], (str, list))
                 else np.asarray(arr.score(qs[i]), dtype=np.float32) for i in sample_i}
        cells = {}
        for mname in list(masks) + ["perq10"]:
            if mname == "perq10":
                m = np.random.default_rng(7).random((n_pq, n)) < 0.1
                batch = qs[:n_pq]
            else:
                m, batch = masks[mname], qs
            d, s = arr.search_topk([batch[i] for i in sample_i], k=args.k, where=None if m is None else (
                m[sample_i] if m is not None and m.ndim == 2 else m))
            for j, i in enumerate(sample_i):
                mq = True if m is None else (m[i] if m.ndim == 2 else m)
                wd, ws = topk(np.where(mq, dense[i], np.float32(0)), args.k)
                if not (np.array_equal(d[j], wd) and np.array_equal(s[j].view(np.uint32), ws.view(np.uint32))):
                    raise SystemExit(f"{label} / {mname}: differs from the masked composition for {batch[i]!r}")
            t_api = median_time(lambda: arr.search_topk(batch, k=args.k, where=m), args.warmup, args.reps)
            redone = []
            if m is None and isinstance(batch[0], (str, list)):
                # today's plain batch: sa_score_batch_topk, as search_topk calls it
                terms, starts, idfs = arr._topk_queries(batch, lambda x: compute_idf(arr.corpus_size, x))
                idfs = np.asarray(idfs, dtype=np.float32)
                dd = np.empty((len(batch), args.k), dtype=np.uint32)
                ss = np.empty((len(batch), args.k), dtype=np.float32)
                t_c = median_time(lambda: _lib.check(_lib.lib().sa_score_batch_topk(
                    h, _lib.p_u32(terms), _lib.p_u32(starts), _lib.p_f32(idfs), len(idfs), 0, arr.avg_doc_length,
                    sim.k1, sim.b, args.k, _lib.p_u32(dd), _lib.p_f32(ss))), args.warmup, args.reps)
            else:
                # for `none`, the same prepared call without a mask: the unmasked instances, for a kernel-level
                # comparison
                call = arr._prepare_bool(batch, sim, None if m is None else pack_where(m, n, len(batch)))
                t_c = median_time(lambda: redone.append(call.run(args.k, 0)[2]), args.warmup, args.reps)
            cells[mname] = {"queries": len(batch), "qps": len(batch) / t_api, "c_call_qps": len(batch) / t_c,
                            "n_redone": redone[-args.reps:], "verified": len(sample_i)}
            print(f"[where_topk_bench] {label} {mname}: {json.dumps(cells[mname])}", file=sys.stderr, flush=True)
        # the host composition a user writes today, under rand10
        m = masks["rand10"]

        def compose():
            for q in qs[:args.compose]:
                v = compose_nested(arr.score, q) if not isinstance(q, (str, list)) else arr.score(q)
                v = np.where(m, v, np.float32(0))
                np.argpartition(v, -args.k)[-args.k:]
        t_comp = median_time(compose, 1, 3)
        out["workloads"][label] = {"cells": cells, "compose_qps": args.compose / t_comp}
        print(f"[where_topk_bench] {label} compose_qps {args.compose / t_comp:.2f}", file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
