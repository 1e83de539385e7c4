#!/usr/bin/env python
"""Boolean queries over two DataFrame fields (solr.fields_topk, sa_multi_score_batch_topk_bool) on the bench corpus,
next to the same clauses as a single-field Bool (search_topk) measured in the same run.

    python tools/fields_topk_bench.py [--docs 10000000] [--queries 1024] [--phrase-queries 64] [--k 10] [--reps 5]

Corpus and terms are bench.py's: the seeded 10M-doc synthetic corpus and its 1,024 stratified single-term queries.  The
corpus is uploaded as TWO columns with identical data, f1 and f2, so a query split across them moves the same bytes
as the same query on one column and must give the same ids and score bits.  Workloads (a, b, c, d: random stratified
terms; rare / common: the rarest and the most common df bucket, as tools/bool_occur_bench.py):
  must_a_b_c         +f1:a f2:b f2:c                Bool(must=[f1:a], should=[f2:b, f2:c])
  most_fields        f1:a^2 f2:a                    Or([f1:a^2, f2:a])
  a_b_not_c          f1:a f1:b -f2:c                Bool(should=[f1:a, f1:b], must_not=[f2:c])
  must_rare_common   +f1:rare f2:common             Bool(must=[f1:rare], should=[f2:common]): a MUST on one field
                                                    prunes the tiles of a clause on the other
  phrase_f2          f1:a f1:b -f2:"c d"            in its own, smaller batch (each phrase row is built synchronously)
Per workload, after a sample has been checked against the composition of per-field .score and the whole batch
against the single-field Bool (ids and score bits):
  qps               fields_topk, host clock around the synchronous call, median of --reps after --warmup;
  c_call_qps        the C entry point alone on arrays prepared once (flattening, slots, per-clause idf taken out);
  one_index_c_call_qps  the C entry point on the same queries with every clause on f1: the field-aware kernel
                    over one copy of the data;
  single_qps        search_topk of the same clauses on f1 (Bool), and single_c_call_qps its C entry point alone;
  ratio_c_call      c_call_qps / single_c_call_qps, the figure to watch: both move the same bytes;
  numpy_qps         the composition of dense per-field .score vectors on the host, over --numpy-queries queries;
  n_redone          queries of the timed batch re-run exactly (candidate overflow).
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
from _bool_occur_compose import compose_occur  # noqa: E402


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
    ap.add_argument("--phrase-queries", type=int, default=64)
    ap.add_argument("--numpy-queries", type=int, default=3)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--verify", type=int, default=6)
    args = ap.parse_args()

    import pandas as pd
    from searcharray_b200 import Bool, Boost, Field, Or, SearchArray, bm25_similarity, synth
    from searcharray_b200.postings import _PreparedBool
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

    nq, npq = len(names), min(args.phrase_queries, len(names))

    def build(F, label):
        """The workload `label`'s queries, with F(field, clause) making each clause."""
        n = npq if label == "phrase_f2" else nq
        make = {
            "must_a_b_c": lambda i: Bool(must=[F("f1", t(i, 0))], should=[F("f2", t(i, 1)), F("f2", t(i, 2))]),
            "most_fields": lambda i: Or([Boost(F("f1", t(i, 0)), 2), F("f2", t(i, 0))]),
            "a_b_not_c": lambda i: Bool(should=[F("f1", t(i, 0)), F("f1", t(i, 1))], must_not=[F("f2", t(i, 2))]),
            "must_rare_common": lambda i: Bool(must=[F("f1", rare_i(i))], should=[F("f2", common_i(i))]),
            "phrase_f2": lambda i: Bool(should=[F("f1", t(i, 0)), F("f1", t(i, 1))],
                                        must_not=[F("f2", [t(i, 2), t(i, 3)])]),
        }[label]
        return [make(i) for i in range(n)]

    sim = bm25_similarity()
    score = field_scorer({f: (lambda c, f=f: frame[f].array.score(c)) for f in ("f1", "f2")})
    out = {"card": info, "docs": host.n_docs, "k": args.k, "reps": args.reps, "warmup": args.warmup,
           "rare_df_mean": float(np.mean([dfs[x] for x in rare])), "common_df_mean": float(np.mean([dfs[x] for x in common])),
           "workloads": {}}
    for label in ("must_a_b_c", "most_fields", "a_b_not_c", "must_rare_common", "phrase_f2"):
        fq = build(Field, label)
        sq = build(lambda f, c: c, label)
        # correctness: a sample against the composition, the whole batch against the single-field Bool
        sample = fq[::max(1, len(fq) // args.verify)][:args.verify]
        d, s, _ = _fields_topk(frame, sample, args.k, sim, 0)
        for i, q in enumerate(sample):
            wd, ws = topk(compose_occur(score, q), args.k)
            if not (np.array_equal(d[i], wd) and np.array_equal(s[i].view(np.uint32), ws.view(np.uint32))):
                raise SystemExit(f"{label}: fields_topk differs from the composition for {q!r}")
        fd, fs, _ = _fields_topk(frame, fq, args.k, sim, 0)
        sd, ss, _ = f1._search_topk_bool(sq, args.k, sim, 0)
        if not (np.array_equal(fd, sd) and np.array_equal(fs.view(np.uint32), ss.view(np.uint32))):
            raise SystemExit(f"{label}: fields_topk on two copies differs from search_topk on one")

        redone = []

        def run_fields():
            redone.append(_fields_topk(frame, fq, args.k, sim, 0)[2])
        t_fields = median_time(run_fields, args.warmup, args.reps)
        t_single = median_time(lambda: f1._search_topk_bool(sq, args.k, sim, 0), args.warmup, args.reps)

        # the C calls alone on prepared arrays: the two-column queries, the same with every clause on f1 (the
        # field-aware kernel on one index's data), and the single-field Bool
        def fields_c_time(queries):
            batch, slot_of, arrays, sims = _fields_plan(frame, queries, sim)
            call = _PreparedBool(arrays, sims, _clause_slots(batch, slot_of), queries, batch,
                             multi=_multi_for(arrays))
            return median_time(lambda: call.run(args.k, 0), args.warmup, args.reps)
        t_c = fields_c_time(fq)
        t_c1 = fields_c_time(build(lambda f, c: Field("f1", c), label))
        single_call = f1._prepare_bool(sq, sim)
        t_single_c = median_time(lambda: single_call.run(args.k, 0), args.warmup, args.reps)

        # the host composition of dense per-field .score vectors
        nn = min(args.numpy_queries, len(fq))
        t0 = time.perf_counter()
        for q in fq[:nn]:
            topk(compose_occur(score, q), args.k)
        t_numpy = (time.perf_counter() - t0) / nn

        n = len(fq)
        rec = {"queries": n, "verified_queries": len(sample), "qps": n / t_fields, "c_call_qps": n / t_c,
               "one_index_c_call_qps": n / t_c1, "single_qps": n / t_single, "single_c_call_qps": n / t_single_c, "ratio_c_call": t_single_c / t_c,
               "ratio_qps": t_single / t_fields, "numpy_qps": 1.0 / t_numpy, "numpy_queries": nn,
               "n_redone": redone[-args.reps:]}
        out["workloads"][label] = rec
        print(f"[fields_topk_bench] {label}: {json.dumps(rec)}", file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
