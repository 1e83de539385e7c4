"""Fixture for boolean queries with required / optional / filter / prohibited clauses and per-clause boosts,
composed through the REAL reference's `.score` the way its tests compose multi-clause queries
(test/test_search.py:126-226), extended in the obvious numpy way:

    scoring = must + should                                       fold order
    s   = np.float32(w0) * arr.score(c0); s = s + np.float32(w1) * arr.score(c1); ...
    ok  = (np.sum([arr.score(c) > 0 for c in should], axis=0) >= mm)
          & all(arr.score(c) > 0 for c in must + filter) & ~any(arr.score(c) > 0 for c in must_not)
    rank iff ok and s > 0; top 10 by (score desc, id asc)

    python tests/golden/make_golden_bool_occur.py      (build container only)

Writes tests/golden/bool_occur.json: per query its clauses, weights and resolved mm, the top 10 ids, their float32
score bits and the number of ranked docs, on the TMDB title and overview fields and on the reference's 4-doc x 25
scenario corpus (test/test_search.py's and/or scenarios; the docs are data, no reference source is copied).
"""
import json
import os

import numpy as np

from make_golden import import_reference, HERE
from make_golden_scenarios import period_compress
from make_golden_tmdb import load_corpus

SCENARIO_DOCS = ["foo bar bar baz", "data2", "data3 bar", "bunny funny wunny"] * 25


def Q(corpus, must=(), should=(), filter=(), must_not=(), mm=None, kind="bool"):
    """A query record.  Clauses of must / should are a clause or (clause, weight); mm None is Bool's default (0 with
    must or filter clauses, else 1); kind "or" is Or(should, mm) with boosts (should only)."""
    def split(cs):
        return [c[0] if isinstance(c, tuple) else c for c in cs], [float(c[1]) if isinstance(c, tuple) else 1.0 for c in cs]
    must, must_w = split(must)
    should, should_w = split(should)
    if mm is None:
        mm = 0 if (must or filter) else 1
    assert kind == "bool" or not (must or filter or must_not)
    return {"corpus": corpus, "kind": kind, "must": must, "must_w": must_w, "should": should, "should_w": should_w,
            "filter": list(filter), "must_not": list(must_not), "mm": mm}


T, O, S = "title_tokens", "overview_tokens", "scenario"
QUERIES = [
    # must + should, mm 0 / 1 / 2
    Q(T, must=["Star"], should=["Wars", "Trek"], mm=0),
    Q(T, must=["Star"], should=["Wars", "Trek"], mm=1),
    Q(T, must=["the"], should=["of", "a", "Star"], mm=2),
    Q(O, must=["war"], should=["love", "family"], mm=2),
    Q(O, must=["galactic"], should=["empire", "rebel"], mm=1),
    # must_not on a frequent term and on a phrase
    Q(T, should=["Star", "Wars"], must_not=["the"]),
    Q(T, should=["Star", "Trek"], must_not=[["Star", "Wars"]]),
    Q(O, must=[["New", "York"]], should=["police", "city"], must_not=["murder"]),
    Q(O, should=["murder", "detective", "mystery", "killer"], must_not=["the"], mm=2),
    # filter-only restriction plus should
    Q(T, filter=["the"], should=["Lord", "Rings"]),
    Q(T, filter=["of"], should=["the", "Lord"], mm=1),
    Q(O, filter=[["in", "the"]], should=[("city", 2), "police"]),
    # boosts 0, 0.5, 2, 3 on terms and phrases
    Q(T, should=[("Star", 2), "Wars", ("Trek", 0.5)], kind="or"),
    Q(T, should=[("the", 0), "Star"], mm=2, kind="or"),
    Q(T, should=[(["Star", "Wars"], 3), "Empire", "Strikes"], kind="or"),
    Q(T, should=[(["Star", "Wars"], 0.5), "Empire"], kind="or"),
    Q(T, must=[("Black", 0.5)], should=[(["Black", "Mirror:"], 2)]),
    Q(O, should=[("war", 0.5), ("love", 3), (["New", "York"], 2), "family"], kind="or"),
    Q(O, should=[(["New", "York"], 0), "young"], mm=2),
    Q(O, must=[("young", 2)], should=[("the", 0.5)], filter=["a"]),
    Q(T, must=[("the", 0)], should=["Star"]),
    # duplicate clauses and unknown tokens in every role
    Q(T, must=["Star", "Star"], should=["Wars", "Wars"], filter=["Star"], must_not=["Trek", "Trek"]),
    Q(T, must=["zzzzunknown"], should=["Star"]),
    Q(T, should=["zzzzunknown", "Star"], must_not=["qqqqunknown"], mm=1),
    Q(T, filter=["zzzzunknown"], should=["Star"]),
    Q(T, should=["Star", (["zzzzunknown", "Wars"], 2)], must_not=[["Star", "zzzzunknown"]]),
    Q(O, must=["the"], should=["zzzzunknown"]),
    Q(O, should=[("zzzzunknown", 3), "war", "war"], kind="or"),
    # the reference's scenario corpus
    Q(S, must=["foo"], should=["bar"], mm=0),
    Q(S, should=["bar"], must_not=["foo"]),
    Q(S, should=["bar", "baz"], must_not=[["foo", "bar"]]),
    Q(S, filter=["bar"], should=[("baz", 2), "data3"]),
    Q(S, should=[(["foo", "bar"], 3), ("data2", 0.5)], kind="or"),
    Q(S, must=[("bar", 0)], should=["foo"]),
    Q(S, must=["bar"], should=["zzzz", "foo", "foo"], filter=["bar"], must_not=["zzzz", "data2"], mm=1),
]


def composed(arr, q):
    cache = {}

    def sc(c):
        key = json.dumps(c)
        if key not in cache:
            v = arr.score(c)
            assert v.dtype == np.float32
            cache[key] = v
        return cache[key]
    scoring, weights = q["must"] + q["should"], q["must_w"] + q["should_w"]
    s = np.float32(weights[0]) * sc(scoring[0])
    for c, w in zip(scoring[1:], weights[1:]):
        s = s + np.float32(w) * sc(c)
    n = len(s)
    hits = np.sum([sc(c) > 0 for c in q["should"]], axis=0) if q["should"] else np.zeros(n, dtype=np.int64)
    ok = hits >= q["mm"]
    for c in q["must"] + q["filter"]:
        ok &= sc(c) > 0
    for c in q["must_not"]:
        ok &= ~(sc(c) > 0)
    assert s.dtype == np.float32
    return np.where(ok & (s > 0), s, np.float32(0)).astype(np.float32)


def top10(v):
    order = np.lexsort((np.arange(len(v)), -v.astype(np.float64)))[:10]
    order = order[v[order] > 0]
    return [int(i) for i in order], [int(b) for b in v[order].view(np.uint32)]


def main():
    import_reference()
    from searcharray.postings import SearchArray
    titles, overviews = load_corpus()
    arrs = {T: SearchArray.index(titles), O: SearchArray.index(overviews), S: SearchArray.index(SCENARIO_DOCS)}
    out = {"scenario_docs": period_compress(SCENARIO_DOCS), "queries": []}
    for q in QUERIES:
        v = composed(arrs[q["corpus"]], q)
        ids, bits = top10(v)
        out["queries"].append(dict(q, top_ids=ids, top_bits=bits, n_ranked=int(np.count_nonzero(v > 0))))
    path = os.path.join(HERE, "bool_occur.json")
    with open(path, "w") as f:
        json.dump(out, f)
    print(len(out["queries"]), [r["n_ranked"] for r in out["queries"]], os.path.getsize(path))


if __name__ == "__main__":
    main()
