"""Fixture for disjunction-max clauses (query.DisMax) in batched boolean queries, composed through the REAL reference's
`.score` on the TMDB title and overview fields, in numpy float32:

    score(leaf)  = frame[f].array.score(c, similarity=bm25(k1, b), slop=slop)       f: the leaf's field
    v_j = np.float32(w_j) * score(member j)
    m   = np.maximum.reduce(vs);  t = v_0 + v_1 + ... (left fold);  d = m + (t - m) * np.float32(tie)
    hit = any_j score(member j) > 0
    then the Bool composition of make_golden_bool_fields.py, a DisMax being one clause of weight 1 whose score is d
    and whose match is hit; a top-level DisMax is Bool(should=[it])

    python tests/golden/make_golden_dismax.py      (build container only)

Every term-centric query without pf (an Or of one DisMax per term over title^w | overview) is also checked against
the reference's own solr.edismax(frame, q, qf, mm, tie): the float32 composition must agree within 1e-5 relative at
every doc, and the docs scoring > 0 must be the same set.

Writes tests/golden/dismax.json: per record its clauses (a leaf is {"f": field or null, "c": clause, "w": weight}, a
DisMax {"dismax": [leaves], "tie": tie}), the Solr mm spec and the mm the reference resolves it to, slop, per-field
(k1, b), "field" (the one column of a search_topk record, else null), the top 10 ids, their float32 score bits and
the number of ranked docs.
"""
import json
import os

import numpy as np

from make_golden import import_reference, HERE
from make_golden_tmdb import load_corpus

T, O = "title_tokens", "overview_tokens"


def L(field, clause, w=1.0):
    return {"f": field, "c": clause, "w": float(w)}


def D(members, tie=0.0):
    return {"dismax": list(members), "tie": float(tie)}


def Q(must=(), should=(), filter=(), must_not=(), mm=None, kind="bool", slop=0, sim=None, field=None, edismax=None):
    """A record.  kind "or": Or(should, mm); "dismax": the one DisMax in should as a query of its own; "bool": Bool
    (mm None: 0 with must / filter clauses, else 1).  field: the column of a search_topk record (leaves without a
    field).  edismax: (q, qf, mm, tie) of the reference edismax call this record must agree with."""
    if mm is None:
        mm = 0 if (must or filter) else 1
    assert kind == "bool" or not (must or filter or must_not)
    assert kind != "dismax" or (len(should) == 1 and "dismax" in should[0])
    return {"kind": kind, "must": list(must), "should": list(should), "filter": list(filter),
            "must_not": list(must_not), "mm_spec": str(mm), "slop": slop, "sim": sim or {}, "field": field,
            "edismax": edismax}


def best_fields(terms, tie, wt=2.0, mm="1", sim=None):
    """edismax's term-centric qf over title^wt | overview: Or(DisMax per term, mm), with its edismax cross-check."""
    should = [D([L(T, t, wt), L(O, t)], tie) for t in terms]
    qf = [f"{T}^{wt:g}", O]
    return Q(should=should, mm=mm, kind="or", sim=sim, edismax=(" ".join(terms), qf, mm, tie))


def S(clause, w=1.0):
    """A leaf of a single-field (search_topk) record."""
    return {"f": None, "c": clause, "w": float(w)}


QUERIES = [
    # per-term best_fields over title^2 | overview inside Or, Solr mm specs, tie 0 / 0.1 / 0.3 / 1.0
    best_fields(["Star", "Wars"], 0.0),
    best_fields(["Star", "Wars"], 0.1, mm="2"),
    best_fields(["Star", "Wars"], 0.3),
    best_fields(["Star", "Wars"], 1.0),
    best_fields(["The", "Dark", "Knight"], 0.1, mm="2"),
    best_fields(["The", "Dark", "Knight"], 0.3, mm="75%"),
    best_fields(["Love", "Story", "New", "York"], 0.1, mm="2<-25%"),
    best_fields(["Love", "Story", "New", "York"], 0.0, mm="-1"),
    best_fields(["Man", "Woman"], 1.0, wt=1.0),
    best_fields(["Alien", "Space", "War"], 0.3, wt=3.0, mm="2"),
    # per-field k1 / b (the cross-check passes the same similarities)
    best_fields(["Star", "War"], 0.1, sim={T: [0.9, 0.4], O: [1.6, 0.9]}),
    best_fields(["Dark", "City"], 0.3, mm="2", sim={O: [2.0, 0.3]}),
    # a DisMax in each role
    Q(must=[D([L(T, "Star", 2), L(O, "star")], 0.1)], should=[L(O, "war"), L(O, "space")]),
    Q(should=[D([L(T, "Love"), L(O, "love")], 0.3), D([L(T, "War"), L(O, "war")], 0.3)], mm=2),
    Q(filter=[D([L(T, "Star"), L(O, "star")])], should=[L(O, "war"), L(T, "Trek")]),
    Q(should=[L(O, "murder"), L(O, "detective")], must_not=[D([L(T, "The"), L(O, "police")])]),
    Q(must=[D([L(T, "Dark"), L(O, "dark")], 0.5)], should=[D([L(T, "Knight"), L(O, "knight")], 0.2)],
      must_not=[D([L(O, "comedy"), L(T, "Comedy")])], filter=[D([L(O, "the"), L(T, "The")])]),
    # phrase members at slop 0 and 2
    Q(should=[D([L(T, ["Star", "Wars"], 3), L(O, ["Death", "Star"])], 0.1), L(O, "empire")]),
    Q(must=[D([L(O, ["New", "York"]), L(T, ["New", "York"], 2)], 0.3)], should=[L(O, "city")]),
    Q(should=[D([L(T, ["Star", "Wars"], 3), L(O, ["young", "man"])], 0.1), L(O, "war")], slop=2),
    Q(must=[D([L(O, ["New", "York"]), L(T, ["New", "York"], 2)], 0.3)], should=[L(O, "city")], slop=2),
    # a zero-weight member still matches
    Q(must=[D([L(T, "Dark", 0), L(O, "dark", 0)], 0.5)], should=[L(O, "night")]),
    Q(should=[D([L(T, "Love", 0), L(O, "love")], 0.2), L(O, "young")], mm=2),
    # single-member DisMax
    Q(must=[D([L(T, "Star", 2)], 0.7)], should=[D([L(O, "war")], 1.0)]),
    Q(should=[L(O, "police")], must_not=[D([L(T, "The")], 0.4)]),
    # DisMax mixed with plain leaves and boosts
    Q(must=[L(T, "Love", 1.5)], should=[D([L(T, "Story"), L(O, "story", 0.5)], 0.1), L(O, "young", 2)]),
    Q(should=[L(T, "Star"), D([L(T, "Trek"), L(O, "trek"), L(O, "enterprise", 0.5)], 0.3), L(O, "space")], mm=2),
    # unknown tokens
    Q(should=[D([L(T, "zzzzunknown"), L(O, "star")], 0.3), L(O, "war")]),
    Q(must=[D([L(T, "zzzzunknown"), L(O, "qqqqunknown")])], should=[L(O, "war")]),
    Q(should=[D([L(T, ["Star", "zzzzunknown"]), L(O, "war", 2)], 0.1)], must_not=[D([L(O, "zzzzunknown")])]),
    # top-level DisMax (Elasticsearch's dis_max query)
    Q(should=[D([L(T, "Alien", 2), L(O, "alien")], 0.3)], kind="dismax"),
    Q(should=[D([L(T, "Love"), L(O, "love"), L(O, ["fall", "in", "love"], 3)], 0.1)], kind="dismax"),
    Q(should=[D([L(T, "Star", 2), L(O, "star")], 0.0)], kind="dismax", sim={T: [1.5, 0.5]}),
    # single-field synonyms for search_topk (overview)
    Q(should=[D([S("film"), S("movie")], 0.1)], kind="dismax", field=O),
    Q(should=[D([S("murder"), S("killing", 0.8), S("homicide", 0.8)], 0.2), S("detective")], mm=1, field=O),
    Q(must=[D([S("car"), S("truck"), S("vehicle")], 0.0)], should=[S("chase")], field=O),
    Q(should=[S("police")], must_not=[D([S("comedy"), S("funny")])], field=O),
    Q(should=[D([S(["New", "York"]), S("Manhattan")], 0.3), S("city")], field=O, slop=2),
    Q(should=[D([S("love"), S("romance")], 0.5), D([S("war"), S("battle")], 0.5)], mm="100%", kind="or", field=O),
]


def members(c):
    return c["dismax"] if "dismax" in c else [c]


def composed(arrs, q, parse_mm, bm25):
    """The record's ranked dense float32 vector (0 where a doc does not rank), and its resolved mm."""
    cache = {}

    def sc(leaf):
        f = leaf["f"] or q["field"]
        key = json.dumps([f, leaf["c"]])
        if key not in cache:
            k1, b = q["sim"].get(f, [1.2, 0.75])
            v = arrs[f].score(leaf["c"], similarity=bm25(k1=k1, b=b), slop=q["slop"])
            assert v.dtype == np.float32
            cache[key] = v
        return cache[key]

    def value(c):
        """(the clause's score, its match) for a leaf or a DisMax."""
        if "dismax" not in c:
            return np.float32(c["w"]) * sc(c), sc(c) > 0
        vs = [np.float32(m["w"]) * sc(m) for m in c["dismax"]]
        m = np.maximum.reduce(vs)
        t = vs[0]
        for v in vs[1:]:
            t = t + v
        d = m + (t - m) * np.float32(c["tie"])
        hit = np.any([sc(x) > 0 for x in c["dismax"]], axis=0)
        assert d.dtype == np.float32
        return d, hit

    mm = parse_mm(len(q["should"]), q["mm_spec"]) if q["kind"] != "dismax" else 1
    scoring = q["must"] + q["should"]
    s = value(scoring[0])[0]
    for c in scoring[1:]:
        s = s + value(c)[0]
    n = len(s)
    hits = np.sum([value(c)[1] for c in q["should"]], axis=0) if q["should"] else np.zeros(n, dtype=np.int64)
    ok = hits >= mm
    for c in q["must"] + q["filter"]:
        ok &= value(c)[1]
    for c in q["must_not"]:
        ok &= ~value(c)[1]
    assert s.dtype == np.float32
    return np.where(ok & (s > 0), s, np.float32(0)).astype(np.float32), mm


def top10(v):
    order = np.lexsort((np.arange(len(v)), -v.astype(np.float64)))[:10]
    order = order[v[order] > 0]
    return [int(i) for i in order], [int(b) for b in v[order].view(np.uint32)]


def check_edismax(arrs, q, v, bm25, edismax):
    """The float32 composition against the reference's own edismax (term-centric qf, no pf)."""
    import pandas as pd
    text, qf, mm, tie = q["edismax"]
    frame = pd.DataFrame({T: arrs[T], O: arrs[O]})
    sims = {f: bm25(k1=q["sim"].get(f, [1.2, 0.75])[0], b=q["sim"].get(f, [1.2, 0.75])[1]) for f in (T, O)}
    ref, explain = edismax(frame, text, qf=qf, mm=mm, tie=tie, similarity=sims)
    assert "~" in explain, explain
    ref = np.asarray(ref, dtype=np.float64)
    assert np.array_equal(ref > 0, v > 0), (text, int(np.count_nonzero(ref > 0)), int(np.count_nonzero(v > 0)))
    np.testing.assert_allclose(v.astype(np.float64), ref, rtol=1e-5, atol=0, err_msg=text)


def main():
    import_reference()
    from searcharray.postings import SearchArray
    from searcharray.similarity import bm25_similarity
    from searcharray.solr import edismax, parse_min_should_match
    titles, overviews = load_corpus()
    arrs = {T: SearchArray.index(titles), O: SearchArray.index(overviews)}
    out = {"queries": []}
    n_checked = 0
    for q in QUERIES:
        v, mm = composed(arrs, q, parse_min_should_match, bm25_similarity)
        if q["edismax"] is not None:
            check_edismax(arrs, q, v, bm25_similarity, edismax)
            n_checked += 1
        ids, bits = top10(v)
        rec = dict(q, mm=int(mm), top_ids=ids, top_bits=bits, n_ranked=int(np.count_nonzero(v > 0)))
        rec["edismax"] = None if q["edismax"] is None else list(q["edismax"])
        out["queries"].append(rec)
    path = os.path.join(HERE, "dismax.json")
    with open(path, "w") as f:
        json.dump(out, f)
    print(len(out["queries"]), n_checked, [r["n_ranked"] for r in out["queries"]], os.path.getsize(path))


if __name__ == "__main__":
    main()
