"""Fixture for nested boolean queries (an Or / And / Bool used as a clause of another) in batched boolean queries,
composed through the REAL reference's `.score` on the TMDB title and overview fields, in numpy float32:

    score(leaf)  = frame[f].array.score(c, similarity=bm25(k1, b), slop=slop)       f: the leaf's field
    a DisMax     as make_golden_dismax.py composes it
    a nested N   r_N = the ranked vector of N composed as a query of its own (0 where N does not rank), matching where
                 r_N > 0, weighted by its Boost like a leaf
    then the Bool composition of make_golden_bool_fields.py over the clauses' (score, match)

    python tests/golden/make_golden_nested.py      (build container only)

Writes tests/golden/nested.json: per record its clauses (a leaf is {"f": field or null, "c": clause, "w": weight}, a
DisMax {"dismax": [leaves], "tie": tie}, a nested query {"node": {"kind", "must", "should", "filter", "must_not",
"mm_spec"}, "w": weight}), its kind ("or" or "bool"), the Solr mm spec and the mm the reference resolves it to, slop,
per-field (k1, b), "field" (the one column of a search_topk record, else null), the top 10 ids, their float32 score
bits and the number of ranked docs.
"""
import json
import os

import numpy as np

from make_golden import import_reference, HERE
from make_golden_tmdb import load_corpus

T, O = "title_tokens", "overview_tokens"


def L(field, clause, w=1.0):
    return {"f": field, "c": clause, "w": float(w)}


def S(clause, w=1.0):
    """A leaf of a single-field (search_topk) record."""
    return {"f": None, "c": clause, "w": float(w)}


def D(members, tie=0.0):
    return {"dismax": list(members), "tie": float(tie)}


def node(must=(), should=(), filter=(), must_not=(), mm=None, kind="bool"):
    if mm is None:
        mm = 0 if (must or filter) else 1
    assert kind == "bool" or not (must or filter or must_not)
    return {"kind": kind, "must": list(must), "should": list(should), "filter": list(filter),
            "must_not": list(must_not), "mm_spec": str(mm)}


def N(q, w=1.0):
    """A nested query as a clause."""
    return {"node": q, "w": float(w)}


def OR(should, mm=1):
    return node(should=should, mm=mm, kind="or")


def AND(clauses):
    return node(should=clauses, mm=len(clauses), kind="or")


def Q(q, slop=0, sim=None, field=None):
    """A record: the top-level node q and the call's arguments."""
    return dict(q, slop=slop, sim=sim or {}, field=field)


def qf_pf(terms, mm="75%", pf_w=3.0):
    """edismax's qf + pf shape: Bool(must=[Or([DisMax(title^2 | overview) per term], mm)], should=[title phrase^pf_w])."""
    qf = OR([D([L(T, t, 2), L(O, t)], 0.1) for t in terms], mm=mm)
    return Q(node(must=[N(qf)], should=[L(T, list(terms), pf_w)]))


QUERIES = [
    # (star AND wars) OR (star AND trek), on the fields and on one column
    Q(OR([N(AND([L(T, "Star"), L(T, "Wars")])), N(AND([L(T, "Star"), L(T, "Trek")]))])),
    Q(OR([N(AND([S("Star"), S("Wars")])), N(AND([S("Star"), S("Trek")]))]), field=T),
    # a required sub-query with its own mm: +title:alien +(overview:the overview:crew overview:a)~2
    Q(node(must=[L(T, "Alien"), N(OR([L(O, "the"), L(O, "crew"), L(O, "a")], mm=2))])),
    # excluding a conjunction: foo -(spam AND eggs)
    Q(node(should=[L(O, "war")], must_not=[N(AND([L(O, "world"), L(O, "ii")]))])),
    Q(node(should=[S("love")], must_not=[N(AND([S("new"), S("york")]))]), field=O),
    # a nested query as a filter, and as a should next to leaves, with mm outside
    Q(node(filter=[N(OR([L(T, "Dark"), L(T, "Night")]))], should=[L(O, "city"), L(O, "hero")])),
    Q(node(should=[N(AND([L(O, "young"), L(O, "man")])), L(O, "love"), L(T, "Story")], mm=2)),
    # Boost of a nested query, weight 0 included (matches without scoring)
    Q(OR([N(AND([L(T, "Star"), L(O, "war")]), 2.5), L(O, "space")])),
    Q(node(must=[N(OR([L(T, "Love"), L(O, "love")]), 0)], should=[L(O, "young")])),
    Q(node(should=[N(OR([L(O, "murder"), L(O, "police")]), 0), L(O, "detective", 0.5)], mm=1)),
    # Solr mm specs inside and outside
    Q(OR([N(OR([L(O, "war"), L(O, "battle"), L(O, "army"), L(O, "soldier")], mm="50%")), L(T, "War"),
          N(OR([L(O, "love"), L(O, "romance")], mm="-1"))], mm="-1")),
    Q(OR([N(OR([S("war"), S("battle"), S("army")], mm="2")), N(OR([S("love"), S("story")], mm="100%")), S("world")],
         mm="-1"), field=O),
    # depth 3
    Q(OR([N(node(must=[N(AND([L(T, "Star"), N(OR([L(T, "Wars"), L(T, "Trek")]))]))], should=[L(O, "space")])),
          L(O, "galaxy")])),
    Q(node(must=[N(OR([N(AND([S("new"), N(OR([S("york"), S("city")]))])), S("manhattan")]))], should=[S("crime")]),
      field=O),
    # a DisMax inside a nested Or
    Q(node(must=[N(OR([D([L(T, "Dark", 2), L(O, "dark")], 0.3), D([L(T, "Knight", 2), L(O, "knight")], 0.3)]))],
           should=[L(O, "batman")])),
    Q(OR([N(OR([D([S("film"), S("movie")], 0.1), S("director")], mm=2)), S("actor")]), field=O),
    # phrase leaves inside nested queries at slop 0 and 2
    Q(OR([N(AND([L(O, ["New", "York"]), L(O, "city")])), N(OR([L(T, ["Star", "Wars"], 2), L(O, "empire")]))])),
    Q(OR([N(AND([L(O, ["New", "York"]), L(O, "city")])), N(OR([L(T, ["Star", "Wars"], 2), L(O, "empire")]))]),
      slop=2),
    Q(node(should=[S("police")], must_not=[N(OR([S(["serial", "killer"]), S("murder")], mm=2))]), field=O, slop=2),
    # per-field k1 / b
    Q(OR([N(AND([L(T, "Star"), L(O, "star")])), L(O, "war")]), sim={T: [0.9, 0.4], O: [1.6, 0.9]}),
    # unknown tokens: a nested query that ranks nothing anywhere
    Q(node(should=[L(O, "war")], must=[N(OR([L(T, "zzzzunknown"), L(O, "qqqqunknown")]))])),
    Q(OR([N(AND([L(T, "zzzzunknown"), L(O, "war")])), L(O, "peace")])),
    # the same sub-query twice
    Q(node(should=[N(AND([L(O, "young"), L(O, "woman")])), N(AND([L(O, "young"), L(O, "woman")]), 2)],
           must_not=[N(AND([L(O, "young"), L(O, "woman"), L(O, "man")]))])),
    # edismax's qf + pf shape
    qf_pf(["Star", "Wars"]),
    qf_pf(["The", "Dark", "Knight"]),
    qf_pf(["Love", "Story", "New", "York"], mm="2<-25%", pf_w=5.0),
]


def composed(arrs, q, rec, parse_mm, bm25, cache):
    """The ranked dense float32 vector of node q of record rec (0 where a doc does not rank), and q's resolved mm."""
    def sc(leaf):
        f = leaf["f"] or rec["field"]
        key = json.dumps([f, leaf["c"]])
        if key not in cache:
            k1, b = rec["sim"].get(f, [1.2, 0.75])
            v = arrs[f].score(leaf["c"], similarity=bm25(k1=k1, b=b), slop=rec["slop"])
            assert v.dtype == np.float32
            cache[key] = v
        return cache[key]

    def value(c):
        """(the clause's weighted score, its match) for a leaf, a DisMax or a nested query."""
        if "node" in c:
            r, _ = composed(arrs, c["node"], rec, parse_mm, bm25, cache)
            return np.float32(c["w"]) * r, r > 0
        if "dismax" not in c:
            return np.float32(c["w"]) * sc(c), sc(c) > 0
        vs = [np.float32(m["w"]) * sc(m) for m in c["dismax"]]
        m = np.maximum.reduce(vs)
        t = vs[0]
        for v in vs[1:]:
            t = t + v
        return m + (t - m) * np.float32(c["tie"]), np.any([sc(x) > 0 for x in c["dismax"]], axis=0)

    mm = parse_mm(len(q["should"]), q["mm_spec"])
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


def main():
    import_reference()
    from searcharray.postings import SearchArray
    from searcharray.similarity import bm25_similarity
    from searcharray.solr import parse_min_should_match
    titles, overviews = load_corpus()
    arrs = {T: SearchArray.index(titles), O: SearchArray.index(overviews)}
    out = {"queries": []}
    for q in QUERIES:
        v, mm = composed(arrs, q, q, parse_min_should_match, bm25_similarity, {})
        ids, bits = top10(v)
        out["queries"].append(dict(q, mm=int(mm), top_ids=ids, top_bits=bits, n_ranked=int(np.count_nonzero(v > 0))))
    path = os.path.join(HERE, "nested.json")
    with open(path, "w") as f:
        json.dump(out, f)
    print(len(out["queries"]), [r["n_ranked"] for r in out["queries"]], os.path.getsize(path))


if __name__ == "__main__":
    main()
