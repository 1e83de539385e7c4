"""Fixture for boolean queries over several DataFrame fields (solr.fields_topk), composed through the REAL reference's
`.score` on each clause's own field, the way its users compose multi-field queries (a sum of per-column vectors):

    scoring = must + should                                       fold order
    score(f:c) = frame[f].array.score(c, similarity=sim[f], slop=slop)
    s   = np.float32(w0) * score(c0); s = s + np.float32(w1) * score(c1); ...
    ok  = (np.sum([score(c) > 0 for c in should], axis=0) >= mm)
          & all(score(c) > 0 for c in must + filter) & ~any(score(c) > 0 for c in must_not)
    rank iff ok and s > 0; top 10 by (score desc, id asc)

    python tests/golden/make_golden_bool_fields.py      (build container only)

Writes tests/golden/bool_fields.json: per query its clauses ({"f": field, "c": clause}), weights, the Solr mm spec and
the mm the reference's parse_min_should_match resolves it to, slop, per-field (k1, b), the top 10 ids, their float32
score bits and the number of ranked docs, on the TMDB title and overview fields.
"""
import json
import os

import numpy as np

from make_golden import import_reference, HERE
from make_golden_tmdb import load_corpus

T, O = "title_tokens", "overview_tokens"


def F(field, clause, w=None):
    c = {"f": field, "c": clause}
    return c if w is None else (c, w)


def Q(must=(), should=(), filter=(), must_not=(), mm=None, kind="bool", slop=0, sim=None):
    """A query record.  Clauses of must / should are F(...) or F(..., weight); mm None is Bool's default (0 with must
    or filter clauses, else 1), otherwise a Solr spec over the should clauses; kind "or" is Or(should, mm).  sim:
    {field: [k1, b]} (fields left out take bm25_similarity())."""
    def split(cs):
        return [c[0] if isinstance(c, tuple) else c for c in cs], [float(c[1]) if isinstance(c, tuple) else 1.0 for c in cs]
    must, must_w = split(must)
    should, should_w = split(should)
    if mm is None:
        mm = 0 if (must or filter) else 1
    assert kind == "bool" or not (must or filter or must_not)
    return {"kind": kind, "must": must, "must_w": must_w, "should": should, "should_w": should_w,
            "filter": list(filter), "must_not": list(must_not), "mm_spec": str(mm), "slop": slop, "sim": sim or {}}


QUERIES = [
    # cross-field must / should / filter / must_not
    Q(must=[F(T, "Star")], should=[F(O, "war"), F(O, "space")]),
    Q(must=[F(T, "Star")], should=[F(O, "war")], must_not=[F(O, "trek")]),
    Q(should=[F(T, "Wars"), F(O, "war")], mm=2),
    Q(filter=[F(O, "the")], should=[F(T, "Star"), F(T, "Trek")]),
    Q(filter=[F(T, "The")], should=[F(O, "love"), F(O, "family")], mm=1),
    Q(should=[F(O, "murder"), F(O, "detective"), F(T, "Murder")], must_not=[F(T, "The")]),
    Q(must=[F(O, "young")], should=[F(T, "Love")], must_not=[F(T, "The"), F(O, "war")]),
    Q(must=[F(O, "love"), F(T, "Love")], should=[F(O, "young")]),
    # the same term on both fields with boosts (most_fields)
    Q(should=[F(T, "Alien", 2), F(O, "alien")], kind="or"),
    Q(should=[F(T, "Star", 2), F(O, "star")], kind="or"),
    Q(should=[F(T, "War", 3), F(O, "war", 0.5)], kind="or"),
    Q(should=[F(T, "Love"), F(O, "love")], mm=2, kind="or"),
    Q(must=[F(T, "Star")], should=[F(O, "galaxy")], mm=0),
    Q(should=[F(T, "Lord", 2), F(O, "ring"), F(O, "rings")]),
    Q(must=[F(T, "Dark", 0)], should=[F(O, "dark")]),
    # phrases on each field at slop 0 and 2
    Q(must=[F(O, ["New", "York"])], should=[F(T, "New"), F(T, "York")]),
    Q(should=[F(T, ["Star", "Wars"], 3), F(O, ["Death", "Star"])], kind="or"),
    Q(should=[F(O, "police"), F(O, "city")], must_not=[F(T, ["The", "Dark"])]),
    Q(filter=[F(O, ["in", "the"])], should=[F(T, "City"), F(O, "city", 2)]),
    Q(must=[F(O, ["New", "York"])], should=[F(T, "New"), F(T, "York")], slop=2),
    Q(should=[F(T, ["Star", "Wars"], 3), F(O, ["young", "man"])], kind="or", slop=2),
    Q(should=[F(O, "police"), F(O, "city")], must_not=[F(T, ["The", "Dark"])], slop=2),
    # Solr mm specs
    Q(should=[F(T, "The"), F(T, "of"), F(O, "the"), F(O, "of")], mm="75%"),
    Q(should=[F(T, "Star"), F(O, "star"), F(O, "war"), F(O, "galaxy"), F(T, "Wars")], mm="2<-60%", kind="or"),
    Q(must=[F(O, "love")], should=[F(T, "Love"), F(O, "young"), F(O, "family")], mm="-1"),
    # per-field k1 / b
    Q(should=[F(T, "Star"), F(O, "star"), F(O, "war")], sim={T: [0.9, 0.4], O: [1.6, 0.9]}),
    Q(must=[F(O, "murder")], should=[F(T, "Murder"), F(O, "detective", 2)], sim={O: [2.0, 0.3]}),
    Q(should=[F(T, "Love"), F(O, "love")], mm=2, sim={T: [2.0, 0.3], O: [2.0, 0.3]}),
    # an unknown token in one field
    Q(must=[F(T, "zzzzunknown")], should=[F(O, "star")]),
    Q(should=[F(T, "zzzzunknown"), F(O, "war")], must_not=[F(O, "qqqqunknown")]),
    Q(should=[F(T, "Star"), F(O, ["zzzzunknown", "war"], 2)], must_not=[F(T, ["Star", "zzzzunknown"])]),
]


def composed(arrs, q, parse_mm, bm25):
    cache = {}

    def sc(c):
        key = json.dumps(c)
        if key not in cache:
            k1, b = q["sim"].get(c["f"], [1.2, 0.75])
            v = arrs[c["f"]].score(c["c"], similarity=bm25(k1=k1, b=b), slop=q["slop"])
            assert v.dtype == np.float32
            cache[key] = v
        return cache[key]
    mm = parse_mm(len(q["should"]), q["mm_spec"])
    scoring, weights = q["must"] + q["should"], q["must_w"] + q["should_w"]
    s = np.float32(weights[0]) * sc(scoring[0])
    for c, w in zip(scoring[1:], weights[1:]):
        s = s + np.float32(w) * sc(c)
    n = len(s)
    hits = np.sum([sc(c) > 0 for c in q["should"]], axis=0) if q["should"] else np.zeros(n, dtype=np.int64)
    ok = hits >= mm
    for c in q["must"] + q["filter"]:
        ok &= sc(c) > 0
    for c in q["must_not"]:
        ok &= ~(sc(c) > 0)
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
        v, mm = composed(arrs, q, parse_min_should_match, bm25_similarity)
        ids, bits = top10(v)
        out["queries"].append(dict(q, mm=int(mm), top_ids=ids, top_bits=bits, n_ranked=int(np.count_nonzero(v > 0))))
    path = os.path.join(HERE, "bool_fields.json")
    with open(path, "w") as f:
        json.dump(out, f)
    print(len(out["queries"]), [r["n_ranked"] for r in out["queries"]], os.path.getsize(path))


if __name__ == "__main__":
    main()
