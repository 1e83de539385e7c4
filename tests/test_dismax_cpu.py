"""CPU: disjunction-max clauses (query.DisMax) -- validation, flattening to groups and ties, every refusal (raised
before any device work, so on CPU-built arrays), and the oracle composition against the real reference's composed
results (tests/golden/dismax.json, make_golden_dismax.py)."""
import json
import os

import numpy as np
import pandas as pd
import pytest

from _bool_compose import oracle_score, topk
from _bool_fields_compose import field_scorer
from _dismax_compose import compose_dismax, query_of, record_groups
from _tmdb_index import load_field
from conftest import GOLDEN

T, O = "title_tokens", "overview_tokens"


@pytest.fixture(scope="module")
def fixture():
    with open(os.path.join(GOLDEN, "dismax.json")) as f:
        return json.load(f)


def frame_of(**cols):
    from searcharray_b200 import SearchArray
    return pd.DataFrame({name: SearchArray.index(docs) for name, docs in cols.items()})


def test_dismax_validation():
    from searcharray_b200 import And, Bool, Boost, DisMax, Field, Or
    d = DisMax(["a", ["b", "c"], Field("t", "x"), Boost(Field("o", "y"), 2), Boost("z", 0)], tie=0.1)
    assert d.clauses[:2] == ["a", ["b", "c"]] and d.clauses[2].field == "t" and d.clauses[3].field == "o"
    assert d.weights == [1.0, 1.0, 1.0, 2.0, 0.0] and d.tie == np.float32(0.1) and d.tie.dtype == np.float32
    assert d.boosted and not DisMax(["a", "b"]).boosted and DisMax(["a"]).tie == 0
    assert repr(DisMax(["a", Boost("b", 2)], tie=0.5)) == "DisMax(['a', Boost('b', 2.0)], tie=0.5)"
    for tie in (-0.1, 1.5, float("nan"), float("inf"), -float("inf")):
        with pytest.raises(ValueError):
            DisMax(["a"], tie=tie)
    for tie in (0, 1, 0.0, 1.0):
        DisMax(["a"], tie=tie)
    with pytest.raises(ValueError):
        DisMax([])
    # no nesting, no boosted DisMax, no DisMax in a Field
    for inner in (DisMax(["a"]), Or(["a"]), And(["a"]), Bool(should=["a"])):
        with pytest.raises(TypeError):
            DisMax(["a", inner])
    for inner in (Or(["a"]), Bool(should=["a"])):
        with pytest.raises(TypeError):
            DisMax([Boost(inner, 2)])
    with pytest.raises(TypeError):
        Boost(DisMax(["a", "b"]), 2)
    with pytest.raises(TypeError):
        Field("t", DisMax(["a"]))
    for bad in (3, None, [], ["a", 3]):
        with pytest.raises(TypeError):
            DisMax([bad])
    # accepted wherever a clause is; one clause towards mm
    q = Or([DisMax(["a", "b"]), "c"], mm=2)
    assert isinstance(q.clauses[0], DisMax) and q.weights == [1.0, 1.0] and q.mm == 2 and not q.boosted
    assert And([DisMax(["a", "b"]), "c"]).mm == 2
    b = Bool(must=[DisMax(["a", Boost("b", 2)])], should=[DisMax(["c", "d"]), "e"], filter=[DisMax(["f", "g"])],
             must_not=[DisMax(["h"])], mm="100%")
    assert b.mm == 2 and b.must_weights == [1.0]
    # a boosted member in filter / must_not
    for role in ("filter", "must_not"):
        with pytest.raises(ValueError):
            Bool(should=["a"], **{role: [DisMax(["b", Boost("c", 2)])]})
        Bool(should=["a"], **{role: [DisMax(["b", Boost("c", 1)])]})
    # the 64-clause limit counts members
    DisMax([f"t{i}" for i in range(64)])
    with pytest.raises(ValueError, match="at most 64"):
        DisMax([f"t{i}" for i in range(65)])
    Or([DisMax([f"t{i}" for i in range(32)]), DisMax([f"u{i}" for i in range(32)])])
    with pytest.raises(ValueError, match="at most 64"):
        Or([DisMax([f"t{i}" for i in range(32)]), DisMax([f"u{i}" for i in range(32)]), "x"])
    with pytest.raises(ValueError, match="at most 64"):
        Bool(should=["x"], must_not=[DisMax([f"t{i}" for i in range(64)])])


def test_flatten_groups_and_ties():
    from searcharray_b200 import Bool, Boost, DisMax, Field, Or
    from searcharray_b200.query import (SA_OCCUR_FILTER, SA_OCCUR_MUST, SA_OCCUR_MUST_NOT, SA_OCCUR_SHOULD,
                                        DISMAX, OCCUR, OR_AND, dismax_members, flatten_bool, has_dismax, has_field,
                                        is_boolean)
    qs = [Or(["a", DisMax(["b", Boost("c", 2)], tie=0.25)], mm=2),
          Bool(must=[DisMax([["p", "q"], "r"], tie=1)], should=["s", DisMax(["t"], tie=0.5)],
               filter=[DisMax(["u", "v"])], must_not=["w", DisMax(["x", "y", "z"], tie=0.1)]),
          DisMax(["m", Boost("n", 3)], tie=0.3),
          Bool(must=["plain"], should=[Boost("k", 2)])]
    clauses, starts, cnode, mm, weights, occurs, groups, ties, nq = flatten_bool(qs, DISMAX)
    assert cnode is None and nq == 4
    assert clauses == ["a", "b", "c", ["p", "q"], "r", "s", "t", "u", "v", "w", "x", "y", "z", "m", "n", "plain", "k"]
    assert starts.tolist() == [0, 3, 13, 15, 17] and starts.dtype == np.uint32
    assert mm.tolist() == [2, 0, 1, 0]
    assert weights.tolist() == [1, 1, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 3, 1, 2] and weights.dtype == np.float32
    S, M, F, N = SA_OCCUR_SHOULD, SA_OCCUR_MUST, SA_OCCUR_FILTER, SA_OCCUR_MUST_NOT
    assert occurs.tolist() == [S, S, S, M, M, S, S, F, F, N, N, N, N, S, S, M, S] and occurs.dtype == np.uint8
    assert groups.tolist() == [0, 1, 1, 3, 3, 5, 6, 7, 7, 9, 10, 10, 10, 13, 13, 15, 16] and groups.dtype == np.uint32
    assert ties.dtype == np.float32
    assert ties.tolist() == [0, .25, .25, 1, 1, 0, .5, 0, 0, 0, np.float32(.1), np.float32(.1), np.float32(.1),
                             np.float32(.3), np.float32(.3), 0, 0]
    assert dismax_members(qs) == [1, 2, 3, 4, 6, 7, 8, 10, 11, 12, 13, 14]
    assert [has_dismax(q) for q in qs] == [True, True, True, False] and all(is_boolean(q) for q in qs)
    # queries without a DisMax: flattened for DISMAX, the OCCUR arrays plus plain groups; OR_AND / OCCUR unchanged
    plain = [Or(["a", "b"]), Bool(must=["c"], should=[Boost("d", 2)], must_not=["e"])]
    got, want = flatten_bool(plain, DISMAX), flatten_bool(plain, OCCUR)
    assert got.clauses == want.clauses and want.groups is None and want.ties is None
    for f in ("node_starts", "mm", "weights", "occurs"):
        assert np.array_equal(getattr(got, f), getattr(want, f))
    assert got.groups.tolist() == [0, 1, 2, 3, 4] and not got.ties.any()
    assert flatten_bool(plain[:1], OR_AND).clauses == ["a", "b"]
    # Field members are seen inside a DisMax
    assert has_field(Or([DisMax(["a", Field("t", "b")])])) and has_field(DisMax([Field("t", "b")]))
    assert not has_field(Or([DisMax(["a", "b"])]))


def test_refusals():
    """Every refusal, before any device work."""
    from searcharray_b200 import Bool, Boost, DisMax, Field, Or, bm25_impact, bm25_similarity, fields_topk
    fr = frame_of(t=["a b", "b c", "c"], o=["x a", "a", "y"])
    arr = fr["t"].array
    dq = [DisMax(["a", "b"], tie=0.1), Or([DisMax(["a", "c"]), "b"])]
    # views and non-BM25 similarities, as Bool
    with pytest.raises(NotImplementedError):
        arr[np.array([True, False, True])].search_topk(dq, k=2)
    with pytest.raises(TypeError):
        arr.search_topk(dq, k=2, similarity=bm25_impact())
    # Field members in search_topk
    with pytest.raises(ValueError, match="fields_topk"):
        arr.search_topk([DisMax([Field("t", "a"), "b"])], k=2)
    with pytest.raises(ValueError, match="fields_topk"):
        arr.search_topk(["a", Bool(should=["a"], must_not=[DisMax([Field("t", "b")])])], k=2)
    # members need sparse-safe parameters; plain queries in the same batch do not run first
    for sim in (bm25_similarity(k1=0.0), bm25_similarity(b=1.0), bm25_similarity(b=1.5), bm25_similarity(b=-0.1),
                bm25_similarity(k1=float("nan"))):
        with pytest.raises(ValueError, match="DisMax members"):
            arr.search_topk(["a", dq[0]], k=2, similarity=sim)
        with pytest.raises(ValueError, match="DisMax members"):
            fields_topk(fr, [DisMax([Field("t", "a"), Field("o", "a")])], similarity={"o": sim})
    # fields_topk: every member names its column, views, similarities
    with pytest.raises(ValueError, match="names its column"):
        fields_topk(fr, [DisMax([Field("t", "a"), "a"])])
    with pytest.raises(ValueError, match="names its column"):
        fields_topk(fr, [Bool(should=[Field("t", "a")], must_not=[DisMax([Field("o", "x"), ["a", "b"]])])])
    with pytest.raises(TypeError):
        fields_topk(fr, [DisMax([Field("t", "a"), Field("o", "a")])], similarity=bm25_impact())
    view = pd.DataFrame({"t": fr["t"].array[np.array([True, False, True])],
                         "o": fr["o"].array[np.array([True, False, True])]})
    with pytest.raises(NotImplementedError):
        fields_topk(view, [DisMax([Field("t", "a"), Field("o", "a")])])
    wide = frame_of(**{f"f{i}": ["a", "b"] for i in range(9)})
    with pytest.raises(ValueError, match="at most 8"):
        fields_topk(wide, [DisMax([Field(f"f{i}", "a") for i in range(9)])])
    with pytest.raises(ValueError):
        Bool(should=[Field("t", "a")], filter=[DisMax([Boost(Field("o", "a"), 2)])])
    # none of the above touched a device
    for col in ("t", "o"):
        assert fr[col].array._shared["dev"] is None
    assert wide["f0"].array._shared["dev"] is None


def oracle_scorer(hosts, rec):
    """score(clause) over the oracle: a Field on its column, a plain clause on the record's one column."""
    from oracle import search as osearch
    out = {}
    for f, host in hosts.items():
        o = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                                avg_doc_length=host.avg_doc_length)
        k1, b = rec["sim"].get(f, [1.2, 0.75])
        out[f] = oracle_score(o, host.term_dict, k1=k1, b=b, slop=rec["slop"])
    from searcharray_b200 import Field
    by_field = field_scorer(out)
    return lambda c: by_field(c) if isinstance(c, Field) else out[rec["field"]](c)


def test_oracle_composition_golden(fixture):
    """The oracle's composition reproduces the real reference's composed top 10 (ids, score bits, n_ranked) of every
    record, and our mm parsing resolves each Solr spec as the reference's did."""
    from searcharray_b200 import DisMax
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    hosts = {f: load_field(z, f) for f in (T, O)}
    recs = fixture["queries"]
    assert len(recs) >= 35 and sum(r["edismax"] is not None for r in recs) >= 10
    for group in record_groups(recs).values():
        score = oracle_scorer(hosts, group[0])
        for rec in group:
            q = query_of(rec)
            assert (1 if isinstance(q, DisMax) else q.mm) == rec["mm"], rec["mm_spec"]
            v = compose_dismax(score, q)
            ids, scores = topk(v, 10)
            n = len(rec["top_ids"])
            what = f"{q!r} slop={rec['slop']} sim={rec['sim']}"
            assert int(np.count_nonzero(v > 0)) == rec["n_ranked"], what
            assert ids[:n].tolist() == rec["top_ids"] and np.all(ids[n:] == 0xFFFFFFFF), what
            assert scores[:n].view(np.uint32).tolist() == rec["top_bits"], what


def test_single_member_composes_as_its_member(fixture):
    """DisMax([c]) composes bit for bit as c, in every role, at every tie (v + (v - v) * tie == v for v >= +0)."""
    from searcharray_b200 import Bool, Boost, DisMax
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    rec = {"sim": {}, "slop": 0, "field": O}
    score = oracle_scorer({O: load_field(z, O)}, rec)
    for tie in (0.0, 0.3, 1.0):
        for c in ("love", Boost("war", 2.5), ["New", "York"], Boost("zzzz", 3)):
            def one(x):
                return DisMax([x], tie=tie)
            for build in (lambda x: Bool(must=[x], should=["young"]), lambda x: Bool(should=[x, "man"], mm=1),
                          lambda x: Bool(filter=[x], should=["city"]), lambda x: Bool(should=["city"], must_not=[x])):
                try:
                    plain = build(c)
                except ValueError:                  # a boost in filter / must_not
                    continue
                a, b = compose_dismax(score, plain), compose_dismax(score, build(one(c)))
                assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), (c, tie)
