"""CPU: Bool (must / should / filter / must_not) and Boost in search_topk (searcharray_b200/query.py) --
validation, mm defaults, the clause limit, flattening into the OCCUR arrays -- and the oracle
composition against the real reference's composed results (tests/golden/bool_occur.json,
make_golden_bool_occur.py)."""
import json
import os

import numpy as np
import pytest

from _bool_compose import expand, oracle_score, topk
from _bool_occur_compose import compose_occur, query_of
from _tmdb_index import load_field
from conftest import GOLDEN


@pytest.fixture(scope="module")
def fixture():
    with open(os.path.join(GOLDEN, "bool_occur.json")) as f:
        return json.load(f)


def test_boost_validation():
    from searcharray_b200 import And, Bool, Boost, Or
    b = Boost("a", 0.1)
    assert b.clause == "a" and b.weight.dtype == np.float32 and b.weight == np.float32(0.1)
    assert Boost(("a", "b"), 2).clause == ["a", "b"] and Boost("a", 0).weight == 0
    for w in (-1.0, -1e-30, float("inf"), float("-inf"), float("nan")):
        with pytest.raises(ValueError):
            Boost("a", w)
    for bad in (3, [], ["a", 3], None, Boost("a", 2.0)):
        with pytest.raises(TypeError):
            Boost(bad, 2.0)
    # accepted wherever a clause scores
    q = Or(["a", Boost(["b", "c"], 2.5), Boost("d", 0)], mm=2)
    assert q.clauses == ["a", ["b", "c"], "d"] and q.weights == [1.0, 2.5, 0.0] and q.mm == 2 and q.boosted
    assert And([Boost("a", 3), "b"]).mm == 2
    assert not Or(["a", Boost("b", 1.0)]).boosted
    bq = Bool(must=[Boost("a", 2)], should=[Boost(["b", "c"], 0.5), "d"])
    assert bq.must == ["a"] and bq.must_weights == [2.0] and bq.should_weights == [0.5, 1.0]
    for role in ("filter", "must_not"):
        with pytest.raises(ValueError):
            Bool(should=["a"], **{role: [Boost("b", 2)]})
    # Or's TypeErrors are unchanged, and Bool raises the same in every list
    for bad in (3, [], ["a", 3], None):
        with pytest.raises(TypeError):
            Or(["x", bad])
        for role in ("must", "filter", "must_not"):
            with pytest.raises(TypeError):
                Bool(should=["x"], **{role: ["y", bad]})
        with pytest.raises(TypeError):
            Bool(should=["x", bad])


def test_bool_validation_and_mm():
    from searcharray_b200 import Bool
    from searcharray_b200.query import SA_BOOL_MAX_CLAUSES
    assert Bool(should=["a", "b"]).mm == 1
    assert Bool(must=["a"], should=["b", "c"]).mm == 0
    assert Bool(filter=["a"], should=["b", "c"]).mm == 0
    assert Bool(must_not=["a"], should=["b", "c"]).mm == 1
    assert Bool(must=["a"]).mm == 0
    assert Bool(must=["a"], should=["b", "c", "d"], mm=2).mm == 2
    assert Bool(must=["a"], should=["b", "c", "d", "e"], mm="75%").mm == 3
    assert Bool(should=["b", "c"], mm=5).mm == 2                       # clamped to the should clauses
    assert Bool(must=["a", "x"], should=["b", "c", "d"], mm=-1).mm == 2
    assert Bool(must=["a"], mm=3).mm == 0
    with pytest.raises(ValueError):
        Bool(should=["a"], mm="x")
    for kw in ({}, {"filter": ["a"]}, {"must_not": ["a"]}, {"filter": ["a"], "must_not": ["b"]}):
        with pytest.raises(ValueError):
            Bool(**kw)
    n = SA_BOOL_MAX_CLAUSES
    Bool(must=["a"] * 16, should=["b"] * 16, filter=["c"] * 16, must_not=["d"] * 16)
    for split in ((n - 2, 1, 1, 1), (1, n - 2, 1, 1), (1, 1, n - 2, 1), (1, 1, 1, n - 2), (n + 1, 0, 0, 0)):
        with pytest.raises(ValueError):
            Bool(must=["a"] * split[0], should=["b"] * split[1], filter=["c"] * split[2], must_not=["d"] * split[3])


def test_flatten_occur():
    from searcharray_b200 import And, Bool, Boost, Or
    from searcharray_b200.query import OCCUR, OR_AND, flatten_bool
    queries = [Or(["a", Boost(["b", "c"], 2)], mm=2), And(["d"]),
               Bool(must=[Boost("m", 0.5)], should=["s", "t"], filter=[["f", "g"]], must_not=["n"], mm=1),
               Bool(must_not=["x"], should=[Boost("y", 3)])]
    clauses, starts, _, mm, weights, occurs, _, _, _ = flatten_bool(queries, OCCUR)
    assert clauses == ["a", ["b", "c"], "d", "m", "s", "t", ["f", "g"], "n", "y", "x"]
    assert starts.dtype == np.uint32 and starts.tolist() == [0, 2, 3, 8, 10]
    assert mm.dtype == np.uint32 and mm.tolist() == [2, 1, 1, 1]
    assert weights.dtype == np.float32 and weights.tolist() == [1, 2, 1, 0.5, 1, 1, 1, 1, 3, 1]
    assert occurs.dtype == np.uint8 and occurs.tolist() == [0, 0, 0, 1, 0, 0, 2, 3, 0, 3]
    # the plain flatten of unboosted Or / And is what it was; a boosted Or flattens to its clauses
    c, s, _, m, *_ = flatten_bool([Or(["a", ["b", "c"]], mm=2), And(["d"]), Or(["a", Boost("e", 2)], mm=0)], OR_AND)
    assert c == ["a", ["b", "c"], "d", "a", "e"] and s.tolist() == [0, 2, 3, 5] and m.tolist() == [2, 1, 0]
    # an Or / And batch flattened for OCCUR: the same arrays, every clause SHOULD with weight 1
    plain = [Or(["a", ["b", "c"]], mm=2), And(["d"])]
    lo, hi = flatten_bool(plain, OR_AND), flatten_bool(plain, OCCUR)
    assert hi.clauses == lo.clauses and np.array_equal(hi.node_starts, lo.node_starts)
    assert np.array_equal(hi.mm, lo.mm) and hi.weights.tolist() == [1, 1, 1] and hi.occurs.tolist() == [0, 0, 0]


def test_rejected_without_a_device():
    """A Bool or boosted Or on a view, or under a similarity other than bm25_similarity, is refused as Or is."""
    from searcharray_b200 import Bool, Boost, Or, SearchArray, bm25_impact
    arr = SearchArray.index(["foo bar", "bar baz", "baz"])
    for q in (Bool(must=["foo"], should=["bar"]), Or(["foo", Boost("bar", 2)])):
        with pytest.raises(NotImplementedError):
            arr[np.array([True, False, True])].search_topk([q], k=2)
        with pytest.raises(NotImplementedError):
            arr[1:].search_topk(["foo", q], k=2)
        with pytest.raises(TypeError):
            arr.search_topk([q], k=2, similarity=bm25_impact())


def golden_scorers(fixture):
    from oracle import search as osearch
    from searcharray_b200 import ws_tokenizer
    from searcharray_b200.indexing import build_index
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    hosts = {f: load_field(z, f) for f in ("title_tokens", "overview_tokens")}
    hosts["scenario"] = build_index(expand(fixture["scenario_docs"]), ws_tokenizer)
    score = {}
    for name, host in hosts.items():
        o = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                                avg_doc_length=host.avg_doc_length)
        score[name] = oracle_score(o, host.term_dict)
    return score


def test_oracle_composition_golden(fixture):
    """The oracle's composition reproduces the real reference's composed top 10 (ids, score bits, n_ranked) of every
    Bool / boosted Or record."""
    score = golden_scorers(fixture)
    recs = fixture["queries"]
    assert len(recs) >= 20
    for rec in recs:
        q = query_of(rec)
        v = compose_occur(score[rec["corpus"]], q)
        ids, scores = topk(v, 10)
        n = len(rec["top_ids"])
        what = f"{rec['corpus']} {q!r}"
        assert int(np.count_nonzero(v > 0)) == rec["n_ranked"], what
        assert ids[:n].tolist() == rec["top_ids"] and np.all(ids[n:] == 0xFFFFFFFF), what
        assert scores[:n].view(np.uint32).tolist() == rec["top_bits"], what
