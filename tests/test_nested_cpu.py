"""CPU: nested boolean queries (an Or / And / Bool as a clause of another) -- accepted forms, every refusal (raised
before any device work, so on CPU-built arrays), flatten_bool's node arrays, and the oracle composition against the
real reference's composed results (tests/golden/nested.json, make_golden_nested.py)."""
import json
import os

import numpy as np
import pandas as pd
import pytest

from _bool_compose import oracle_score, topk
from _bool_fields_compose import field_scorer
from _nested_compose import compose_nested, query_of
from _tmdb_index import load_field
from conftest import GOLDEN

T, O = "title_tokens", "overview_tokens"


@pytest.fixture(scope="module")
def fixture():
    with open(os.path.join(GOLDEN, "nested.json")) as f:
        return json.load(f)


def frame_of(**cols):
    from searcharray_b200 import SearchArray
    return pd.DataFrame({name: SearchArray.index(docs) for name, docs in cols.items()})


def test_accepted_forms():
    from searcharray_b200 import And, Bool, Boost, DisMax, Field, Or
    from searcharray_b200.query import is_nested
    a_b = And(["a", "b"])
    q = Or([a_b, And(["a", "c"])])
    assert q.clauses[0] is a_b and q.weights == [1.0, 1.0] and q.mm == 1 and is_nested(q)
    assert Or([a_b, "c"], mm=2).mm == 2                      # a nested query counts once towards mm
    b = Bool(must=[Boost(Or(["x", "y"]), 2)], should=[a_b], filter=[Or(["f"])], must_not=[Bool(should=["n"])])
    assert b.must_weights == [2.0] and isinstance(b.must[0], Or) and is_nested(b)
    assert Boost(a_b, 0).weight == 0 and Boost(Bool(should=["x"]), 1.5).clause.should == ["x"]
    assert is_nested(Or([Or([Or([DisMax(["a", "b"])])])]))  # depth and a DisMax inside
    assert is_nested(Or([Field("t", "a"), And([Field("o", "b")])]))
    assert not is_nested(Or(["a", DisMax(["b"])])) and not is_nested(DisMax(["a"]))


def test_refusals_in_the_api():
    from searcharray_b200 import And, Bool, Boost, DisMax, Field, Or
    from searcharray_b200.query import SA_BOOL_MAX_CLAUSES, SA_BOOL_MAX_NESTED
    sub = Or(["a", "b"])
    for role in ("filter", "must_not"):                      # a Boost where nothing scores
        with pytest.raises(ValueError):
            Bool(should=["x"], **{role: [Boost(sub, 2)]})
    for inner in (sub, And(["a"]), Bool(should=["a"])):
        with pytest.raises(TypeError):
            DisMax(["a", inner])                              # no nested query in a DisMax
        with pytest.raises(TypeError):
            DisMax([Boost(inner, 2)])
        with pytest.raises(TypeError):
            Field("t", inner)                                 # fields sit on leaves
        with pytest.raises(TypeError):
            Boost(Boost(inner, 2), 2)
    with pytest.raises(TypeError):
        Boost(DisMax(["a"]), 2)
    # 64 leaves in the whole tree, DisMax members counted
    half = Or(["a"] * 32)
    Or([half, half])
    with pytest.raises(ValueError, match="clauses"):
        Or([half, half, "x"])
    with pytest.raises(ValueError, match="clauses"):
        Bool(must=[Or([DisMax(["a"] * 40)])], should=[Or(["b"] * 24)], filter=["c"])
    with pytest.raises(ValueError, match="clauses"):
        Or([And([Or(["a"] * 60)]), Or(["b"] * 5)])
    # 64 nested queries, at any depth, a reused object counting each time
    leaf = Or(["a"])
    assert Or([leaf] * SA_BOOL_MAX_NESTED).n_nested == SA_BOOL_MAX_NESTED
    chain = Or(["a"])
    for _ in range(SA_BOOL_MAX_NESTED - 1):
        chain = Or([chain])
    Or([chain])
    with pytest.raises(ValueError, match="nested"):
        Or([Or([chain])])
    pair = Or([Or(["a"]) for _ in range(32)])                # 33 nested queries each
    with pytest.raises(ValueError, match="nested"):
        Bool(must=[pair], should=[pair])
    assert SA_BOOL_MAX_CLAUSES == 64


def test_flatten_nested_arrays():
    """A hand-written tree: nodes in pre-order after the top-level queries, a shared sub-query as two nodes."""
    from searcharray_b200 import And, Bool, Boost, DisMax, Or
    from searcharray_b200.query import SA_NO_NODE as X, DISMAX, NESTED, dismax_members, flatten_bool
    shared = And(["s", "t"])
    q0 = Bool(must=["a", Or([shared, ["p", "q"]], mm=2)], should=[Boost(shared, 2), DisMax(["d", "e"], tie=0.5)],
              must_not=[shared])
    q1 = Or(["z"])
    clauses, starts, cnode, mm, weights, occurs, groups, ties, nq = flatten_bool([q0, q1], NESTED)
    assert nq == 2
    # nodes: 0 q0, 1 q1, 2 Or([shared, p q]), 3 shared (in 2), 4 Boost(shared), 5 shared (must_not)
    assert starts.tolist() == [0, 6, 7, 9, 11, 13, 15]
    assert clauses == ["a", None, None, "d", "e", None, "z", None, ["p", "q"], "s", "t", "s", "t", "s", "t"]
    assert cnode.tolist() == [X, 2, 4, X, X, 5, X, 3, X, X, X, X, X, X, X]
    assert mm.tolist() == [0, 1, 2, 2, 2, 2]
    assert weights.tolist() == [1, 1, 2, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1, 1]
    assert occurs.tolist() == [1, 1, 0, 0, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0]
    assert groups.tolist() == [0, 1, 2, 3, 3, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14]
    assert ties.tolist() == [0, 0, 0, 0.5, 0.5, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0]
    assert dismax_members([q0, q1]) == [3, 4]
    # every reference points forward, to a nested node, once
    refs = [int(c) for c in cnode if c != X]
    assert sorted(refs) == list(range(2, 6))
    for n in range(len(starts) - 1):
        for c in range(starts[n], starts[n + 1]):
            assert cnode[c] == X or cnode[c] > n
    # a batch without nested queries flattened for NESTED: the DISMAX arrays, with no nested clause
    plain = [Or(["a", DisMax(["b", "c"])]), Bool(must=["m"], should=[Boost("s", 2)], must_not=["n"])]
    got, want = flatten_bool(plain, NESTED), flatten_bool(plain, DISMAX)
    assert got.clauses == want.clauses and all(c == X for c in got.clause_node) and want.clause_node is None
    for f in ("node_starts", "mm", "weights", "occurs", "groups", "ties"):
        assert np.array_equal(getattr(got, f), getattr(want, f))
    assert got.n_queries == want.n_queries == 2


def test_helpers_see_inside_nested_queries():
    from searcharray_b200 import And, Bool, DisMax, Field, Or
    from searcharray_b200.query import has_dismax, has_field
    assert has_field(Or(["a", Or(["b", And([Field("t", "c")])])]))
    assert has_field(Bool(should=["a"], must_not=[Or([DisMax(["x", Field("t", "y")])])]))
    assert not has_field(Or(["a", Or(["b", And(["c"])])]))
    assert has_dismax(Or(["a", Or([DisMax(["b", "c"])])])) and not has_dismax(Or(["a", Or(["b"])]))


def test_refusals_before_device_work():
    """A Field hidden in a nested query, views, similarities, DisMax parameters and fields_topk's checks."""
    from searcharray_b200 import And, Bool, DisMax, Field, Or, bm25_impact, bm25_similarity, fields_topk
    fr = frame_of(t=["a b", "b c", "c"], o=["x a", "a", "y"])
    arr = fr["t"].array
    nq = [Or([And(["a", "b"]), "c"]), Bool(must=[Or(["a", "c"])], should=["b"])]
    with pytest.raises(ValueError, match="fields_topk"):
        arr.search_topk(["a", Or(["b", And(["c", Field("t", "a")])])], k=2)
    with pytest.raises(ValueError, match="fields_topk"):
        arr.search_topk([Bool(should=["a"], must_not=[Or([DisMax(["x", Field("t", "b")])])])], k=2)
    with pytest.raises(NotImplementedError):
        arr[np.array([True, False, True])].search_topk(nq, k=2)
    with pytest.raises(TypeError):
        arr.search_topk(nq, k=2, similarity=bm25_impact())
    # DisMax members inside nested queries need sparse-safe parameters
    with pytest.raises(ValueError, match="DisMax members"):
        arr.search_topk(["a", Or([And([DisMax(["a", "b"]), "c"])])], k=2, similarity=bm25_similarity(k1=0.0))
    with pytest.raises(ValueError, match="DisMax members"):
        fields_topk(fr, [Or([Or([DisMax([Field("t", "a"), Field("o", "a")])])])], similarity={"o": bm25_similarity(b=1.0)})
    # fields_topk: every leaf at any depth names its column
    with pytest.raises(ValueError, match="names its column"):
        fields_topk(fr, [Or([Field("t", "a"), And([Field("o", "a"), "b"])])])
    with pytest.raises(ValueError, match="names its column"):
        fields_topk(fr, [Bool(should=[Field("t", "a")], must_not=[Or([Or([["a", "b"]])])])])
    with pytest.raises(TypeError):
        fields_topk(fr, [Or([And([Field("t", "a"), Field("o", "a")])])], similarity=bm25_impact())
    view = pd.DataFrame({"t": fr["t"].array[np.array([True, False, True])],
                         "o": fr["o"].array[np.array([True, False, True])]})
    with pytest.raises(NotImplementedError):
        fields_topk(view, [Or([And([Field("t", "a"), Field("o", "a")])])])
    wide = frame_of(**{f"f{i}": ["a", "b"] for i in range(9)})
    with pytest.raises(ValueError, match="at most 8"):
        fields_topk(wide, [Or([Field("f0", "a"), Or([Field(f"f{i}", "a") for i in range(1, 9)])])])
    for col in ("t", "o"):
        assert fr[col].array._shared["dev"] is None
    assert wide["f0"].array._shared["dev"] is None


def oracle_scorer(hosts, rec):
    """score(clause) over the oracle: a Field on its column, a plain clause on the record's one column."""
    from oracle import search as osearch
    from searcharray_b200 import Field
    out = {}
    for f, host in hosts.items():
        o = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                                avg_doc_length=host.avg_doc_length)
        k1, b = rec["sim"].get(f, [1.2, 0.75])
        out[f] = oracle_score(o, host.term_dict, k1=k1, b=b, slop=rec["slop"])
    by_field = field_scorer(out)
    return lambda c: by_field(c) if isinstance(c, Field) else out[rec["field"]](c)


def test_oracle_composition_golden(fixture):
    """The oracle's composition reproduces the real reference's composed top 10 (ids, score bits, n_ranked) of every
    record, and our mm parsing resolves each Solr spec as the reference's did."""
    from searcharray_b200.query import is_nested
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    hosts = {f: load_field(z, f) for f in (T, O)}
    recs = fixture["queries"]
    assert len(recs) >= 25
    for rec in recs:
        q = query_of(rec)
        assert is_nested(q) and q.mm == rec["mm"], rec["mm_spec"]
        v = compose_nested(oracle_scorer(hosts, rec), q)
        ids, scores = topk(v, 10)
        n = len(rec["top_ids"])
        what = f"{q!r} slop={rec['slop']} sim={rec['sim']}"
        assert int(np.count_nonzero(v > 0)) == rec["n_ranked"], what
        assert ids[:n].tolist() == rec["top_ids"] and np.all(ids[n:] == 0xFFFFFFFF), what
        assert scores[:n].view(np.uint32).tolist() == rec["top_bits"], what


def test_one_leaf_or_composes_as_its_leaf(fixture):
    """Or([a, Or([b])]) composes bit for bit as Or([a, b]); a nested Or of two leaves in general does not flatten."""
    from searcharray_b200 import Bool, Or
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    rec = {"sim": {}, "slop": 0, "field": O}
    score = oracle_scorer({O: load_field(z, O)}, rec)
    for a, b in (("love", "war"), ("young", ["New", "York"]), ("city", "zzzz")):
        for flat, nest in ((Or([a, b]), Or([a, Or([b])])), (Or([a, b], mm=2), Or([a, Or([b])], mm=2)),
                           (Bool(must=[a], should=[b]), Bool(must=[a], should=[Or([b])])),
                           (Bool(should=[a], must_not=[b]), Bool(should=[a], must_not=[Or([b])]))):
            x, y = compose_nested(score, flat), compose_nested(score, nest)
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), (a, b)
    flat, nest = Or(["young", "man", "love"], mm=2), Or(["young", Or(["man", "love"])], mm=2)
    assert not np.array_equal(compose_nested(score, flat), compose_nested(score, nest))
