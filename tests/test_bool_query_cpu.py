"""CPU: boolean queries for search_topk (searcharray_b200/query.py) -- validation, mm parsing, flattening into the
C-ABI arrays, the rejected cases -- and the oracle composition against the reference's own and/or scenarios and
its composed TMDB results (tests/golden/bool_scenarios.json, make_golden_bool.py)."""
import json
import os

import numpy as np
import pytest

from _bool_compose import compose, expand, oracle_score, topk
from _tmdb_index import load_field
from conftest import GOLDEN


@pytest.fixture(scope="module")
def fixture():
    with open(os.path.join(GOLDEN, "bool_scenarios.json")) as f:
        return json.load(f)


def test_or_and_validation():
    from searcharray_b200 import And, Or
    from searcharray_b200.query import SA_BOOL_MAX_CLAUSES
    q = Or(["a", ["b", "c"], ("d", "e")])
    assert q.clauses == ["a", ["b", "c"], ["d", "e"]] and q.mm == 1
    assert And(["a", "b", ["c", "d"]]).mm == 3
    assert Or(["a"] * SA_BOOL_MAX_CLAUSES).mm == 1
    with pytest.raises(ValueError):
        Or([])
    with pytest.raises(ValueError):
        And([])
    with pytest.raises(ValueError):
        Or(["a"] * (SA_BOOL_MAX_CLAUSES + 1))
    for bad in (3, [], ["a", 3], None):
        with pytest.raises(TypeError):
            Or(["x", bad])


@pytest.mark.parametrize("mm, n, want", [(0, 3, 0), (1, 3, 1), (3, 3, 3), (5, 3, 3), (-1, 3, 2), (-7, 3, 0),
                                         ("2", 4, 2), ("75%", 4, 3), ("-25%", 4, 3), ("2<-25%", 2, 2),
                                         ("2<-25%", 8, 6), ("100%", 5, 5)])
def test_mm_parsing(mm, n, want):
    """mm goes through solr.parse_min_should_match(n, str(mm)): clamped to [0, n] as edismax clamps it."""
    from searcharray_b200 import Or
    from searcharray_b200.solr import parse_min_should_match
    assert Or([f"t{i}" for i in range(n)], mm=mm).mm == want == parse_min_should_match(n, str(mm))
    with pytest.raises(ValueError):
        Or(["a", "b"], mm="x")


def test_flatten():
    from searcharray_b200 import And, Or
    from searcharray_b200.query import OR_AND, flatten_bool
    clauses, starts, _, mm, *_ = flatten_bool([Or(["a", ["b", "c"]], mm=2), And(["d"]), Or(["a", "a", "e"], mm=0)],
                                             OR_AND)
    assert clauses == ["a", ["b", "c"], "d", "a", "a", "e"]
    assert starts.dtype == np.uint32 and starts.tolist() == [0, 2, 3, 6]
    assert mm.dtype == np.uint32 and mm.tolist() == [2, 1, 0]


def test_bool_form_and_the_arrays_each_form_leaves_none():
    """bool_form orders the query kinds OR_AND < OCCUR < DISMAX < NESTED, and flatten_bool builds only the arrays the
    form reads: the others are None, passed as NULL, which selects that form's instance."""
    from searcharray_b200 import And, Bool, Boost, DisMax, Or
    from searcharray_b200.query import DISMAX, NESTED, OCCUR, OR_AND, bool_form, flatten_bool
    assert OR_AND < OCCUR < DISMAX < NESTED
    kinds = {OR_AND: [Or(["a", "b"]), And(["a", ["b", "c"]]), Or(["a", Boost("b", 1.0)])],
             OCCUR: [Or(["a", Boost("b", 2)]), Bool(must=["a"]), Bool(should=["a"], must_not=["b"])],
             DISMAX: [DisMax(["a", "b"]), Or(["a", DisMax(["b"])]), Bool(filter=[DisMax(["a", "b"])], should=["c"])],
             NESTED: [Or(["a", And(["b", "c"])]), Bool(must=[Boost(Or(["a"]), 2)]),
                      Or([DisMax(["a", "b"]), Bool(should=["c"])])]}
    for form, qs in kinds.items():
        assert [bool_form(q) for q in qs] == [form] * len(qs), form
    for form, qs in kinds.items():
        b = flatten_bool(qs, form)
        assert b.n_queries == len(qs) and b.node_starts is not None and b.mm is not None
        assert (b.weights is None, b.occurs is None) == ((form == OR_AND,) * 2)
        assert (b.groups is None, b.ties is None) == ((form < DISMAX,) * 2)
        assert (b.clause_node is None) == (form < NESTED)


def test_rejected_without_a_device():
    """A boolean query on a view, or under a similarity other than bm25_similarity, is refused before any device
    work."""
    from searcharray_b200 import Or, SearchArray, bm25_impact
    arr = SearchArray.index(["foo bar", "bar baz", "baz"])
    with pytest.raises(NotImplementedError):
        arr[np.array([True, False, True])].search_topk([Or(["foo", "bar"])], k=2)
    with pytest.raises(NotImplementedError):
        arr[1:].search_topk(["foo", Or(["foo"])], k=2)
    with pytest.raises(TypeError):
        arr.search_topk([Or(["foo", "bar"])], k=2, similarity=bm25_impact())


def scenario_oracle(rec):
    from oracle import search as osearch
    from searcharray_b200 import ws_tokenizer
    from searcharray_b200.indexing import build_index
    host = build_index(expand(rec["docs"]), ws_tokenizer)
    o = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                            avg_doc_length=host.avg_doc_length)
    return oracle_score(o, host.term_dict)


@pytest.mark.parametrize("kind", ["and", "or"])
def test_oracle_composition_scenarios(fixture, kind):
    """The oracle's composition reproduces the reference's and/or scenario masks and its composed top 10."""
    for rec in fixture[kind]:
        s, ok = compose(scenario_oracle(rec), rec["clauses"], rec["mm"])
        assert np.array_equal(ok, np.asarray(expand(rec["expected"]))), rec["name"]
        ids, scores = topk(s, 10)
        n = len(rec["top_ids"])
        assert ids[:n].tolist() == rec["top_ids"] and np.all(ids[n:] == 0xFFFFFFFF), rec["name"]
        assert scores[:n].view(np.uint32).tolist() == rec["top_bits"], rec["name"]


def test_oracle_composition_tmdb(fixture):
    """The oracle's composition on the TMDB fields reproduces the real reference's composed top 10, id and bits."""
    from oracle import search as osearch
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    score = {}
    for field in ("title_tokens", "overview_tokens"):
        host = load_field(z, field)
        o = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                                avg_doc_length=host.avg_doc_length)
        score[field] = oracle_score(o, host.term_dict)
    assert len(fixture["tmdb"]) >= 20
    for rec in fixture["tmdb"]:
        s, _ = compose(score[rec["field"]], rec["clauses"], rec["mm"])
        ids, scores = topk(s, 10)
        n = len(rec["top_ids"])
        what = f"{rec['field']} {rec['clauses']} mm={rec['mm']}"
        assert int(np.count_nonzero(s > 0)) == rec["n_ranked"], what
        assert ids[:n].tolist() == rec["top_ids"], what
        assert scores[:n].view(np.uint32).tolist() == rec["top_bits"], what
