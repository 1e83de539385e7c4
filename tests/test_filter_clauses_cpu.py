"""CPU: range and code-set filter clauses (query.Range over SearchArray.set_feature columns, query.In over
SearchArray.set_facet columns) -- construction refusals, the outward float32 rounding of range bounds, the encoded
clause entries (SA_RANGE_TERM / SA_IN_TERM), and the refusals of search_topk, score_docs and fields_topk, every one
raised before any device work (the device entry points are replaced by a trap here)."""
from fractions import Fraction

import numpy as np
import pandas as pd
import pytest

F32_MAX = float(np.finfo(np.float32).max)


class DeviceTouched(Exception):
    pass


@pytest.fixture
def no_device(monkeypatch):
    """Any device work raises DeviceTouched."""
    from searcharray_b200 import SearchArray, solr

    def trap(*a, **k):
        raise DeviceTouched()
    monkeypatch.setattr(SearchArray, "_device", trap)
    monkeypatch.setattr(solr, "_multi_for", trap)


def arr_of(docs):
    from searcharray_b200 import SearchArray
    return SearchArray.index(docs)


def f32(x):
    return float(np.float32(x))


def test_range_construction_refusals():
    from searcharray_b200 import Range
    r = Range("year", gte=1977, lt=1990)
    assert (r.name, r.gt, r.gte, r.lt, r.lte) == ("year", None, 1977.0, 1990.0, None)
    assert repr(r) == "Range('year', gte=1977.0, lt=1990.0)"
    Range("year", gt=np.float32(3)), Range("year", lte=np.int64(5)), Range("year", gte=Fraction(1, 3))
    Range("year", gte=5, lt=5)                                 # empty ranges are accepted
    Range("year", gte=1e300), Range("year", lte=-1e300), Range("year", gte=10 ** 400)
    for kw in ({}, dict(gt=1, gte=1), dict(lt=2, lte=2), dict(gte=float("nan")), dict(lt=float("inf")),
               dict(gt=-float("inf")), dict(lte=np.float64("nan"))):
        with pytest.raises(ValueError):
            Range("year", **kw)
    for kw in (dict(gte=True), dict(lt=np.bool_(False)), dict(gte="1990"), dict(lte=None, gt=[1]), dict(gte=1 + 2j),
               dict(gt=b"1")):
        with pytest.raises(TypeError):
            Range("year", **kw)
    for name in (3, None, ["year"]):
        with pytest.raises(TypeError):
            Range(name, gte=1)


def test_in_construction_refusals():
    from searcharray_b200 import In
    c = In("lang", [3, 0, 3, np.int64(7)])
    assert c.name == "lang" and c.codes == [3, 0, 3, 7] and repr(c) == "In('lang', [3, 0, 3, 7])"
    assert In("lang", (1,)).codes == [1] and In("lang", np.asarray([2, 5], dtype=np.uint16)).codes == [2, 5]
    for codes in ([], (), np.zeros(0, dtype=np.int64), [-1], [0, -3]):
        with pytest.raises(ValueError):
            In("lang", codes)
    for codes in (3, "en", None, [1.0], [True], ["en"], [1, None], np.asarray([1.5])):
        with pytest.raises(TypeError):
            In("lang", codes)
    with pytest.raises(TypeError):
        In(3, [1])


def test_outward_rounding():
    """Each bound becomes the float32 that keeps the comparison exact: gte a -> the least float32 >= a, gt a -> the
    least float32 > a, lte b -> the greatest float32 <= b, lt b -> the greatest float32 < b; +-inf where absent or
    beyond float32's range."""
    from searcharray_b200 import Range
    inf = float("inf")
    up = lambda x: float(np.nextafter(np.float32(x), np.float32(inf)))      # noqa: E731
    down = lambda x: float(np.nextafter(np.float32(x), np.float32(-inf)))   # noqa: E731
    # 0.1 is not a float32: float32(0.1) > 0.1, so gte keeps it and lte steps down
    assert f32(0.1) > 0.1
    assert Range("x", gte=0.1).bounds() == (f32(0.1), inf)
    assert Range("x", gt=0.1).bounds() == (f32(0.1), inf)
    assert Range("x", lte=0.1).bounds() == (-inf, down(0.1))
    assert Range("x", lt=0.1).bounds() == (-inf, down(0.1))
    # an exactly representable value: inclusive bounds keep it, exclusive ones step past it
    assert Range("x", gte=2.5, lte=7.0).bounds() == (2.5, 7.0)
    assert Range("x", gt=2.5, lt=7.0).bounds() == (up(2.5), down(7.0))
    # 16,777,217 = 2^24 + 1 lies between the float32s 2^24 and 2^24 + 2
    big = 16_777_217
    assert Range("x", gte=big).bounds() == (16_777_218.0, inf)
    assert Range("x", gt=big).bounds() == (16_777_218.0, inf)
    assert Range("x", lte=big).bounds() == (-inf, 16_777_216.0)
    assert Range("x", lt=big).bounds() == (-inf, 16_777_216.0)
    assert Range("x", gt=2 ** 24).bounds() == (16_777_218.0, inf)
    # beyond float32's range: the infinities
    assert Range("x", gte=1e39, lte=1e40).bounds() == (inf, inf)
    assert Range("x", gt=-1e39, lt=-1e38 * 10).bounds() == (-inf, -inf)
    assert Range("x", gt=F32_MAX).bounds() == (inf, inf)
    assert Range("x", gte=F32_MAX, lte=F32_MAX).bounds() == (F32_MAX, F32_MAX)
    assert Range("x", gte=10 ** 400).bounds() == (inf, inf)
    # the rule holds against float64 comparisons over many values and bounds
    rng = np.random.default_rng(1)
    xs = np.concatenate([rng.random(2000) * 100, rng.integers(0, 2 ** 26, 2000), [0.1, 2.5, 16_777_216, 16_777_218]])
    xs = xs.astype(np.float32)
    x64 = xs.astype(np.float64)
    for a in list(rng.random(40) * 100) + [0.1, 2.5, 16_777_217, 16_777_216, 2 ** 25 + 3]:
        for key, op in (("gte", np.greater_equal), ("gt", np.greater), ("lte", np.less_equal), ("lt", np.less)):
            lo, hi = Range("x", **{key: a}).bounds()
            want = op(x64, a)
            got = (np.float32(lo) <= xs) & (xs <= np.float32(hi))
            assert np.array_equal(got, want), (key, a)


def test_match_in_numpy():
    """Range.match / In.match, the oracles the GPU tests compare against: 0 never matches."""
    from searcharray_b200 import In, Range
    x = np.asarray([0, 0.5, 1, 1990, 1991, 2 ** 24 + 2], dtype=np.float32)
    assert Range("y", gte=1990).match(x).tolist() == [False, False, False, True, True, True]
    assert Range("y", lte=1).match(x).tolist() == [False, True, True, False, False, False]
    assert Range("y", gt=-5, lt=1991).match(x).tolist() == [False, True, True, True, False, False]
    assert not Range("y", gte=5, lt=5).match(x).any()
    codes = np.asarray([-1, 0, 3, 7, 3], dtype=np.int32)
    assert In("l", [3, 7, 3]).match(codes).tolist() == [False, False, True, True, True]


def test_encoded_entries():
    from searcharray_b200 import Bool, Boost, Feature, In, Or, Range
    from searcharray_b200.query import NESTED, OCCUR, bool_form, column_terms, flatten_bool, has_feature
    r, i = Range("year", gte=1977, lt=1990), In("lang", [4, 1, 4])
    assert bool_form(Or(["a", r])) == OCCUR and has_feature(Or(["a", i])) and bool_form(Or(["a", Or([i])])) == NESTED
    queries = [Bool(must=[Or(["star", "wars"])], filter=[r, i]), Or(["trek", Boost(r, 2), Feature("pop")])]
    batch = flatten_bool(queries, NESTED)
    assert batch.clauses[1] is r and batch.clauses[2] is i and batch.clauses[4] is r
    feature_slots, facet_slots = {"year": 2, "pop": 0}, {"lang": (5, 8)}
    enc = column_terms(batch.clauses, lambda i, c: feature_slots[c.name], lambda i, c: facet_slots[c.name])
    lo, hi = np.float32(1977).view(np.uint32), np.nextafter(np.float32(1990), np.float32(0)).view(np.uint32)
    assert enc == {1: ([0xFF001002, int(lo), int(hi)], np.float32(0)),
                   2: ([0xFF001105, 4, 1, 4], np.float32(0)),
                   4: ([0xFF001002, int(lo), int(hi)], np.float32(0)),
                   5: ([0xFF000000], np.float32(0))}
    inf = np.float32(np.inf).view(np.uint32)
    assert Range("y", gt=3).entries(7) == [0xFF001007, int(np.float32(3).view(np.uint32)) + 1, int(inf)]
    assert Range("y", lte=3).entries(0)[1] == int(np.float32(-np.inf).view(np.uint32))
    with pytest.raises(ValueError):                            # a code of the last bucket is fine, one past it not
        column_terms([In("lang", [7, 8])], None, lambda i, c: (5, 8))
    assert column_terms([In("lang", [7])], None, lambda i, c: (5, 8)) == {0: ([0xFF001105, 7], np.float32(0))}


def test_where_they_are_accepted_and_refused():
    from searcharray_b200 import And, Bool, Boost, DisMax, Field, In, Or, Range
    r, i = Range("year", gte=1990), In("lang", [0, 1])
    for c in (r, i):
        Or(["a", c]), And([c, "b"]), Bool(must=[c], should=[Boost(c, 2)], filter=[c], must_not=[c])
        Or([Bool(must=["a"], should=[Or([c, "b"])])])
        assert Field("t", c).clause is c
        for member in (c, Boost(c, 2), Field("t", c)):
            with pytest.raises(TypeError):
                DisMax(["a", member])
        with pytest.raises(ValueError):
            Bool(should=["a"], filter=[Boost(c, 2)])


def facet_arr():
    arr = arr_of(["a b", "b c", "c d", "d"])
    arr.set_feature("year", [1990, 0, 2001, 1977])
    arr.set_facet("lang", [0, 2, -1, 1], n_buckets=3)
    return arr


def test_search_topk_and_score_docs_refusals(no_device):
    from searcharray_b200 import Bool, In, Or, Range, bm25_impact
    from searcharray_b200.query import Field
    arr = facet_arr()
    r, i = Range("year", gte=1990), In("lang", [0, 2])
    docs = np.zeros((1, 2), dtype=np.uint32)
    for c in (r, i):
        with pytest.raises(TypeError, match="Bool"):           # a clause, not a query
            arr.search_topk([c])
        with pytest.raises(TypeError):
            arr.search_topk(["a", c], where=np.ones(4, dtype=bool))
        with pytest.raises(TypeError, match="Bool"):
            arr.score_docs([c], docs)
        with pytest.raises(NotImplementedError):               # views
            arr[np.asarray([True, True, False, True])].search_topk([Bool(must=["a"], filter=[c])])
        with pytest.raises(NotImplementedError):
            arr[np.asarray([True, True, False, True])].score_docs([Bool(must=["a"], filter=[c])], docs)
        with pytest.raises(TypeError):                         # non-BM25 similarities
            arr.search_topk([Bool(must=["a"], filter=[c])], similarity=bm25_impact())
        with pytest.raises(TypeError):
            arr.score_docs([Bool(must=["a"], filter=[c])], docs, similarity=bm25_impact())
        with pytest.raises(ValueError):                        # a Field clause in search_topk
            arr.search_topk([Or(["a", Field("t", c)])])
        with pytest.raises(DeviceTouched):
            arr.search_topk([Bool(must=["a"], filter=[c])])
        with pytest.raises(DeviceTouched):
            arr.score_docs([Bool(must=["a"], filter=[c])], docs)
    # names not set, on the kind of column each reads
    for c in (Range("lang", gte=1), Range("votes", lt=3), In("year", [0]), In("genre", [1])):
        with pytest.raises(ValueError):
            arr.search_topk([Bool(must=["a"], filter=[c])])
        with pytest.raises(ValueError):
            arr.search_topk([Bool(must=["a"], should=[Or(["b", c])])], facets=["lang"])
        with pytest.raises(ValueError):
            arr.score_docs([Bool(must=["a"], filter=[c])], docs)
    # a code past the facet's buckets (3)
    with pytest.raises(ValueError):
        arr.search_topk([Bool(must=["a"], filter=[In("lang", [1, 3])])])
    with pytest.raises(ValueError):
        arr.score_docs([Bool(must=["a"], filter=[In("lang", [3])])], docs)
    with pytest.raises(DeviceTouched):
        arr.search_topk([Bool(must=["a"], filter=[In("lang", [2])])])


def test_fields_topk_refusals(no_device):
    from searcharray_b200 import Bool, Field, In, Or, Range, SearchArray, fields_score_docs, fields_topk
    from searcharray_b200.postings import _PreparedBool
    from searcharray_b200.solr import _clause_slots, _fields_plan
    t = facet_arr()
    o = SearchArray.index(["x", "y", "x y", "z"])
    fr = pd.DataFrame({"t": t, "o": o})
    fr["t2"] = fr["t"]
    r, i = Range("year", gte=1990), In("lang", [0, 2])
    rows = np.zeros((1, 1), dtype=np.uint32)
    for c in (r, i):
        with pytest.raises(TypeError):
            fields_topk(fr, [c])
        with pytest.raises(TypeError):
            fields_topk(fr, [Field("t", c)])
        with pytest.raises(ValueError):                        # every clause names its column
            fields_topk(fr, [Bool(must=[Field("t", "a")], filter=[c])])
        with pytest.raises(ValueError):                        # not set on column o
            fields_topk(fr, [Bool(must=[Field("t", "a")], filter=[Field("o", c)])])
        with pytest.raises(ValueError):
            fields_score_docs(fr, [Bool(must=[Field("t", "a")], filter=[Field("o", c)])], rows)
        with pytest.raises(TypeError):                         # non-BM25 similarities
            from searcharray_b200 import bm25_impact
            fields_topk(fr, [Bool(must=[Field("t", "a")], filter=[Field("t", c)])], similarity=bm25_impact())
        with pytest.raises(NotImplementedError):               # views
            fv = pd.DataFrame({"t": t[np.asarray([True, True, False, True])]})
            fields_topk(fv, [Bool(must=[Field("t", "a")], filter=[Field("t", c)])])
        with pytest.raises(DeviceTouched):
            fields_topk(fr, [Bool(must=[Field("o", "x")], filter=[Field("t", c)])])
    with pytest.raises(ValueError):
        fields_topk(fr, [Bool(must=[Field("o", "x")], filter=[Field("t", In("lang", [5]))])])
    # columns that share an index share its columns: t2 is t's column
    q = Bool(must=[Field("o", "x")], filter=[Field("t2", r), Field("t", i)])
    batch, slot_of, arrays, sims = _fields_plan(fr, [q], {})
    assert slot_of["t"] == slot_of["t2"]
    enc = _PreparedBool.columns(batch.clauses, _clause_slots(batch, slot_of), arrays)
    assert enc == {1: (r.entries(0), np.float32(0)), 2: (i.entries(0), np.float32(0))}
    assert _PreparedBool.features(batch.clauses, _clause_slots(batch, slot_of), arrays) == {}
    assert Or([Field("t", r), Field("o", "x")]).form == 2
