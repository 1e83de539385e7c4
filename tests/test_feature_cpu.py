"""CPU: feature clauses (query.Feature, SearchArray.set_feature) -- validation, every refusal (raised before any
device work: the device entry points are replaced by a trap here), the form and the flattened encoding (reserved term
ids, parameters in the idf slot), pickling of registered values, and the numpy transform against hand-computed
values."""
import pickle

import numpy as np
import pandas as pd
import pytest


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


def test_feature_validation():
    from searcharray_b200 import Feature
    f = Feature("pop")
    assert f.function == "linear" and f.param == 0 and f.fn == 0
    s = Feature("pop", "saturation", pivot=50)
    assert s.param == np.float32(50) and s.param.dtype == np.float32 and s.fn == 1
    lg = Feature("pop", "log", scaling_factor=1.5)
    assert lg.param == np.float32(1.5) and lg.fn == 2
    assert repr(s) == "Feature('pop', 'saturation', pivot=50.0)"
    for bad in (3, None, b"pop", ["pop"]):
        with pytest.raises(TypeError):
            Feature(bad)
    bad_args = [dict(function="sigmoid"), dict(function="linear", pivot=1.0), dict(function="linear", scaling_factor=1),
                dict(function="saturation"), dict(function="saturation", pivot=0), dict(function="saturation", pivot=-1),
                dict(function="saturation", pivot=float("nan")), dict(function="saturation", pivot=float("inf")),
                dict(function="saturation", pivot=1e39),             # inf in float32
                dict(function="saturation", pivot=1e-50),            # 0 in float32
                dict(function="saturation", pivot=1.0, scaling_factor=1.0),
                dict(function="log"), dict(function="log", scaling_factor=0.5),
                dict(function="log", scaling_factor=float("inf")), dict(function="log", pivot=1.0),
                dict(function="log", scaling_factor=2.0, pivot=1.0)]
    for kw in bad_args:
        with pytest.raises(ValueError):
            Feature("pop", **kw)


def test_transform_by_hand():
    from searcharray_b200 import Feature
    x = np.asarray([0, -0.0, 1, 3, 50, 1e-45, 2 ** 24 + 1], dtype=np.float64)
    got = Feature("p").apply(x)
    assert got.dtype == np.float32
    assert got.tolist() == [0, 0, 1, 3, 50, np.float32(1e-45), np.float32(2 ** 24)]
    assert not np.signbit(got[1])                             # -0.0 lacks the feature: +0
    sat = Feature("p", "saturation", pivot=1).apply([0, 1, 3, 1e-45])
    assert sat.tolist() == [0, 0.5, 0.75, np.float32(1e-45)]
    assert Feature("p", "saturation", pivot=1e30).apply([1e-45, 1e-8]).tolist() == [0, np.float32(1e-38)]   # underflow
    sat50 = Feature("p", "saturation", pivot=50).apply([50, 150])
    assert sat50.tolist() == [0.5, 0.75]
    lg = Feature("p", "log", scaling_factor=1).apply([0, 1, np.e - 1, 1e-45, 1e-9])
    assert lg[0] == 0 and lg[1] == np.float32(np.log(2.0)) and lg[2] == np.float32(1.0)
    assert lg[3] == 0                                          # log(1 + 1e-45) == 0 in double: no match
    # the sum is rounded to double before the log, as Lucene's log(scalingFactor + x) is: not log1p
    assert lg[4] == np.float32(np.log(1.0 + np.float64(np.float32(1e-9)))) != np.float32(np.log1p(np.float32(1e-9)))
    assert Feature("p", "log", scaling_factor=2).apply([2, 1e-30])[0:2].tolist() == [np.float32(np.log(4.0)),
                                                                                     np.float32(np.log(2.0))]


def test_where_features_are_accepted_and_refused():
    from searcharray_b200 import And, Bool, Boost, DisMax, Feature, Field, Or
    f = Feature("pop", "log", scaling_factor=1)
    Or(["a", f]), And([f, "b"]), Bool(must=[f], should=[Boost(f, 2)], filter=[f], must_not=[f])
    Or([Bool(must=["a"], should=[Or([f, "b"])])])
    assert Field("title", f).clause is f
    Or([Field("t", "a"), Boost(Field("t", f), 3)])
    for member in (f, Boost(f, 2), Field("t", f), Boost(Field("t", f), 2)):
        with pytest.raises(TypeError):
            DisMax(["a", member])
    for role in ("filter", "must_not"):
        with pytest.raises(ValueError):
            Bool(should=["a"], **{role: [Boost(f, 2)]})
        with pytest.raises(ValueError):
            Bool(should=["a"], **{role: [Boost(Field("t", f), 2)]})


def test_form_and_encoding():
    from searcharray_b200 import Bool, Boost, DisMax, Feature, Or
    from searcharray_b200.query import (DISMAX, NESTED, OCCUR, OR_AND, SA_NO_NODE, bool_form, feature_terms,
                                        flatten_bool, has_feature, needs_occur)
    sat = Feature("pop", "saturation", pivot=50)
    lin = Feature("votes")
    assert bool_form(Or(["a", "b"])) == OR_AND
    assert bool_form(Or(["a", lin])) == OCCUR and needs_occur(Or(["a", lin])) and has_feature(Or(["a", lin]))
    assert bool_form(Or([DisMax(["a", "b"]), sat])) == DISMAX
    assert bool_form(Or(["a", Or([lin, "b"])])) == NESTED and has_feature(Or(["a", Or([lin, "b"])]))
    assert not has_feature(Or(["a", "b"]))
    queries = [Bool(must=[Or(["star", "wars"])], should=[Boost(sat, 2.0)]), Or(["trek", lin])]
    batch = flatten_bool(queries, NESTED)
    assert batch.clauses[1] is sat and batch.clauses[2] == "trek" and batch.clauses[3] is lin
    assert batch.clause_node.tolist() == [2, SA_NO_NODE, SA_NO_NODE, SA_NO_NODE, SA_NO_NODE, SA_NO_NODE]
    assert batch.weights.tolist() == [1, 2, 1, 1, 1, 1] and batch.occurs.tolist() == [1, 0, 0, 0, 0, 0]
    slots = {"pop": 3, "votes": 0}
    enc = feature_terms(batch.clauses, lambda i, f: slots[f.name])
    assert enc == {1: (0xFF000000 | 1 << 8 | 3, np.float32(50)), 3: (0xFF000000, np.float32(0))}
    assert Feature("x", "log", scaling_factor=2).term_id(15) == 0xFF00020F


def test_set_feature_validation(no_device):
    from searcharray_b200 import SearchArray
    arr = arr_of(["a b", "b c", "c d", "d"])
    arr.set_feature("pop", [1, 0, 2.5, 3])
    assert arr.host.features["pop"].dtype == np.float32 and arr.host.features["pop"].tolist() == [1, 0, 2.5, 3]
    arr.set_feature("votes", np.arange(4, dtype=np.int64))
    arr.set_feature("pop", np.asarray([0, 0, 0, 7], dtype=np.float64))        # replaced, slot kept
    assert list(arr.host.features) == ["pop", "votes"] and arr._feature_slot("pop") == 0
    assert arr.host.features["pop"].tolist() == [0, 0, 0, 7] and arr._feature_slot("votes") == 1
    for bad in ([1, 2, 3], [1, 2, 3, 4, 5], [[1, 2, 3, 4]], [1, np.nan, 0, 0], [1, np.inf, 0, 0], [1, -1, 0, 0],
                [1e39, 0, 0, 0], [1, -1e-50, 0, 0]):
        with pytest.raises(ValueError):
            arr.set_feature("bad", bad)
    for bad in (["a", "b", "c", "d"], np.asarray([True, False, True, False]), [1 + 1j, 0, 0, 0]):
        with pytest.raises(TypeError):
            arr.set_feature("bad", bad)
    with pytest.raises(TypeError):
        arr.set_feature(3, [1, 2, 3, 4])
    assert "bad" not in arr.host.features
    with pytest.raises(ValueError):
        arr[np.asarray([True, False, True, True])].set_feature("x", [1, 2, 3])
    for i in range(14):
        arr.set_feature(f"f{i}", np.ones(4))
    with pytest.raises(ValueError):
        arr.set_feature("seventeenth", np.ones(4))
    arr.set_feature("f3", np.zeros(4))                         # replacing one of the 16 is fine
    # copies share the index and its features; pickles carry them
    c = arr.copy()
    assert c.host.features is arr.host.features
    back = pickle.loads(pickle.dumps(arr))
    assert isinstance(back, SearchArray) and list(back.host.features) == list(arr.host.features)
    for name, v in arr.host.features.items():
        assert back.host.features[name].dtype == np.float32 and np.array_equal(back.host.features[name], v)


def test_shard_slices_features():
    arr = arr_of(["a b", "b c", "c d", "d"])
    arr.set_feature("pop", [1, 2, 3, 4])
    assert arr.host.shard(1, 3).features["pop"].tolist() == [2, 3]


def test_search_topk_refusals(no_device):
    from searcharray_b200 import Bool, DisMax, Feature, Field, Or, bm25_impact
    arr = arr_of(["a b", "b c", "c d", "d"])
    arr.set_feature("pop", [1, 0, 2, 3])
    pop = Feature("pop", "saturation", pivot=2)
    with pytest.raises(TypeError):
        arr.search_topk([pop])
    with pytest.raises(TypeError):
        arr.search_topk(["a", pop], where=np.ones(4, dtype=bool))
    with pytest.raises(ValueError):                            # not set on this array
        arr.search_topk([Or(["a", Feature("votes")])])
    with pytest.raises(ValueError):
        arr.search_topk([Bool(must=["a"], should=[Or(["b", Feature("votes", "log", scaling_factor=1)])])])
    with pytest.raises(ValueError):                            # a Field clause in search_topk, as before
        arr.search_topk([Or(["a", Field("t", pop)])])
    with pytest.raises(NotImplementedError):                   # views, as before
        arr[np.asarray([True, True, False, True])].search_topk([Or(["a", pop])])
    with pytest.raises(TypeError):                             # non-BM25 similarities, as before
        arr.search_topk([Or(["a", pop])], similarity=bm25_impact())
    with pytest.raises(TypeError):
        DisMax([pop])
    # accepted queries reach the device (the trap) only after the checks
    with pytest.raises(DeviceTouched):
        arr.search_topk([Or(["a", pop])])


def test_fields_topk_refusals(no_device):
    from searcharray_b200 import Bool, Feature, Field, Or, SearchArray, fields_topk
    from searcharray_b200.query import ED_MAX_FIELDS
    from searcharray_b200.solr import _fields_plan
    t = SearchArray.index(["a b", "b c", "c d", "d"])
    o = SearchArray.index(["x", "y", "x y", "z"])
    t.set_feature("pop", [1, 0, 2, 3])
    fr = pd.DataFrame({"t": t, "o": o})
    fr["t2"] = fr["t"]
    pop = Feature("pop", "log", scaling_factor=1)
    with pytest.raises(TypeError):
        fields_topk(fr, [pop])
    with pytest.raises(TypeError):
        fields_topk(fr, [Field("t", pop)])
    with pytest.raises(ValueError):                            # every clause names its column
        fields_topk(fr, [Or([Field("t", "a"), pop])])
    with pytest.raises(ValueError):                            # not set on column o
        fields_topk(fr, [Bool(must=[Field("t", "a")], should=[Field("o", pop)])])
    # a feature column counts towards the field limit
    cols = {f"c{i}": SearchArray.index(["a", "b", "c", "d"]) for i in range(ED_MAX_FIELDS)}
    cols["c0"].set_feature("pop", [1, 2, 3, 4])
    big = pd.DataFrame(cols)
    big["extra"] = SearchArray.index(["a", "b", "c", "d"])
    big["extra"].array.set_feature("pop", [1, 2, 3, 4])
    qs = [Or([Field(f"c{i}", "a") for i in range(ED_MAX_FIELDS)] + [Field("extra", pop)])]
    with pytest.raises(ValueError):
        fields_topk(big, qs)
    # columns sharing an index share its features: t2 is t's column
    batch, slot_of, arrays, sims = _fields_plan(fr, [Bool(must=[Field("t", "a")], should=[Field("t2", pop)])], {})
    assert slot_of["t"] == slot_of["t2"]
    from searcharray_b200.postings import _PreparedBool
    from searcharray_b200.solr import _clause_slots
    assert _PreparedBool.features(batch.clauses, _clause_slots(batch, slot_of), arrays) == {
        1: (pop.term_id(0), np.float32(1))}
    with pytest.raises(DeviceTouched):
        fields_topk(fr, [Bool(must=[Field("t", "a")], should=[Field("t2", pop)])])
