"""CPU: facet columns (SearchArray.set_facet) and the `facets=` argument of search_topk / fields_topk -- every refusal,
raised before any device work (the device entry points are replaced by a trap here), and facets carried by copies,
pickles and shards; the constants mirrored from the C header."""
import os
import pickle
import re

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


DOCS = ["foo bar", "bar baz", "foo foo", "qux", "baz foo bar", "nothing here"]


def arr_of(docs=DOCS):
    from searcharray_b200 import SearchArray
    return SearchArray.index(docs)


def test_constants_match_the_header():
    from searcharray_b200 import query
    with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include",
                           "searcharray_b200.h")) as f:
        h = f.read()
    for name in ("SA_MAX_FACETS", "SA_FACET_MAX_BUCKETS", "SA_BOOL_MAX_FACETS"):
        assert int(re.search(rf"#define {name} (\d+)", h).group(1)) == getattr(query, name), name


def test_set_facet_and_defaults(no_device):
    arr = arr_of()
    arr.set_facet("cat", [0, 1, 2, -1, 1, 0])
    codes, nb = arr.host.facets["cat"]
    assert nb == 3 and codes.dtype == np.int32 and codes.tolist() == [0, 1, 2, -1, 1, 0]
    arr.set_facet("none", np.full(6, -1, dtype=np.int64))
    assert arr.host.facets["none"][1] == 1                   # at least one bucket
    arr.set_facet("cat", np.zeros(6, dtype=np.uint8), n_buckets=1024)   # replaced
    assert arr.host.facets["cat"][1] == 1024 and list(arr.host.facets) == ["cat", "none"]


def test_set_facet_refusals(no_device):
    arr = arr_of()
    for bad in (np.zeros(6, dtype=np.float32), ["a"] * 6, np.zeros(6, dtype=bool)):
        with pytest.raises(TypeError):
            arr.set_facet("x", bad)
    with pytest.raises(TypeError):
        arr.set_facet(3, [0] * 6)
    for codes, nb in (([0] * 5, None), ([0] * 7, None), ([0, 0, 0, 0, 0, -2], None), ([0, 1, 2, 3, 4, 5], 5),
                      ([0] * 6, 0), ([0] * 6, 1025), ([1024] * 6, None), (np.zeros((6, 1), dtype=int), None)):
        with pytest.raises(ValueError):
            arr.set_facet("x", codes, nb)
    assert arr.host.facets == {}
    for i in range(8):
        arr.set_facet(f"f{i}", [0] * 6)
    with pytest.raises(ValueError, match="at most 8"):
        arr.set_facet("f8", [0] * 6)
    arr.set_facet("f3", [1] * 6)                             # replacing a name is not a ninth
    with pytest.raises(ValueError, match="view"):
        arr[1:3].set_facet("y", [0, 0])


def test_copy_pickle_shard(no_device):
    arr = arr_of()
    arr.set_facet("cat", [0, 1, 2, -1, 1, 0])
    c = arr.copy()
    assert c.host.facets["cat"][0] is arr.host.facets["cat"][0]
    back = pickle.loads(pickle.dumps(arr))
    assert back.host.facets["cat"][0].tolist() == [0, 1, 2, -1, 1, 0] and back.host.facets["cat"][1] == 3
    sh = arr.host.shard(2, 5)
    assert sh.facets["cat"][0].tolist() == [2, -1, 1] and sh.facets["cat"][1] == 3
    # a pickle made before facets existed
    st = dict(arr.host.__dict__)
    del st["facets"]
    old = type(arr.host).__new__(type(arr.host))
    old.__setstate__(st)
    assert old.facets == {}


def test_search_topk_refusals(no_device):
    from searcharray_b200 import Bool, Feature, Field, Or, bm25_impact
    arr = arr_of()
    arr.set_facet("cat", [0, 1, 2, -1, 1, 0])
    arr.set_facet("b", [0, 0, 0, 0, 0, 0])
    qs = ["foo", Or(["foo", "bar"])]
    for bad in (["nope"], ["cat", "cat"], ["cat", "b", "cat"], ["cat", "b", "c", "d", "e"]):
        with pytest.raises(ValueError):
            arr.search_topk(qs, facets=bad)
    for bad in ("cat", ("cat",), 3):
        with pytest.raises(TypeError):
            arr.search_topk(qs, facets=bad)
    with pytest.raises(NotImplementedError):
        arr[1:4].search_topk(["foo"], facets=["cat"])
    with pytest.raises(NotImplementedError):
        arr[1:4].search_topk([Or(["foo"])], facets=[])
    with pytest.raises(TypeError):
        arr.search_topk(["foo"], similarity=bm25_impact(), facets=["cat"])
    with pytest.raises(TypeError):                            # the boolean path's own refusals stay
        arr.search_topk([Feature("pop")], facets=["cat"])
    with pytest.raises(ValueError):
        arr.search_topk([Bool(should=[Field("t", "foo")])], facets=["cat"])
    with pytest.raises(ValueError):                           # where= is checked as without facets
        arr.search_topk(qs, where=np.ones(5, dtype=bool), facets=["cat"])
    with pytest.raises(TypeError):
        arr.search_topk(qs, where=np.ones(6, dtype=int), facets=["cat"])
    with pytest.raises(DeviceTouched):                        # a good call reaches the device
        arr.search_topk(qs, facets=["cat", "b"])


def test_fields_topk_refusals(no_device):
    from searcharray_b200 import Field, Or, SearchArray, fields_topk
    frame = pd.DataFrame({"a": arr_of(), "b": arr_of(DOCS[::-1]), "c": SearchArray.index(DOCS + ["x"])[:6]})
    frame["a"].array.set_facet("cat", [0, 1, 2, -1, 1, 0])
    frame["b"].array.set_facet("cat", [0, 0, 0, 0, 0, 0])
    qs = [Or([Field("a", "foo"), Field("a", "bar")])]
    for bad in ([("a", "nope")], [("b", "other")], [("zz", "cat")], [("a", "cat"), ("a", "cat")],
                [("a", "cat")] * 5):
        with pytest.raises(ValueError):
            fields_topk(frame, qs, facets=bad)
    for bad in (["cat"], [("a",)], ("a", "cat"), [("a", 3)]):
        with pytest.raises(TypeError):
            fields_topk(frame, qs, facets=bad)
    with pytest.raises(NotImplementedError):                  # a sliced facet column: a view
        frame["c"].array.host.facets["cat"] = (np.zeros(7, dtype=np.int32), 1)
        fields_topk(frame, qs, facets=[("c", "cat")])
    with pytest.raises(DeviceTouched):
        fields_topk(frame, qs, facets=[("b", "cat"), ("a", "cat")])
