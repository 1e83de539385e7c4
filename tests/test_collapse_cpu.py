"""CPU: group columns (SearchArray.set_group) and the `collapse=` argument of search_topk / fields_topk -- every
refusal, raised before any device work (the device entry points are replaced by a trap here), group columns carried by
copies, pickles and shards, and collapse_ref, the numpy statement of the collapse contract the GPU tests compare
against, on hand-built vectors."""
import os
import pickle
import re

import numpy as np
import pandas as pd
import pytest

NO_DOC = 0xFFFFFFFF


def collapse_ref(S, codes, k):
    """The collapsed top k of the dense vector S under group codes (-1: no group): of the docs with S > 0, each
    group's leader is its doc with the highest S, ties to the lower id, and a doc with code -1 is a group of its own;
    the k best leaders by (S desc, id asc) as (docs uint32[k], scores float32[k]), NO_DOC / 0 past the last one."""
    S = np.asarray(S, dtype=np.float32)
    codes = np.asarray(codes)
    ranked = np.flatnonzero(S > 0)
    order = ranked[np.lexsort((ranked, -S[ranked].astype(np.float64)))]
    c = codes[order]
    grouped = c != -1
    first = np.zeros(int(grouped.sum()), dtype=bool)
    first[np.unique(c[grouped], return_index=True)[1]] = True
    lead = np.ones(len(order), dtype=bool)
    lead[grouped] = first
    top = order[lead][:k]
    docs = np.full(k, NO_DOC, dtype=np.uint32)
    scores = np.zeros(k, dtype=np.float32)
    docs[:len(top)] = top
    scores[:len(top)] = S[top]
    return docs, scores


def test_collapse_ref_hand_built():
    S = np.asarray([0.0, 2.0, 3.0, 3.0, 1.0, 3.0, 0.5, 2.0], dtype=np.float32)
    codes = np.asarray([7, 1, 2, 1, 2, 5, -1, -1])
    # 3.0 ties across groups 2, 1 and 5 go by id; group 2's 1.0 and group 1's 2.0 are not leaders; -1 docs each stand
    d, s = collapse_ref(S, codes, 8)
    assert d.tolist() == [2, 3, 5, 7, 6] + [NO_DOC] * 3
    assert s.tolist() == [3.0, 3.0, 3.0, 2.0, 0.5, 0.0, 0.0, 0.0]
    assert collapse_ref(S, codes, 1)[0].tolist() == [2]
    d2, s2 = collapse_ref(S, codes, 3)                    # a prefix of the deeper result
    assert d2.tolist() == d[:3].tolist() and s2.tolist() == s[:3].tolist()
    # all -1, or all distinct: the plain top k
    plain = np.lexsort((np.arange(8), -S.astype(np.float64)))[:7]
    assert collapse_ref(S, np.full(8, -1), 7)[0].tolist() == plain.tolist()
    assert collapse_ref(S, np.arange(8), 7)[0].tolist() == plain.tolist()
    # fewer groups than k: one group holds every ranked doc
    d, s = collapse_ref(S, np.zeros(8, dtype=int), 4)
    assert d.tolist() == [2, NO_DOC, NO_DOC, NO_DOC] and s.tolist() == [3.0, 0.0, 0.0, 0.0]
    # nothing ranks (0, negative and NaN never do)
    d, s = collapse_ref(np.asarray([0, -1, np.nan], dtype=np.float32), [0, 1, 2], 2)
    assert d.tolist() == [NO_DOC, NO_DOC] and s.tolist() == [0.0, 0.0]


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
    assert int(re.search(r"#define SA_MAX_GROUPS (\d+)", h).group(1)) == query.SA_MAX_GROUPS
    assert re.search(r"#define SA_GROUP_NONE 0xFFFFFFFFu", h)


def test_set_group(no_device):
    arr = arr_of()
    arr.set_group("g", [0, 1, 2, -1, 1, 2 ** 31 - 2])
    codes = arr.host.groups["g"]
    assert codes.dtype == np.int32 and codes.tolist() == [0, 1, 2, -1, 1, 2 ** 31 - 2]
    arr.set_group("g", np.zeros(6, dtype=np.uint8))           # replaced
    assert arr.host.groups["g"].tolist() == [0] * 6 and list(arr.host.groups) == ["g"]


def test_set_group_refusals(no_device):
    arr = arr_of()
    for bad in (np.zeros(6, dtype=np.float32), ["a"] * 6, np.zeros(6, dtype=bool)):
        with pytest.raises(TypeError):
            arr.set_group("x", bad)
    with pytest.raises(TypeError):
        arr.set_group(3, [0] * 6)
    for codes in ([0] * 5, [0] * 7, [0, 0, 0, 0, 0, -2], [0, 0, 0, 0, 0, 2 ** 31 - 1], [2 ** 40] * 6,
                  np.zeros((6, 1), dtype=int)):
        with pytest.raises(ValueError):
            arr.set_group("x", codes)
    assert arr.host.groups == {}
    for i in range(4):
        arr.set_group(f"g{i}", [0] * 6)
    with pytest.raises(ValueError, match="at most 4"):
        arr.set_group("g4", [0] * 6)
    arr.set_group("g2", [1] * 6)                              # replacing a name is not a fifth
    with pytest.raises(ValueError, match="view"):
        arr[1:3].set_group("y", [0, 0])


def test_copy_pickle_shard(no_device):
    arr = arr_of()
    arr.set_group("g", [0, 1, 2, -1, 1, 0])
    c = arr.copy()
    assert c.host.groups["g"] is arr.host.groups["g"]
    back = pickle.loads(pickle.dumps(arr))
    assert back.host.groups["g"].tolist() == [0, 1, 2, -1, 1, 0]
    sh = arr.host.shard(2, 5)
    assert sh.groups["g"].tolist() == [2, -1, 1]
    st = dict(arr.host.__dict__)                              # a pickle made before group columns existed
    del st["groups"]
    old = type(arr.host).__new__(type(arr.host))
    old.__setstate__(st)
    assert old.groups == {}


def test_search_topk_refusals(no_device):
    from searcharray_b200 import Bool, Feature, Field, Or, Rescore, bm25_impact
    arr = arr_of()
    arr.set_group("g", [0, 1, 2, -1, 1, 0])
    arr.set_facet("cat", [0, 1, 2, -1, 1, 0])
    qs = ["foo", Or(["foo", "bar"])]
    for bad in (3, ("g",), ["g"]):
        with pytest.raises(TypeError):
            arr.search_topk(qs, collapse=bad)
    with pytest.raises(ValueError, match="not set"):
        arr.search_topk(qs, collapse="nope")
    with pytest.raises(NotImplementedError):
        arr[1:4].search_topk(["foo"], collapse="g")
    with pytest.raises(TypeError):
        arr.search_topk(["foo"], similarity=bm25_impact(), collapse="g")
    with pytest.raises(ValueError, match="rescore"):
        arr.search_topk(qs, k=2, collapse="g", rescore=Rescore(qs, window=4))
    with pytest.raises(TypeError):                            # the boolean path's own refusals stay
        arr.search_topk([Feature("pop")], collapse="g")
    with pytest.raises(ValueError):
        arr.search_topk([Bool(should=[Field("t", "foo")])], collapse="g")
    with pytest.raises(ValueError):
        arr.search_topk(qs, k=0, collapse="g")
    with pytest.raises(ValueError):                           # where= and facets= are checked as without collapse
        arr.search_topk(qs, where=np.ones(5, dtype=bool), collapse="g")
    with pytest.raises(ValueError):
        arr.search_topk(qs, facets=["nope"], collapse="g")
    for ok in (dict(), dict(facets=["cat"], where=np.ones(6, dtype=bool))):
        with pytest.raises(DeviceTouched):                    # a good call reaches the device
            arr.search_topk(qs, collapse="g", **ok)


def test_fields_topk_refusals(no_device):
    from searcharray_b200 import Field, Or, Rescore, SearchArray, fields_topk
    frame = pd.DataFrame({"a": arr_of(), "b": arr_of(DOCS[::-1]), "c": SearchArray.index(DOCS + ["x"])[:6]})
    frame["a"].array.set_group("g", [0, 1, 2, -1, 1, 0])
    frame["b"].array.set_group("h", [0, 0, 0, 0, 0, 0])
    qs = [Or([Field("a", "foo"), Field("a", "bar")])]
    for bad in (("a", "nope"), ("b", "g"), ("zz", "g")):
        with pytest.raises(ValueError):
            fields_topk(frame, qs, collapse=bad)
    for bad in ("g", ("a",), ["a", "g"], ("a", 3)):
        with pytest.raises(TypeError):
            fields_topk(frame, qs, collapse=bad)
    with pytest.raises(ValueError, match="rescore"):
        fields_topk(frame, qs, k=2, collapse=("a", "g"), rescore=Rescore(qs, window=4))
    with pytest.raises(NotImplementedError):                  # a sliced group column: a view
        frame["c"].array.host.groups["g"] = np.zeros(7, dtype=np.int32)
        fields_topk(frame, qs, collapse=("c", "g"))
    with pytest.raises(DeviceTouched):
        fields_topk(frame, qs, collapse=("b", "h"))
