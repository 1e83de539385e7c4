"""CPU: scoring at given documents (SearchArray.score_docs, solr.fields_score_docs) and window rescoring
(query.Rescore) -- every refusal, raised before any device work (the device entry points are replaced by a trap here),
and the host combine and order (query.rescore_window) against a brute-force np.lexsort."""
import numpy as np
import pandas as pd
import pytest

NO_DOC = 0xFFFFFFFF


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


@pytest.fixture
def arr():
    from searcharray_b200 import SearchArray
    return SearchArray.index(["foo bar", "bar baz", "foo foo", "qux"] * 5)


def test_score_docs_refusals(arr, no_device):
    from searcharray_b200 import Bool, Feature, Field, Or, bm25_impact, classic_similarity
    ok = np.zeros((2, 3), dtype=np.int64)
    with pytest.raises(TypeError):
        arr.score_docs(["foo", "bar"], ok.astype(np.float32))
    with pytest.raises(TypeError):
        arr.score_docs(["foo", "bar"], ok.astype(bool))
    for shape in [(3,), (1, 3), (3, 3), (2, 3, 1)]:
        with pytest.raises(ValueError, match="shape"):
            arr.score_docs(["foo", "bar"], np.zeros(shape, dtype=np.int64))
    for bad in (-1, 20, 21, NO_DOC - 1, NO_DOC + 1):
        d = ok.copy()
        d[1, 2] = bad
        with pytest.raises(ValueError, match=r"docs\[1, 2\]"):
            arr.score_docs(["foo", "bar"], d)
    with pytest.raises(TypeError):
        arr.score_docs(["foo"], ok[:1], similarity=bm25_impact)
    with pytest.raises(TypeError):
        arr.score_docs([Or(["foo", "bar"])], ok[:1], similarity=classic_similarity)
    with pytest.raises(NotImplementedError):
        arr[:10].score_docs(["foo"], ok[:1])
    with pytest.raises(TypeError):
        arr.score_docs([Feature("pop")], ok[:1])
    with pytest.raises(ValueError, match="Field"):
        arr.score_docs([Bool(should=[Field("t", "foo")])], ok[:1])


def test_score_docs_accepts_no_doc_and_empty(arr, no_device):
    """NO_DOC in any integer dtype that holds it, and an empty batch or window, need no device."""
    for dt in (np.uint32, np.int64, np.uint64):
        with pytest.raises(DeviceTouched):
            arr.score_docs(["foo"], np.asarray([[NO_DOC, 0, 19]], dtype=dt))
    assert arr.score_docs(["foo", "bar"], np.zeros((2, 0), dtype=np.int64)).shape == (2, 0)
    assert arr.score_docs([], np.zeros((0, 5), dtype=np.int64)).shape == (0, 5)


def test_fields_score_docs_refusals(arr, no_device):
    from searcharray_b200 import Bool, Field, Or, bm25_impact, fields_score_docs
    from searcharray_b200 import SearchArray
    frame = pd.DataFrame({"t": arr, "b": SearchArray.index(["x y"] * 20)})
    q = [Bool(should=[Field("t", "foo"), Field("b", "x")])]
    ok = np.zeros((1, 4), dtype=np.int32)
    with pytest.raises(TypeError):
        fields_score_docs(frame, q, ok.astype(np.float64))
    with pytest.raises(ValueError, match="shape"):
        fields_score_docs(frame, q, np.zeros((2, 4), dtype=np.int32))
    with pytest.raises(ValueError, match=r"docs\[0, 3\]"):
        fields_score_docs(frame, q, np.asarray([[0, 1, 2, 20]]))
    with pytest.raises(TypeError):
        fields_score_docs(frame, ["foo"], ok)
    with pytest.raises(ValueError, match="Field"):
        fields_score_docs(frame, [Or(["foo"])], ok)
    with pytest.raises(TypeError):
        fields_score_docs(frame, q, ok, similarity=bm25_impact)
    view = pd.DataFrame({"t": arr[:10], "b": frame["b"].array[:10]})
    with pytest.raises(NotImplementedError):
        fields_score_docs(view, q, np.zeros((1, 2), dtype=np.int32))


def test_rescore_refusals(arr, no_device):
    from searcharray_b200 import Bool, Field, Rescore, bm25_impact, fields_topk
    from searcharray_b200 import SearchArray
    for kw in [dict(query_weight=0), dict(query_weight=-1), dict(rescore_weight=-0.5), dict(query_weight=np.inf),
               dict(rescore_weight=np.nan), dict(rescore_weight=1e39), dict(query_weight=1e-50),
               dict(query_weight="1"), dict(window=10.0), dict(window=True)]:
        with pytest.raises(ValueError):
            Rescore(["foo"], **kw)
    r = Rescore(["foo", "bar"], window=8)
    with pytest.raises(ValueError, match="one per query"):
        arr.search_topk(["foo"], k=5, rescore=r)
    with pytest.raises(ValueError, match="window"):
        arr.search_topk(["foo", "bar"], k=9, rescore=r)
    with pytest.raises(ValueError, match="window"):
        arr.search_topk(["foo", "bar"], k=5, rescore=Rescore(["foo", "bar"], window=1025))
    with pytest.raises(ValueError):
        arr.search_topk(["foo", "bar"], k=0, rescore=r)
    with pytest.raises(TypeError):
        arr.search_topk(["foo", "bar"], k=5, rescore=["foo", "bar"])
    with pytest.raises(TypeError):
        arr.search_topk(["foo", "bar"], k=5, similarity=bm25_impact, rescore=r)
    with pytest.raises(NotImplementedError):
        arr[:10].search_topk(["foo", "bar"], k=5, rescore=r)
    frame = pd.DataFrame({"t": arr, "b": SearchArray.index(["x y"] * 20)})
    q = [Bool(should=[Field("t", "foo")])]
    with pytest.raises(ValueError, match="one per query"):
        fields_topk(frame, q, k=3, rescore=Rescore(q * 2, window=5))
    with pytest.raises(ValueError, match="window"):
        fields_topk(frame, q, k=6, rescore=Rescore(q, window=5))
    with pytest.raises(ValueError, match="Field"):
        fields_topk(frame, q, k=3, rescore=Rescore([Bool(should=["foo"])], window=5))
    with pytest.raises(TypeError):
        fields_topk(frame, q, k=3, similarity=bm25_impact, rescore=Rescore(q, window=5))


def brute(docs, s1, s2, qw, rw, k):
    """The combine and order restated: c in float32 per element, then np.lexsort by (id asc, c desc), empty last."""
    Q = docs.shape[0]
    out_d = np.full((Q, k), NO_DOC, dtype=np.uint32)
    out_c = np.zeros((Q, k), dtype=np.float32)
    for q in range(Q):
        live = docs[q] != NO_DOC
        d = docs[q][live]
        c = (np.float32(qw) * s1[q][live]).astype(np.float32) + (np.float32(rw) * s2[q][live]).astype(np.float32)
        order = np.lexsort((d.astype(np.int64), -c.astype(np.float64)))[:k]
        out_d[q, :len(order)] = d[order]
        out_c[q, :len(order)] = c[order]
    return out_d, out_c


@pytest.mark.parametrize("seed", range(6))
def test_rescore_window_against_lexsort(seed):
    from searcharray_b200.query import rescore_window
    rng = np.random.default_rng(seed)
    Q, W = 7, int(rng.integers(1, 60))
    k = int(rng.integers(1, W + 1))
    docs = np.full((Q, W), NO_DOC, dtype=np.uint32)
    s1 = np.zeros((Q, W), dtype=np.float32)
    s2 = np.zeros((Q, W), dtype=np.float32)
    for q in range(Q):
        n = int(rng.integers(0, W + 1))                              # pass 1 found n docs
        docs[q, :n] = rng.choice(10 ** 6, size=n, replace=False)
        # few distinct values: many ties in s1, s2 and c
        s1[q, :n] = np.sort(rng.choice(np.float32([0.5, 1.0, 1.25, 3.0]), size=n))[::-1]
        s2[q, :n] = rng.choice(np.float32([0.0, 0.25, 0.5, 2.0]), size=n)
    for qw, rw in [(1.0, 1.0), (1.0, 0.0), (0.3, 1.7), (2.0, 0.1)]:
        got_d, got_c = rescore_window(docs, s1, s2, qw, rw, k)
        want_d, want_c = brute(docs, s1, s2, qw, rw, k)
        assert np.array_equal(got_d, want_d)
        assert np.array_equal(got_c.view(np.uint32), want_c.view(np.uint32))
        assert got_d.dtype == np.uint32 and got_c.dtype == np.float32


def test_rescore_window_zero_weight_keeps_pass_one():
    """rescore_weight 0 and query_weight 1: the first k of pass 1, bit for bit."""
    from searcharray_b200.query import rescore_window
    docs = np.asarray([[4, 2, 9, NO_DOC], [1, 3, 7, 0]], dtype=np.uint32)
    s1 = np.asarray([[3.0, 2.0, 2.0, 0.0], [1.5, 1.5, 1.5, 1.0]], dtype=np.float32)
    s2 = np.asarray([[0.0, 9.0, 1.0, 0.0], [5.0, 0.0, 1.0, 2.0]], dtype=np.float32)
    d, c = rescore_window(docs, s1, s2, 1.0, 0.0, 3)
    assert np.array_equal(d, [[4, 2, 9], [1, 3, 7]]) and np.array_equal(c, s1[:, :3])
