"""CPU: the checks of search_topk's and fields_topk's `where=` mask that run before any device work -- dtype
(TypeError), shape (ValueError), the refusals of the unmasked call kept with a mask -- and the host packing
(postings.pack_where) against a restatement of the owner-order layout in include/searcharray_b200.h."""
import numpy as np
import pandas as pd
import pytest

N = 8192 * 2 + 37


@pytest.fixture(scope="module")
def arr():
    from searcharray_b200 import SearchArray
    rng = np.random.default_rng(0)
    return SearchArray.index([" ".join(rng.choice(["a", "b", "c", "d"], 5)) for _ in range(N)])


@pytest.mark.parametrize("bad", [np.ones(N, dtype=np.int64), np.ones(N, dtype=np.float32),
                                 np.array([True] * N, dtype=object), [1] * N])
def test_dtype_type_error(arr, bad):
    from searcharray_b200 import Or
    for queries in (["a"], [Or(["a", "b"])]):
        with pytest.raises(TypeError, match="boolean mask"):
            arr.search_topk(queries, k=5, where=bad)


@pytest.mark.parametrize("shape", [(N - 1,), (N + 1,), (0,), (3, N), (1, N), (2, N - 1), (2, N, 1), ()])
def test_shape_value_error(arr, shape):
    from searcharray_b200 import Or
    bad = np.ones(shape, dtype=bool)
    for queries in (["a", "b"], [Or(["a", "b"]), "c"]):
        with pytest.raises(ValueError, match="shape"):
            arr.search_topk(queries, k=5, where=bad)


def test_fields_topk_checks(arr):
    from searcharray_b200 import Field, Or, fields_topk
    frame = pd.DataFrame({"x": arr})
    q = [Or([Field("x", "a")])]
    with pytest.raises(TypeError, match="boolean mask"):
        fields_topk(frame, q, where=np.zeros(N, dtype=np.uint8))
    with pytest.raises(ValueError, match="shape"):
        fields_topk(frame, q, where=np.ones((2, N), dtype=bool))
    with pytest.raises(NotImplementedError):         # a sliced column is refused as without a mask
        fields_topk(frame[:100], q, where=np.ones(100, dtype=bool))


def test_refusals_kept(arr):
    """Inputs the unmasked call refuses are refused the same way with a valid mask."""
    from searcharray_b200 import Field, Or, bm25_impact
    view = arr[: N // 2]
    with pytest.raises(NotImplementedError):
        view.search_topk([Or(["a", "b"])], where=np.ones(len(view), dtype=bool))
    with pytest.raises(TypeError):
        arr.search_topk([Or(["a", "b"])], similarity=bm25_impact(), where=np.ones(N, dtype=bool))
    with pytest.raises(ValueError, match="Field"):
        arr.search_topk([Or([Field("x", "a")])], where=np.ones(N, dtype=bool))
    with pytest.raises(TypeError):
        arr.search_topk(["a"], similarity=lambda *a: None, where=np.ones(N, dtype=bool))


def test_packing_empty():
    from searcharray_b200.postings import pack_where
    assert pack_where(np.zeros(0, dtype=bool), 0, 2).shape == (1, 0)
    assert pack_where(np.zeros((2, 0), dtype=bool), 0, 2).shape == (2, 0)


@pytest.mark.parametrize("n", [1, 4, 8191, 8192, 8193, N])
def test_packing(n):
    """Bit 4 j + e of word t * 256 + i is doc t * 8192 + 4 (i + 256 j) + e; bits past n are 0; one row per query."""
    from searcharray_b200.postings import pack_where
    rng = np.random.default_rng(n)
    for rows in (1, 3):
        m = rng.random((rows, n)) < 0.5
        bits = pack_where(m if rows > 1 else m[0], n, rows)
        n_tiles = -(-n // 8192)
        assert bits.dtype == np.uint32 and bits.shape == (rows, n_tiles * 256) and bits.flags.c_contiguous
        want = np.zeros((rows, n_tiles * 256), dtype=np.uint64)
        for d in range(n):
            t, g, e = d // 8192, (d % 8192) // 4, d % 4
            i, j = g % 256, g // 256
            want[:, t * 256 + i] |= m[:, d].astype(np.uint64) << np.uint64(4 * j + e)
        assert np.array_equal(bits.astype(np.uint64), want)
    assert pack_where(pd.Series(m[0]), n, 3).shape == (1, n_tiles * 256)
