"""GPU: the exact top-k paths that rank a score row already in HBM -- edismax_topk, and the BM25 batch's re-run of
phrase and span queries -- on inputs that force their candidate overflow re-run or that a float32 key cannot order.
Every result must equal the top k of the dense score vector: ids by (score desc, id asc) over the scores > 0, score
bits included, empty slots NO_DOC / 0."""
import ctypes

import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu

NO_DOC = 0xFFFFFFFF
TILE = 8192


def host_index(postings, doc_lens, doc_base=0):
    """postings: term -> (local docs, per-doc positions).  The words carry ABSOLUTE doc ids (local + doc_base), as
    the shards synth.generate_shard builds."""
    from searcharray_b200.indexing import index_from_term_postings
    from searcharray_b200.roaringish import encode_postings
    words = []
    for docs, posns in postings.values():
        d = np.repeat(np.asarray(docs, dtype=np.int64) + doc_base, [len(p) for p in posns])
        p = np.concatenate(posns) if len(posns) else np.zeros(0, dtype=np.int64)
        words.append(encode_postings(d, p))
    return index_from_term_postings(list(postings), words, np.asarray(doc_lens, dtype=np.float32))


def expected_topk(dense, k, doc_base=0):
    dense = np.asarray(dense)
    nz = np.flatnonzero(dense > 0)
    order = nz[np.lexsort((nz, -dense[nz].astype(np.float64)))][:k]
    docs = np.full(k, NO_DOC, dtype=np.uint32)
    scores = np.zeros(k, dtype=dense.dtype)
    docs[:len(order)] = order + doc_base
    scores[:len(order)] = dense[order]
    return docs, scores


def f32_toward_zero(x):
    """float64 > 0 -> float32 rounded toward zero (the edismax tiles' ranking key)."""
    f = x.astype(np.float32)
    return np.where(f.astype(np.float64) > x, np.nextafter(f, np.float32(0)), f)


def topk_launches(arr, fn):
    from searcharray_b200 import _lib
    h = arr._device().handle
    st = _lib.SaStats()
    _lib.check(_lib.lib().sa_stats_reset(h))
    out = fn()
    _lib.check(_lib.lib().sa_stats_get(h, ctypes.byref(st)))
    return out, st.topk_kernel_launches


def test_edismax_ties_over_tiles_of_a_shard():
    """A shard (doc_base != 0) of five tiles: every doc scores, 300 docs in each of tiles 1-3 tie at the second best
    score and two docs of tile 4 score best.  Tiles 0-3 hold more tied candidates than slots, so the query takes the
    re-run with a slot per doc (two tile passes and two selects); ids come back absolute."""
    from searcharray_b200 import SearchArray
    from searcharray_b200.solr import edismax, edismax_topk
    base, n = 1_000_000, 4 * TILE + 500
    tf = np.ones(n, dtype=np.int64)
    for tile in (1, 2, 3):
        tf[tile * TILE + 37 + 11 * np.arange(300)] = 2
    tf[[4 * TILE + 3, 4 * TILE + 400]] = 3
    host = host_index({"foo": (np.arange(n), [np.arange(c) for c in tf])}, np.full(n, 6.0), doc_base=base)
    arr = SearchArray.from_host_index(host, doc_base=base)
    frame = pd.DataFrame({"t": arr})
    dense, _ = edismax(frame, "foo", qf=["t"])
    assert np.count_nonzero(dense == np.sort(dense)[-3]) == 900
    for k in (1, 10, 32):
        (docs, scores), launches = topk_launches(frame["t"].array, lambda: edismax_topk(frame, "foo", qf=["t"], k=k))
        assert launches == 4, k
        wd, ws = expected_topk(dense, k, base)
        assert np.array_equal(docs, wd), k
        assert np.array_equal(scores.view(np.uint64), ws.view(np.uint64)), k


def test_edismax_tie_breaker_scores_that_share_a_float32_key():
    """Term-centric edismax with tie > 0 over two fields whose doc lengths differ by steps of 1e-5: the top scores
    are float64 sums of close float32 field scores, and some distinct ones round to the same float32.  The ranking
    must follow the float64 scores."""
    from searcharray_b200 import SearchArray
    from searcharray_b200.solr import edismax, edismax_topk
    rng = np.random.default_rng(17)
    n = 3 * TILE + 100
    cols = {}
    for field in ("a", "b"):
        post = {}
        for term in ("x", "y"):
            docs = np.sort(rng.choice(n, n // 2, replace=False))
            post[term] = (docs, [np.zeros(1, dtype=np.int64)] * len(docs))
        dl = 20.0 + rng.integers(0, 4000, n) * 1e-5
        cols[field] = SearchArray.from_host_index(host_index(post, dl))
    frame = pd.DataFrame(cols)
    kw = dict(q="x y", qf=["a", "b^1.5"], tie=0.3)
    dense, _ = edismax(frame, **kw)
    assert dense.dtype == np.float64
    top = np.sort(dense[dense > 0])[::-1][:32]
    assert len(np.unique(top)) > len(np.unique(f32_toward_zero(top)))
    for k in (1, 10, 32):
        docs, scores = edismax_topk(frame, k=k, **kw)
        wd, ws = expected_topk(dense, k)
        assert np.array_equal(docs, wd), k
        assert np.array_equal(scores.view(np.uint64), ws.view(np.uint64)), k


def phrase_overflow_array():
    """The thread layout of test_sim_topk_gpu's overflow test: 992 docs held by 31 threads of tile 0 tie at the best
    score of the phrase ["a", "b"] (slop 0 or 2), 32 docs of 32 other threads score less.  Returns the array and the
    number of tied docs."""
    from searcharray_b200 import SearchArray
    n = 10_000
    high = [4 * (t + 256 * j) + e for t in range(31) for j in range(8) for e in range(4)]
    low = [4 * t for t in range(31, 63)]
    ab = np.sort(high + low)
    reps = np.where(np.isin(ab, high), 5, 1)
    w_docs = np.arange(0, n, 3)
    host = host_index({"a": (ab, [2 * np.arange(r) for r in reps]),
                       "b": (ab, [2 * np.arange(r) + 1 for r in reps]),
                       "w": (w_docs, [np.zeros(1, dtype=np.int64)] * len(w_docs))}, np.full(n, 10.0))
    return SearchArray.from_host_index(host), len(high)


@pytest.mark.parametrize("slop", [0, 2])
def test_batch_phrase_rerun_scores_the_counts(slop):
    """The thread layout of test_sim_topk_gpu's overflow test on the unsliced BM25 batch: 992 docs held by 31
    threads of tile 0 tie at the best phrase score, 32 docs of 32 other threads score less.  More tied docs than
    candidate slots reach the tile bound, so the phrase (slop 0) or span (slop 2) query takes the re-run, which
    scores the raw counts in the tile pass.  Docs and score bits must be the top k of .score, also when the same
    upload runs a second time."""
    from searcharray_b200 import _lib
    from searcharray_b200.similarity import compute_idf, default_bm25
    arr, n_high = phrase_overflow_array()
    queries = [["a", "b"], "w"]
    terms, starts, idfs = arr._topk_queries(queries, lambda dfs: compute_idf(arr.corpus_size, dfs))
    idfs = np.asarray(idfs, dtype=np.float32)
    dense = [arr.score(q, slop=slop) for q in queries]
    assert np.count_nonzero(dense[0] == dense[0].max()) == n_high
    L, h = _lib.lib(), arr._device().handle
    for k in (10, 32):
        with arr._shared["lock"]:
            _lib.check(L.sa_batch_upload(h, _lib.p_u32(terms), _lib.p_u32(starts), _lib.p_f32(idfs), len(queries),
                                         slop, arr.avg_doc_length, default_bm25.k1, default_bm25.b, k))
            for run in range(2):
                docs = np.empty((len(queries), k), dtype=np.uint32)
                scores = np.empty((len(queries), k), dtype=np.float32)
                n_over = ctypes.c_uint32(0)
                _lib.check(L.sa_batch_execute(h))
                _lib.check(L.sa_batch_download(h, _lib.p_u32(docs), _lib.p_f32(scores), ctypes.byref(n_over)))
                if run == 0:
                    assert n_over.value >= 1, (slop, k)
                for i in range(len(queries)):
                    wd, ws = expected_topk(dense[i], k)
                    assert np.array_equal(docs[i], wd), (slop, k, i, run)
                    assert np.array_equal(scores[i].view(np.uint32), ws.view(np.uint32)), (slop, k, i, run)
