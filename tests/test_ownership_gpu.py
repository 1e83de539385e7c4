"""GPU: every device buffer the library allocates has one owner that frees it.  sa_device_allocations counts the
process's live device buffers and bytes (cudaMemGetInfo would also see every other process on the device); each
test reads it before and after."""
import ctypes
import gc

import numpy as np
import pandas as pd
import pytest

from test_topk_rerun_gpu import phrase_overflow_array

pytestmark = pytest.mark.gpu

SA_ERR_ARG = 2


def live():
    from searcharray_b200 import _lib
    n, b = ctypes.c_uint64(), ctypes.c_uint64()
    _lib.check(_lib.lib().sa_device_allocations(ctypes.byref(n), ctypes.byref(b)))
    return n.value, b.value


def drop_multis():
    """Destroys every cached multi-field handle (solr._multis holds up to 16)."""
    from searcharray_b200 import solr
    with solr._multis_lock:
        multis = list(solr._multis.values())
        solr._multis.clear()
    for m in multis:
        m._finalizer()


def settled_baseline():
    """Frees what earlier tests left collectable, so that nothing but this test moves the count."""
    drop_multis()
    gc.collect()
    return live()


def corpus(n_docs, seed):
    rng = np.random.default_rng(seed)
    vocab = ["foo", "bar", "baz", "qux", "quux"]
    return [" ".join(rng.choice(vocab, rng.integers(1, 14))) for _ in range(n_docs)]


def test_lifecycle_returns_to_baseline():
    """Every entry point once on fresh arrays, then everything released: the count returns to where it started, in
    buffers and in bytes."""
    from searcharray_b200 import SearchArray, ops
    from searcharray_b200.solr import edismax, edismax_topk
    from searcharray_b200.similarity import bm25_impact, bm25_legacy_similarity, classic_similarity, default_bm25
    before = settled_baseline()
    docs = corpus(3000, 11)
    body = SearchArray.index(docs)
    title = SearchArray.index([d[:12] for d in docs])
    rerun, _ = phrase_overflow_array()                                  # its phrase takes the exact re-run
    built = SearchArray.index(docs[:300], gpu_build=True)
    arrays = [body, title, rerun, built]

    body.score("foo")
    body.termfreqs("bar")
    body.score(["foo", "bar"])
    body.score(["foo", "bar"], slop=2)
    body.score("baz", similarity=classic_similarity())               # sa_op_similarity
    built.score("qux")
    body.search_topk(["foo", ["foo", "bar"]], k=10)
    body.search_topk(["foo", ["bar", "baz"]], k=10, slop=2)
    for slop in (0, 2):
        rerun.search_topk([["a", "b"], "w"], k=10, slop=slop)
    view = body[np.arange(len(body)) % 3 == 1]
    for sim in (default_bm25, bm25_impact(), bm25_legacy_similarity(), classic_similarity()):
        view.search_topk(["foo", ["foo", "bar"]], k=5, similarity=sim)
    frame = pd.DataFrame({"body": body, "title": title})
    edismax(frame, "foo bar", qf=["body", "title"])
    edismax_topk(frame, "foo bar", qf=["body", "title"], k=5)            # sa_multi_topk
    arrays += [frame[c].array for c in frame.columns]

    lhs, rhs = body.host.term_words(body._term_id("foo")), body.host.term_words(body._term_id("bar"))
    ops.intersect(lhs, rhs)
    ops.bm25_score(np.ones(100, dtype=np.float32), np.full(100, 7.0, dtype=np.float32), 6.0, 1.5, 1.2, 0.75)
    ops.bigram_freqs(lhs, rhs)
    ops.popcount64_reduce(lhs)
    assert live()[0] > before[0]

    drop_multis()
    for a in arrays:
        if a._shared["dev"] is not None:
            a._shared["dev"].close()
    assert live() == before


def test_create_failing_after_upload_frees_it():
    """Term slices that do not tile `words` are rejected after the words reached the device: nothing stays."""
    from searcharray_b200 import _lib
    before = settled_baseline()
    words = (np.arange(8, dtype=np.uint64) << np.uint64(36)) | np.uint64(1)
    offs = np.array([0, 5], dtype=np.uint64)           # [4, 5) belongs to no term
    lens = np.array([4, 3], dtype=np.uint64)
    doc_lens = np.ones(8, dtype=np.float32)
    handle = ctypes.c_void_p()
    rc = _lib.lib().sa_index_create(_lib.p_u64(words), len(words), _lib.p_u64(offs), _lib.p_u64(lens), 2,
                                    _lib.p_f32(doc_lens), 8, 0, 0, ctypes.byref(handle))
    assert rc == SA_ERR_ARG
    assert b"tile" in _lib.lib().sa_last_error()
    assert not handle
    assert live() == before


def test_failed_set_rows_keeps_the_previous_view():
    """sa_index_set_rows with an out-of-range row fails and leaves the installed filter in place and usable."""
    from searcharray_b200 import SearchArray, _lib
    before = settled_baseline()
    arr = SearchArray.index(corpus(2000, 5))
    view = arr[np.arange(len(arr)) % 4 != 2]
    want_docs, want_scores = view.search_topk(["foo", ["bar", "baz"]], k=10)
    want_tf = view.termfreqs("qux")                        # installs the view's rows
    L, h = _lib.lib(), arr._device().handle
    bad = np.array([1, len(arr)], dtype=np.uint64)
    with arr._shared["lock"]:
        assert L.sa_index_set_rows(h, _lib.p_u64(bad), len(bad)) == SA_ERR_ARG
        tf = np.empty(len(view), dtype=np.float32)          # the installed filter, without re-installing it
        _lib.check(L.sa_termfreqs(h, arr._term_id("qux"), 0, _lib.ALL_BITS, _lib.p_f32(tf)))
    assert np.array_equal(tf.view(np.uint32), want_tf.view(np.uint32))
    docs, scores = view.search_topk(["foo", ["bar", "baz"]], k=10)
    assert np.array_equal(docs, want_docs)
    assert np.array_equal(np.asarray(scores).view(np.uint32), np.asarray(want_scores).view(np.uint32))
    arr._shared["dev"].close()
    assert live() == before
