"""GPU: the batched top-k on views (SearchArray.search_topk on arr[key]).  For every query the result must be the
top k of view.score(q) -- positions in the view, score bits, order (score desc, position asc), empty slots
NO_DOC / 0 -- and, for slices, masks and stepped views, the top k of the CPU oracle's sliced index, so it is pinned
to the reference's semantics (FilteredPosns: df, tf and phrase counts of the filtered postings; the parent's
corpus size and avgdl; the stepped-slice doc_lens quirk).  The slice dfs of sa_docfreq_rows_batch are checked the
same way."""
import ctypes
import json
import os
import threading

import numpy as np
import pytest

from conftest import GOLDEN

pytestmark = pytest.mark.gpu

NO_DOC = 0xFFFFFFFF
N_DOCS = 200_000


def random_host(rng, n_docs, n_terms, max_df_frac):
    from searcharray_b200.indexing import index_from_term_postings
    from searcharray_b200.roaringish import encode_postings
    doc_lens = rng.integers(0, 300, n_docs).astype(np.float32)
    words = []
    for t in range(n_terms):
        df = max(1, int(n_docs * max_df_frac * rng.random() ** 3))
        docs = np.sort(rng.choice(n_docs, size=df, replace=False))
        tf = np.minimum(1 + rng.geometric(0.5, size=df), 40)
        d = np.repeat(docs, tf)
        p = np.concatenate([np.sort(rng.choice(700, size=k, replace=False)) for k in tf])
        words.append(encode_postings(d, p))
    return index_from_term_postings([f"t{i}" for i in range(n_terms)], words, doc_lens)


def expected_topk(dense, k):
    dense = np.asarray(dense, dtype=np.float32)
    nz = np.flatnonzero(dense > 0)
    order = nz[np.lexsort((nz, -dense[nz].astype(np.float64)))][:k]
    docs = np.full(k, NO_DOC, dtype=np.uint32)
    scores = np.zeros(k, dtype=np.float32)
    docs[:len(order)] = order
    scores[:len(order)] = dense[order]
    return docs, scores


def assert_topk(docs, scores, dense, what):
    wd, ws = expected_topk(dense, len(docs))
    assert np.array_equal(docs, wd), what
    assert np.array_equal(scores.view(np.uint32), ws.view(np.uint32)), what


@pytest.fixture(scope="module")
def corpus():
    from oracle import search as osearch
    from searcharray_b200 import SearchArray
    rng = np.random.default_rng(11)
    host = random_host(rng, N_DOCS, 12, 0.6)
    arr = SearchArray.from_host_index(host)
    oidx = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                               avg_doc_length=host.avg_doc_length)
    return host, arr, oidx


def view_keys():
    rng = np.random.default_rng(5)
    return {
        "range": slice(50_000, 150_000),
        "stepped": slice(1, None, 3),
        "mask": rng.random(N_DOCS) < 0.3,
        "fancy": rng.permutation(N_DOCS)[:20_000],
        "repeats": rng.integers(0, N_DOCS, 30_000),
        "view_of_view": (rng.random(N_DOCS) < 0.5, slice(1_000, 60_000)),
        "empty": slice(0, 0),
        "one": slice(7, 8),
    }


ORACLE_VIEWS = {"range", "stepped", "mask", "view_of_view", "empty", "one"}


def make_view(arr, key):
    if isinstance(key, tuple):
        return arr[key[0]][key[1]]
    return arr[key]


def make_oracle_view(oidx, key):
    if isinstance(key, tuple):
        return oidx.sliced(key[0]).sliced(key[1])
    return oidx.sliced(key)


@pytest.mark.parametrize("name", list(view_keys()))
def test_terms_on_views(corpus, name):
    host, arr, oidx = corpus
    key = view_keys()[name]
    view = make_view(arr, key)
    names = [f"t{t}" for t in range(host.n_terms)] + ["missing"]
    # (.score on a view without rows has nothing to return; its top k is empty)
    dense = {q: view.score(q) if len(view) else np.zeros(0, dtype=np.float32) for q in names}
    oview = make_oracle_view(oidx, key) if name in ORACLE_VIEWS else None
    for k in (1, 10, 32):
        docs, scores = view.search_topk(names, k=k)
        assert docs.shape == (len(names), k) and docs.dtype == np.uint32 and scores.dtype == np.float32
        assert np.all(docs[docs != NO_DOC] < len(view))
        for i, q in enumerate(names):
            assert_topk(docs[i], scores[i], dense[q], (name, q, k))
            if oview is not None:
                want = oview.score(None if q == "missing" else host.term_dict.get_term_id(q))
                wd, ws = expected_topk(want, k)
                assert np.array_equal(docs[i], wd), (name, q, k, "oracle")
                np.testing.assert_allclose(scores[i], ws, rtol=1e-5, atol=0)
    if name == "empty":
        assert len(view) == 0 and np.all(docs == NO_DOC) and np.all(scores == 0)


@pytest.mark.parametrize("name", list(view_keys()))
def test_slice_docfreqs(corpus, name):
    from searcharray_b200 import _lib
    host, arr, oidx = corpus
    key = view_keys()[name]
    view = make_view(arr, key)
    tids = np.asarray(list(range(host.n_terms)) + [_lib.NO_TERM], dtype=np.uint32)
    dfs = np.zeros(len(tids), dtype=np.uint64)
    dev = view._device()
    with view._shared["lock"]:
        view._apply_rows(dev)
        _lib.check(_lib.lib().sa_docfreq_rows_batch(dev.handle, _lib.p_u32(tids), len(tids), _lib.p_u64(dfs)))
    assert dfs[-1] == 0
    rows = np.unique(view.rows.astype(np.int64))
    oview = make_oracle_view(oidx, key) if name in ORACLE_VIEWS else None
    for t in range(host.n_terms):
        docs = np.unique((host.term_words(t) >> np.uint64(36)).astype(np.int64))
        assert int(dfs[t]) == int(np.isin(docs, rows).sum()), (name, t)
        assert int(dfs[t]) == int(view.docfreq(f"t{t}")), (name, t)
        if oview is not None:
            assert int(dfs[t]) == oview.docfreq(t), (name, t)


@pytest.fixture(scope="module")
def small_vocab():
    from searcharray_b200 import SearchArray
    rng = np.random.default_rng(3)
    vocab = [f"v{i}" for i in range(8)]
    docs = [" ".join(rng.choice(vocab, size=int(rng.integers(1, 60)))) for _ in range(3000)]
    return SearchArray.index(docs), rng


@pytest.mark.parametrize("slop", [0, 2])
def test_terms_and_phrases_mixed(small_vocab, slop):
    arr, rng = small_vocab
    queries = ["v0", ["v1", "v2"], ["v3", "v3"], ["v0", "v1", "v2"], "v5", ["v4", "v5", "v6", "v7"],
               ["v2", "nope"], "nope", ["v1", "v1", "v2"], ["v6", "v7"]]
    views = {"mask": arr[np.random.default_rng(9).random(3000) < 0.3],
             "fancy": arr[np.random.default_rng(10).permutation(3000)[:1200]],
             "stepped": arr[2::5]}
    for vname, view in views.items():
        dense = [view.score(q, slop=slop) for q in queries]
        assert any(np.any(d > 0) for d in dense[1:4])
        for k in (10, 32):
            docs, scores = view.search_topk(queries, k=k, slop=slop)
            for i, q in enumerate(queries):
                assert_topk(docs[i], scores[i], dense[i], (vname, q, slop, k))


@pytest.mark.parametrize("k1,b", [(0.0, 0.75), (1.2, 1.0), (1.2, 0.0), (1.2, 1.5)])
def test_exotic_bm25_parameters(corpus, k1, b):
    from searcharray_b200 import bm25_similarity
    host, arr, oidx = corpus
    sim = bm25_similarity(k1=k1, b=b)
    names = [f"t{t}" for t in range(host.n_terms)] + ["missing"]
    for key in (slice(50_000, 150_000), slice(1, None, 3)):
        view = arr[key]
        docs, scores = view.search_topk(names, k=10, similarity=sim)
        for i, q in enumerate(names):
            assert_topk(docs[i], scores[i], view.score(q, similarity=sim), (key, q, k1, b))


def test_ties_take_the_lowest_positions():
    from searcharray_b200 import SearchArray
    from searcharray_b200.indexing import index_from_term_postings
    from searcharray_b200.roaringish import encode_postings
    n = 120_000
    docs = np.arange(n)
    host = index_from_term_postings(["x", "y"], [encode_postings(docs, np.full(n, 3)),
                                                 encode_postings(docs[::2], np.full(n // 2, 5))],
                                    np.full(n, 10, dtype=np.float32))
    arr = SearchArray.from_host_index(host)
    for view in (arr[10_000:110_000], arr[np.arange(n) % 7 != 3][:100_000]):
        assert len(view) == 100_000
        docs_, scores = view.search_topk(["x", "y"], k=10)
        assert np.array_equal(docs_[0], np.arange(10, dtype=np.uint32))
        assert len(np.unique(scores[0])) == 1 and scores[0][0] > 0
        for i, q in enumerate(["x", "y"]):
            assert_topk(docs_[i], scores[i], view.score(q), q)


def test_candidate_overflow_is_rerun_exactly():
    """A view whose best scores all sit in the 32 positions of each of 31 threads of one tile, the next ones in
    single positions of 32 other threads: the tile bound cannot separate them, more docs than candidate slots
    reach it, and the query takes the exact re-run.  Its result, and the other query's, must still be exact."""
    from searcharray_b200 import SearchArray, _lib
    from searcharray_b200.indexing import index_from_term_postings
    from searcharray_b200.roaringish import encode_postings
    n = 10_000
    high = [4 * (t + 256 * j) + e for t in range(31) for j in range(8) for e in range(4)]
    low = [4 * t for t in range(31, 63)]
    special = high + low
    taken = set(special)
    rest = [p for p in range(8192) if p not in taken]
    perm = np.empty(8192, dtype=np.int64)
    perm[special] = np.arange(len(special))                  # docs 0..991 high, 992..1023 low
    perm[rest] = np.arange(len(special), 8192)
    z_docs = np.arange(len(special))
    z_tf = np.where(z_docs < len(high), 5, 1)
    d = np.repeat(z_docs, z_tf)
    p = np.concatenate([np.arange(t) for t in z_tf])
    w_docs = np.arange(0, n, 3)
    host = index_from_term_postings(["z", "w"], [encode_postings(d, p), encode_postings(w_docs, np.zeros(len(w_docs)))],
                                    np.full(n, 10, dtype=np.float32))
    arr = SearchArray.from_host_index(host)
    view = arr[perm]
    dev = arr._device()
    for k in (10, 32):
        st = _lib.SaStats()
        _lib.check(_lib.lib().sa_stats_reset(dev.handle))
        docs, scores = view.search_topk(["w", "z", "w"], k=k)
        _lib.check(_lib.lib().sa_stats_get(dev.handle, ctypes.byref(st)))
        # one tf scan, one view tile pass and one select for the batch, the same again for the re-run of "z"
        assert (st.term_kernel_launches, st.topk_kernel_launches) == (2, 4), k
        assert np.array_equal(docs[1], np.sort(np.asarray(high))[:k].astype(np.uint32))
        for i, q in enumerate(["w", "z", "w"]):
            assert_topk(docs[i], scores[i], view.score(q), (q, k))


def test_tmdb_overview_mask_view():
    from _tmdb_index import load_field
    from searcharray_b200 import SearchArray
    g = json.load(open(os.path.join(GOLDEN, "tmdb.json")))["fields"]["overview_tokens"]
    host = load_field(np.load(os.path.join(GOLDEN, "tmdb_index.npz")), "overview_tokens")
    arr = SearchArray.from_host_index(host)
    view = arr[np.random.default_rng(1).random(host.n_docs) < 0.4]
    queries = list(g["terms"]) + [r["phrase"] for r in g["phrases"]]
    docs, scores = view.search_topk(queries, k=10)
    for i, q in enumerate(queries):
        assert_topk(docs[i], scores[i], view.score(q), q)
    for slop in sorted({r["slop"] for r in g["slop"]}):
        slop_queries = [r["phrase"] for r in g["slop"] if r["slop"] == slop]
        docs, scores = view.search_topk(slop_queries, k=10, slop=slop)
        for i, q in enumerate(slop_queries):
            assert_topk(docs[i], scores[i], view.score(q, slop=slop), (q, slop))


def test_three_threads_on_views_of_one_array(corpus):
    host, arr, oidx = corpus
    names = [f"t{t}" for t in range(host.n_terms)]
    before = arr.search_topk(names, k=10)
    views = [arr[50_000:150_000], arr[np.random.default_rng(2).random(N_DOCS) < 0.3], arr[1::3]]
    serial = [v.search_topk(names, k=10) for v in views]
    results = [None] * 3

    def work(i):
        out = []
        for _ in range(4):
            d, s = views[i].search_topk(names, k=10)
            out.append(np.array_equal(d, serial[i][0]) and np.array_equal(s.view(np.uint32), serial[i][1].view(np.uint32)))
        results[i] = all(out)

    threads = [threading.Thread(target=work, args=(i,)) for i in range(3)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert results == [True, True, True]
    after = arr.search_topk(names, k=10)
    assert np.array_equal(after[0], before[0]) and np.array_equal(after[1].view(np.uint32), before[1].view(np.uint32))


def test_sharded_view_raises(corpus):
    from searcharray_b200 import SearchArray
    host, arr, oidx = corpus
    sharded = SearchArray.from_host_index(host, global_df=np.ones(host.n_terms, dtype=np.uint64))
    with pytest.raises(ValueError):
        sharded[10:20].search_topk(["t0"], k=5)


def test_2m_docs_ten_percent_mask():
    from searcharray_b200 import SearchArray, synth
    spec = synth.SynthSpec(2_000_000)
    host, _, _ = synth.generate_shard(spec)
    avgdl = synth.global_avg_doc_length(spec)
    host.avg_doc_length = avgdl
    arr = SearchArray.from_host_index(host, avg_doc_length=avgdl)
    view = arr[np.random.default_rng(4).random(host.n_docs) < 0.1]
    names = []
    n_buckets = len(synth.DF_BUCKETS)
    for bi in range(n_buckets):
        terms = spec.bucket_terms[bi]
        want = 64 // n_buckets + (1 if bi < 64 % n_buckets else 0)
        names.extend(terms[j] for j in np.linspace(0, len(terms) - 1, min(want, len(terms))).astype(int))
    assert len(names) >= 48
    docs, scores = view.search_topk(names, k=10)
    for i, q in enumerate(names):
        assert_topk(docs[i], scores[i], view.score(q), q)
