"""GPU: search_topk under bm25_impact, bm25_legacy_similarity and classic_similarity.  For every query the result
must be the top k of `.score(q, similarity=sim, slop=slop)` on the same array or view: ids, score BITS, the dtype
.score returns (float32 impact, float64 legacy / classic), order (score desc, id asc), only scores > 0 (+inf
included, NaN never), empty slots NO_DOC / 0.  For slices, masks and stepped views it must also be the top k of the
CPU oracle's composition (oracle/similarity.py on oracle.search counts and the slice's dfs), which pins the doc
lengths to the view's own ones (not the stepped-slice lengths BM25 uses)."""
import ctypes
import json
import os
import threading

import numpy as np
import pytest

from conftest import GOLDEN

pytestmark = pytest.mark.gpu

NO_DOC = 0xFFFFFFFF
N_DOCS = 120_000


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
    """The top k of a .score vector, in its own dtype: ids by (score desc, id asc) over the scores > 0."""
    dense = np.asarray(dense)
    nz = np.flatnonzero(dense > 0)
    order = nz[np.lexsort((nz, -dense[nz].astype(np.float64)))][:k]
    docs = np.full(k, NO_DOC, dtype=np.uint32)
    scores = np.zeros(k, dtype=dense.dtype)
    docs[:len(order)] = order
    scores[:len(order)] = dense[order]
    return docs, scores


def bits(a):
    return a.view(np.uint64 if a.dtype == np.float64 else np.uint32)


def assert_topk(docs, scores, dense, what):
    wd, ws = expected_topk(dense, len(docs))
    assert scores.dtype == ws.dtype, what
    assert np.array_equal(docs, wd), what
    assert np.array_equal(bits(scores), bits(ws)), what


def sims():
    from searcharray_b200 import bm25_impact, bm25_legacy_similarity, classic_similarity
    return {
        "impact": bm25_impact(),
        "impact_k1_0": bm25_impact(k1=0.0),          # NaN at tf == 0
        "impact_b_1": bm25_impact(b=1.0),
        "impact_neg_k1": bm25_impact(k1=-0.5),        # negative and +inf scores
        "legacy": bm25_legacy_similarity(),
        "legacy_k1_0": bm25_legacy_similarity(k1=0.0, b=1.0),
        "legacy_neg_k1": bm25_legacy_similarity(k1=-1.5, b=0.3),
        "classic": classic_similarity(),
    }


def oracle_sim(sim):
    from oracle import similarity as osim
    from searcharray_b200.similarity import Bm25Impact, Bm25Legacy
    if isinstance(sim, Bm25Impact):
        return lambda *a: osim.bm25_impact(*a, k1=sim.k1, b=sim.b)
    if isinstance(sim, Bm25Legacy):
        return lambda *a: osim.bm25_legacy(*a, k1=sim.k1, b=sim.b)
    return osim.classic


@pytest.fixture(scope="module")
def corpus():
    from oracle import search as osearch
    from searcharray_b200 import SearchArray
    rng = np.random.default_rng(21)
    host = random_host(rng, N_DOCS, 10, 0.6)
    arr = SearchArray.from_host_index(host)
    oidx = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                               avg_doc_length=host.avg_doc_length)
    return host, arr, oidx


def view_keys():
    rng = np.random.default_rng(5)
    return {
        "unsliced": None,
        "range": slice(30_000, 90_000),
        "stepped": slice(1, None, 3),
        "mask": rng.random(N_DOCS) < 0.3,
        "fancy": rng.permutation(N_DOCS)[:20_000],
        "repeats": rng.integers(0, N_DOCS, 30_000),
        "view_of_view": (rng.random(N_DOCS) < 0.5, slice(1_000, 40_000)),
        "empty": slice(0, 0),
        "one": slice(7, 8),
    }


ORACLE_VIEWS = {"range", "stepped", "mask"}


def make_view(arr, key):
    if key is None:
        return arr
    if isinstance(key, tuple):
        return arr[key[0]][key[1]]
    return arr[key]


def dense_score(view, q, sim, slop=0):
    if len(view) == 0:
        return np.zeros(0, dtype=sim.out_dtype)
    return view.score(q, similarity=sim, slop=slop)


@pytest.mark.parametrize("sim_name", list(sims()))
@pytest.mark.parametrize("name", list(view_keys()))
def test_terms_on_arrays_and_views(corpus, name, sim_name):
    host, arr, oidx = corpus
    sim = sims()[sim_name]
    key = view_keys()[name]
    view = make_view(arr, key)
    names = [f"t{t}" for t in range(host.n_terms)] + ["missing"]
    dense = {q: dense_score(view, q, sim) for q in names}
    oview = oidx.sliced(key) if name in ORACLE_VIEWS else None
    for k in (1, 10, 32):
        docs, scores = view.search_topk(names, k=k, similarity=sim)
        assert docs.shape == (len(names), k) and docs.dtype == np.uint32 and scores.dtype == sim.out_dtype
        assert np.all(docs[docs != NO_DOC] < len(view))
        for i, q in enumerate(names):
            assert_topk(docs[i], scores[i], dense[q], (name, sim_name, q, k))
            if oview is not None and q != "missing":
                tid = host.term_dict.get_term_id(q)
                want = oracle_sim(sim)(oview.termfreqs(tid), [oview.docfreq(tid)], oview.doc_lens,
                                       oview.avg_doc_length, oview.corpus_size)
                wd, ws = expected_topk(want, k)
                assert np.array_equal(docs[i], wd), (name, sim_name, q, k, "oracle")
                assert np.array_equal(bits(scores[i]), bits(ws.astype(sim.out_dtype))), (name, sim_name, q, k, "oracle")
    if name == "empty":
        assert np.all(docs == NO_DOC) and np.all(scores == 0)


def test_stepped_view_uses_its_own_doc_lengths(corpus):
    """BM25 on arr[a::s] reads the parent's consecutive doc lengths (a reference quirk); the other similarities
    receive .doclengths(), the view's own.  Both search_topk paths follow their .score."""
    from searcharray_b200 import bm25_similarity, classic_similarity
    host, arr, oidx = corpus
    view = arr[1::3]
    assert not np.array_equal(view._view_bm25_doc_lens(), view.doclengths())
    for sim in (classic_similarity(), bm25_similarity()):
        docs, scores = view.search_topk(["t0", "t3"], k=32, similarity=sim)
        for i, q in enumerate(["t0", "t3"]):
            assert_topk(docs[i], scores[i], view.score(q, similarity=sim), (sim, q))
    # the classic ranking with the parent's consecutive lengths would differ
    tf = view.termfreqs("t0")
    wrong = classic_similarity()(tf, [view.docfreq("t0")], view._view_bm25_doc_lens(), view.avg_doc_length,
                                 view.corpus_size)
    docs, _ = view.search_topk(["t0"], k=32, similarity=classic_similarity())
    assert not np.array_equal(docs[0], expected_topk(wrong, 32)[0])


@pytest.fixture(scope="module")
def small_vocab():
    from searcharray_b200 import SearchArray
    rng = np.random.default_rng(3)
    vocab = [f"v{i}" for i in range(8)]
    docs = [" ".join(rng.choice(vocab, size=int(rng.integers(1, 60)))) for _ in range(3000)]
    return SearchArray.index(docs)


@pytest.mark.parametrize("slop", [0, 2])
@pytest.mark.parametrize("sim_name", ["impact", "legacy", "classic", "legacy_neg_k1"])
def test_terms_and_phrases_mixed(small_vocab, slop, sim_name):
    arr = small_vocab
    sim = sims()[sim_name]
    queries = ["v0", ["v1", "v2"], ["v3", "v3"], ["v0", "v1", "v2"], "v5", ["v4", "v5", "v6", "v7"],
               ["v2", "nope"], "nope", ["v1", "v1", "v2"], ["v6", "v7"]]
    views = {"unsliced": arr, "mask": arr[np.random.default_rng(9).random(3000) < 0.3],
             "fancy": arr[np.random.default_rng(10).permutation(3000)[:1200]], "stepped": arr[2::5]}
    for vname, view in views.items():
        dense = [view.score(q, similarity=sim, slop=slop) for q in queries]
        assert any(np.any(d > 0) for d in dense[1:4])
        for k in (1, 10, 32):
            docs, scores = view.search_topk(queries, k=k, similarity=sim, slop=slop)
            for i, q in enumerate(queries):
                assert_topk(docs[i], scores[i], dense[i], (vname, sim_name, q, slop, k))


def _array(postings, doc_lens, **kw):
    from searcharray_b200 import SearchArray
    from searcharray_b200.indexing import index_from_term_postings
    from searcharray_b200.roaringish import encode_postings
    names = list(postings)
    words = []
    for t in names:
        docs, tfs = postings[t]
        d = np.repeat(np.asarray(docs), tfs)
        p = np.concatenate([np.arange(f) for f in tfs]) if len(tfs) else np.zeros(0, dtype=np.int64)
        words.append(encode_postings(d, p))
    host = index_from_term_postings(names, words, np.asarray(doc_lens, dtype=np.float32))
    return SearchArray.from_host_index(host, **kw)


def test_classic_near_ties_break_a_float32_proxy():
    """(tf, dl) = (1, d), (4, 4d), (9, 9d) score idf / sqrt(d) up to the float64 roundings: their float32 proxies
    tie, their float64 scores may not.  Spread over many docs and tiles, with more tied docs than k."""
    from searcharray_b200 import classic_similarity
    n = 40_000
    rng = np.random.default_rng(8)
    docs = np.sort(rng.choice(n, 3_000, replace=False))
    tfs = np.asarray([1, 4, 9, 16, 25])[rng.integers(0, 5, len(docs))]
    base = rng.integers(1, 200, len(docs))
    dl = np.full(n, 1000.0)
    dl[docs] = base * tfs
    arr = _array({"a": (docs, tfs), "b": (docs[::2], np.ones(len(docs[::2]), dtype=np.int64))}, dl)
    sim = classic_similarity()
    dense = arr.score("a", similarity=sim)
    top = dense[dense > 0]
    assert len(np.unique(top)) > len(np.unique(top.astype(np.float32)))    # the proxy really ties distinct scores
    for view in (arr, arr[np.arange(n) % 5 != 1], arr[5:]):
        for k in (1, 10, 32):
            docs_, scores = view.search_topk(["a", "b"], k=k, similarity=sim)
            for i, q in enumerate(["a", "b"]):
                assert_topk(docs_[i], scores[i], view.score(q, similarity=sim), (q, k))


def test_legacy_one_ulp_apart_and_exact_ties():
    """Doc lengths chosen so that neighbouring sats are one float32 ulp apart, each shared by many docs (exact
    ties): the legacy key must rank them exactly, ties by position."""
    from oracle.similarity import _saturation_denominator
    from searcharray_b200 import bm25_impact, bm25_legacy_similarity
    f32 = np.float32
    cand = f32(50) + np.arange(4000, dtype=np.float32) * np.spacing(f32(50))
    sat = (f32(3) * f32(1.2 + 1)) / _saturation_denominator(f32(3), cand, 50.0, 1.2, 0.75)
    u, first = np.unique(sat, return_index=True)
    adj = np.flatnonzero(np.nextafter(u[:-1], f32(np.inf)) == u[1:])[:3]
    assert len(adj) == 3
    chosen = cand[first[np.concatenate([adj, adj + 1])]]
    n = 30_000
    docs = np.arange(0, n, 7)
    dl = np.full(n, 50.0, dtype=np.float32)
    dl[docs] = chosen[np.arange(len(docs)) % len(chosen)]
    arr = _array({"x": (docs, np.full(len(docs), 3))}, dl, avg_doc_length=50.0)
    for sim in (bm25_legacy_similarity(), bm25_impact()):
        dense = arr.score("x", similarity=sim)
        assert len(np.unique(dense[dense > 0])) >= 3
        for view in (arr, arr[100:]):
            for k in (1, 10, 32):
                d, s = view.search_topk(["x"], k=k, similarity=sim)
                assert_topk(d[0], s[0], view.score("x", similarity=sim), (sim, k))


def test_classic_inf_and_avgdl_zero():
    from searcharray_b200 import bm25_impact, bm25_legacy_similarity, classic_similarity
    n = 20_000
    docs = np.arange(0, n, 3)
    dl = np.full(n, 20.0)
    dl[docs[5:40]] = 0.0                 # count > 0, doc length 0: classic scores +inf
    arr = _array({"x": (docs, np.full(len(docs), 2))}, dl)
    sim = classic_similarity()
    dense = arr.score("x", similarity=sim)
    assert np.isinf(dense).sum() == 35
    for view in (arr, arr[2:]):
        for k in (10, 32):
            d, s = view.search_topk(["x"], k=k, similarity=sim)
            assert np.all(np.isinf(s[0])) and s[0][0] > 0
            assert_topk(d[0], s[0], view.score("x", similarity=sim), k)
    # avg_doc_length == 0: impact and legacy score zeros, classic still ranks
    zero = _array({"x": (docs, np.full(len(docs), 2))}, np.zeros(n))
    assert zero.avg_doc_length == 0
    for sim in (bm25_impact(), bm25_legacy_similarity(), classic_similarity()):
        for view in (zero, zero[::2]):
            d, s = view.search_topk(["x"], k=10, similarity=sim)
            # .score returns the reference's np.zeros_like(tf) there (float32); search_topk keeps the similarity's
            # dtype
            assert_topk(d[0], s[0], view.score("x", similarity=sim).astype(sim.out_dtype), sim)
            assert (d[0][0] == NO_DOC) == (not isinstance(sim, type(classic_similarity())))


@pytest.mark.parametrize("sim_name", ["impact", "legacy", "classic"])
def test_candidate_overflow_is_rerun_exactly(sim_name):
    """The best scores all sit in the 32 positions of each of 31 threads of one tile, the next ones in single
    positions of 32 other threads: more docs than candidate slots reach the tile bound and the query takes the
    exact re-run (as in the BM25 view test).  Its result, and the other query's, must still be exact."""
    from searcharray_b200 import _lib
    sim = sims()[sim_name]
    n = 10_000
    high = [4 * (t + 256 * j) + e for t in range(31) for j in range(8) for e in range(4)]
    low = [4 * t for t in range(31, 63)]
    special = high + low
    taken = set(special)
    rest = [p for p in range(8192) if p not in taken]
    perm = np.empty(8192, dtype=np.int64)
    perm[special] = np.arange(len(special))
    perm[rest] = np.arange(len(special), 8192)
    z_docs = np.arange(len(special))
    z_tf = np.where(z_docs < len(high), 5, 1)
    w_docs = np.arange(0, n, 3)
    arr = _array({"z": (z_docs, z_tf), "w": (w_docs, np.ones(len(w_docs), dtype=np.int64))}, np.full(n, 10.0))
    dev = arr._device()
    for view in (arr[perm], arr[np.concatenate([perm, np.arange(8192, n)])]):
        for k in (10, 32):
            st = _lib.SaStats()
            _lib.check(_lib.lib().sa_stats_reset(dev.handle))
            docs, scores = view.search_topk(["w", "z", "w"], k=k, similarity=sim)
            _lib.check(_lib.lib().sa_stats_get(dev.handle, ctypes.byref(st)))
            # one tf scan, one tile pass and one select for the batch, the same again for the re-run of "z"; classic
            # keeps every tie at a tile's bound, so the thousands of exactly tied "w" docs per tile re-run too
            reruns = 3 if sim_name == "classic" else 1
            assert (st.term_kernel_launches, st.topk_kernel_launches) == (1 + reruns, 2 + 2 * reruns), (sim_name, k)
            assert np.array_equal(docs[1], np.sort(np.asarray(high))[:k].astype(np.uint32))
            for i, q in enumerate(["w", "z", "w"]):
                assert_topk(docs[i], scores[i], view.score(q, similarity=sim), (q, k))


@pytest.mark.parametrize("sim_name", ["impact", "legacy", "classic"])
def test_tmdb_overview(sim_name):
    from _tmdb_index import load_field
    from searcharray_b200 import SearchArray
    sim = sims()[sim_name]
    g = json.load(open(os.path.join(GOLDEN, "tmdb.json")))["fields"]["overview_tokens"]
    host = load_field(np.load(os.path.join(GOLDEN, "tmdb_index.npz")), "overview_tokens")
    arr = SearchArray.from_host_index(host)
    queries = list(g["terms"])[:8] + [r["phrase"] for r in g["phrases"]][:4]
    slop_rows = [r for r in g["slop"]][:4]
    for view in (arr, arr[np.random.default_rng(1).random(host.n_docs) < 0.4]):
        docs, scores = view.search_topk(queries, k=10, similarity=sim)
        for i, q in enumerate(queries):
            assert_topk(docs[i], scores[i], view.score(q, similarity=sim), q)
        for r in slop_rows:
            docs, scores = view.search_topk([r["phrase"]], k=10, similarity=sim, slop=r["slop"])
            assert_topk(docs[0], scores[0], view.score(r["phrase"], similarity=sim, slop=r["slop"]), r)


def test_three_threads_different_similarities(corpus):
    host, arr, oidx = corpus
    names = [f"t{t}" for t in range(host.n_terms)]
    s = sims()
    jobs = [(arr[30_000:90_000], s["impact"]), (arr[np.random.default_rng(2).random(N_DOCS) < 0.3], s["legacy"]),
            (arr[1::3], s["classic"])]
    serial = [v.search_topk(names, k=10, similarity=sim) for v, sim in jobs]
    results = [None] * 3

    def work(i):
        v, sim = jobs[i]
        ok = True
        for _ in range(4):
            d, sc = v.search_topk(names, k=10, similarity=sim)
            ok = ok and np.array_equal(d, serial[i][0]) and np.array_equal(bits(sc), bits(serial[i][1]))
        results[i] = ok

    threads = [threading.Thread(target=work, args=(i,)) for i in range(3)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert results == [True, True, True]


def test_doc_base_and_global_df(corpus):
    from searcharray_b200 import SearchArray
    host, arr, oidx = corpus
    gdf = np.asarray([int(arr.docfreq(f"t{t}")) * 3 + 5 for t in range(host.n_terms)], dtype=np.uint64)
    shard = SearchArray.from_host_index(host, doc_base=1_000_000, corpus_size=4 * N_DOCS, global_df=gdf)
    names = [f"t{t}" for t in range(host.n_terms)] + [["t1", "t2"]]
    for sim_name in ("impact", "legacy", "classic"):
        sim = sims()[sim_name]
        docs, scores = shard.search_topk(names, k=10, similarity=sim)
        for i, q in enumerate(names):
            wd, ws = expected_topk(shard.score(q, similarity=sim), 10)
            wd = np.where(wd == NO_DOC, wd, wd + np.uint32(1_000_000))
            assert np.array_equal(docs[i], wd), (sim_name, q)
            assert np.array_equal(bits(scores[i]), bits(ws)), (sim_name, q)


def test_api_boundaries(corpus):
    from searcharray_b200 import SearchArray, bm25_similarity, classic_similarity
    host, arr, oidx = corpus
    sharded = SearchArray.from_host_index(host, global_df=np.ones(host.n_terms, dtype=np.uint64))
    with pytest.raises(ValueError):
        sharded[10:20].search_topk(["t0"], k=5, similarity=classic_similarity())
    with pytest.raises(TypeError, match="classic_similarity"):
        arr.search_topk(["t0"], k=5, similarity=lambda tf, df, dl, avgdl, n: tf)
    names = [f"t{t}" for t in range(host.n_terms)]
    for view in (arr, arr[30_000:90_000]):
        a = view.search_topk(names, k=10, similarity=bm25_similarity())
        b = view.search_topk(names, k=10)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))
        assert a[1].dtype == np.float32


def test_2m_docs_unsliced_and_ten_percent_mask():
    from searcharray_b200 import SearchArray, synth
    spec = synth.SynthSpec(2_000_000)
    host, _, _ = synth.generate_shard(spec)
    avgdl = synth.global_avg_doc_length(spec)
    host.avg_doc_length = avgdl
    arr = SearchArray.from_host_index(host, avg_doc_length=avgdl)
    names = []
    n_buckets = len(synth.DF_BUCKETS)
    for bi in range(n_buckets):
        terms = spec.bucket_terms[bi]
        want = 256 // n_buckets + (1 if bi < 256 % n_buckets else 0)
        names.extend(terms[j] for j in np.linspace(0, len(terms) - 1, min(want, len(terms))).astype(int))
    assert len(names) >= 128
    mask = arr[np.random.default_rng(4).random(host.n_docs) < 0.1]
    for sim_name in ("impact", "legacy", "classic"):
        sim = sims()[sim_name]
        for view in (arr, mask):
            docs, scores = view.search_topk(names, k=10, similarity=sim)
            for i, q in enumerate(names):
                assert_topk(docs[i], scores[i], view.score(q, similarity=sim), (sim_name, q))
