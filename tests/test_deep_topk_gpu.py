"""GPU: batched top-k deeper than 32 (k up to 1,024; the deep tile collector, sa_term.cuh deep_tile_collect).  For
every query form the result must be the top k of the dense scores the same call ranks -- .score (which the other
suites pin to the CPU oracle bit for bit), or the boolean composition of clause scores -- by (score desc, id asc)
over the scores > 0, score bits exact, empty slots NO_DOC / 0; the first k' results of a k = 1,024 call must be those
of the k' call (the k <= 32 collector); and the deep_tiles counter must show which collector ran."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NO_DOC = 0xFFFFFFFF
TILE = 8192
KS = (33, 64, 100, 257, 1000, 1024)


def expected_topk(dense, k):
    dense = np.asarray(dense)
    nz = np.flatnonzero(dense > 0)
    order = nz[np.lexsort((nz, -dense[nz].astype(np.float64)))][:k]
    docs = np.full(k, NO_DOC, dtype=np.uint32)
    scores = np.zeros(k, dtype=dense.dtype)
    docs[:len(order)] = order
    scores[:len(order)] = dense[order]
    return docs, scores


def assert_topk(docs, scores, dense, what):
    wd, ws = expected_topk(dense, len(docs))
    assert np.array_equal(docs, wd), what
    assert np.array_equal(np.asarray(scores, dtype=ws.dtype).view(np.uint8), ws.view(np.uint8)), what


def stats(arr):
    from searcharray_b200 import _lib
    st = _lib.SaStats()
    _lib.check(_lib.lib().sa_stats_get(arr._device().handle, ctypes.byref(st)))
    return st


def reset(arr):
    from searcharray_b200 import _lib
    _lib.check(_lib.lib().sa_stats_reset(arr._device().handle))


def random_corpus(rng, n_docs, vocab, mean_len=12):
    lens = rng.integers(1, 2 * mean_len, n_docs)
    # Zipf-like term draw: a few dense terms, many sparse ones
    p = 1.0 / np.arange(1, vocab + 1) ** 1.1
    p /= p.sum()
    words = rng.choice(vocab, size=int(lens.sum()), p=p)
    out, i = [], 0
    for n in lens:
        out.append(" ".join(f"w{w}" for w in words[i:i + n]))
        i += n
    return out


@pytest.fixture(scope="module")
def corpus():
    from searcharray_b200 import SearchArray
    rng = np.random.default_rng(7)
    docs = random_corpus(rng, 3 * TILE + 1234, 400)        # n_docs not a multiple of the tile
    return SearchArray.index(docs)


TERMS = ["w0", "w1", "w5", "w30", "w120", "w399", "nope"]
PHRASES = [["w0", "w1"], ["w1", "w0", "w2"], ["w3", "w3"]]


def oracle_dense(arr, terms):
    """The CPU oracle's BM25 rows of single terms over the whole array (an index independent of the device)."""
    from oracle import search as osearch
    host = arr.host
    oidx = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                               avg_doc_length=host.avg_doc_length)
    tid = host.term_dict.term_to_ids
    return [np.asarray(oidx.score(tid.get(q)), dtype=np.float32) if q in tid else np.zeros(len(arr), np.float32)
            for q in terms]


def check_queries(arr, queries, dense, ks=KS, what="", **kw):
    for k in ks:
        reset(arr)
        docs, scores = arr.search_topk(queries, k=k, **kw)[:2]
        assert docs.shape == (len(queries), k)
        assert stats(arr).deep_tiles > 0, (what, k)
        for i, q in enumerate(queries):
            assert_topk(docs[i], scores[i], dense[i], (what, q, k))


def check_prefix(arr, queries, what="", **kw):
    deep_d, deep_s = arr.search_topk(queries, k=1024, **kw)[:2]
    for kp in (1, 10, 32):
        reset(arr)
        d, s = arr.search_topk(queries, k=kp, **kw)[:2]
        assert stats(arr).deep_tiles == 0, (what, kp)
        assert np.array_equal(d, deep_d[:, :kp]), (what, kp)
        assert np.array_equal(np.asarray(s).view(np.uint8), np.asarray(deep_s[:, :kp]).view(np.uint8)), (what, kp)


KNOBS = {
    "default": {},
    "always": {"SA_STAGED_NORM_MIN_RECS": "1", "SA_STAGED_NORM_MIN_WORDS": "1", "SA_TERM_QUAD_MIN_RECS": "1"},
    "never": {"SA_STAGED_NORM_MIN_RECS": str(2 ** 31), "SA_STAGED_NORM_MIN_WORDS": str(2 ** 31),
              "SA_TERM_QUAD_MIN_RECS": str(2 ** 31)},
    "prefetch0": {"SA_TERM_PREFETCH_TILES": "0"},
    "prefetch1": {"SA_TERM_PREFETCH_TILES": "1"},
}


@pytest.mark.parametrize("setting", list(KNOBS))
def test_terms_under_every_knob(corpus, monkeypatch, setting):
    for var in ("SA_STAGED_NORM_MIN_RECS", "SA_STAGED_NORM_MIN_WORDS", "SA_TERM_QUAD_MIN_RECS", "SA_TERM_PREFETCH_TILES"):
        monkeypatch.delenv(var, raising=False)
    for var, val in KNOBS[setting].items():
        monkeypatch.setenv(var, val)
    dense = oracle_dense(corpus, TERMS) if setting == "default" else [corpus.score(q) for q in TERMS]
    check_queries(corpus, TERMS, dense, what=setting)
    check_prefix(corpus, TERMS, what=setting)


def test_terms_words_path_in_a_child_process():
    """SA_NO_TF_TABLE=1 and SA_TERM_QUERY_MAJOR=1 are read once per process: the words path (windows(), staged norms
    on word tiles) of the deep term kernel runs in tests/_deep_topk_worker.py under every knob setting."""
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, SA_NO_TF_TABLE="1", SA_TERM_QUERY_MAJOR="1")
    out = subprocess.run([sys.executable, os.path.join(here, "_deep_topk_worker.py")], env=env, capture_output=True,
                         text=True, timeout=1200)
    assert out.returncode == 0 and out.stdout.strip().endswith("OK"), (out.stdout[-3000:] + out.stderr[-3000:])


@pytest.mark.parametrize("k1,b", [(0.0, 0.75), (1.2, 1.0), (1.2, 1.5)])
def test_terms_exotic_parameters(corpus, k1, b):
    from searcharray_b200 import bm25_similarity
    sim = bm25_similarity(k1=k1, b=b)
    dense = [corpus.score(q, similarity=sim) for q in TERMS]
    check_queries(corpus, TERMS, dense, ks=(33, 1000), what=(k1, b), similarity=sim)


@pytest.mark.parametrize("slop", [0, 2])
def test_phrases(corpus, slop):
    queries = PHRASES + ["w0"]
    dense = [corpus.score(q, slop=slop) for q in queries]
    assert all(np.any(d > 0) for d in dense)
    check_queries(corpus, queries, dense, what=slop, slop=slop)
    check_prefix(corpus, queries, what=slop, slop=slop)


def test_boolean_forms(corpus):
    from searcharray_b200 import And, Bool, DisMax, Or
    s = {t: corpus.score(t) for t in ("w0", "w1", "w2", "w5", "w30")}
    f32 = np.float32
    queries = [Or(["w1", "w5"]), And(["w0", "w2"]), Bool(must=["w0"], should=["w5", "w30"]),
               Or([And(["w1", "w2"]), "w30"]), DisMax(["w1", "w2"], tie=0.0)]
    dense = [
        (s["w1"] + s["w5"]).astype(f32),
        np.where((s["w0"] > 0) & (s["w2"] > 0), s["w0"] + s["w2"], f32(0)).astype(f32),
        np.where(s["w0"] > 0, (f32(1) * s["w0"]) + (f32(1) * s["w5"]) + (f32(1) * s["w30"]), f32(0)).astype(f32),
        (np.where((s["w1"] > 0) & (s["w2"] > 0), s["w1"] + s["w2"], f32(0)) + s["w30"]).astype(f32),
        np.maximum(s["w1"], s["w2"]).astype(f32),
    ]
    check_queries(corpus, queries, dense, what="bool")
    check_prefix(corpus, queries, what="bool")
    mask = np.random.default_rng(3).random(len(corpus)) < 0.4
    check_queries(corpus, queries, [np.where(mask, d, f32(0)) for d in dense], ks=(100, 1024), what="where",
                  where=mask)
    check_queries(corpus, TERMS, [np.where(mask, corpus.score(q), f32(0)) for q in TERMS], ks=(100, 1024),
                  what="where terms", where=mask)


def test_facet_hits_match_k10(corpus):
    from searcharray_b200 import Or
    codes = (np.arange(len(corpus)) % 5).astype(np.int32)
    corpus.set_facet("mod5", codes)
    queries = [Or(["w1", "w5"]), "w0", "w120"]
    d10, s10, h10 = corpus.search_topk(queries, k=10, facets=["mod5"])
    d, s, h = corpus.search_topk(queries, k=1000, facets=["mod5"])
    assert np.array_equal(h.total, h10.total)
    assert np.array_equal(h.facets["mod5"], h10.facets["mod5"])
    assert np.array_equal(d[:, :10], d10)


@pytest.mark.parametrize("view", ["mask", "stepped", "take"])
def test_views_and_similarities(corpus, view):
    from searcharray_b200 import bm25_impact, bm25_legacy_similarity, bm25_similarity
    rng = np.random.default_rng(4)
    v = {"mask": lambda a: a[rng.random(len(a)) < 0.5], "stepped": lambda a: a[1::3],
         "take": lambda a: a.take(rng.permutation(len(a))[:20000])}[view](corpus)
    for sim in (bm25_similarity(), bm25_impact(), bm25_legacy_similarity()):
        queries = TERMS + PHRASES
        dense = [v.score(q, similarity=sim) for q in queries]
        check_queries(v, queries, dense, ks=(33, 257, 1024), what=(view, type(sim).__name__), similarity=sim)
        check_prefix(v, queries, what=(view, type(sim).__name__), similarity=sim)
    for sim in (bm25_impact(), bm25_legacy_similarity()):
        dense = [corpus.score(q, similarity=sim) for q in TERMS]
        check_queries(corpus, TERMS, dense, ks=(64, 1000), what=type(sim).__name__, similarity=sim)


def test_fields_topk(corpus):
    import pandas as pd
    from searcharray_b200 import Field, Or, fields_topk
    from searcharray_b200 import SearchArray
    rng = np.random.default_rng(8)
    n = 20000
    frame = pd.DataFrame({"a": SearchArray.index(random_corpus(rng, n, 200)),
                          "b": SearchArray.index(random_corpus(rng, n, 200, mean_len=5))})
    queries = [Or([Field("a", "w1"), Field("b", "w1")]), Or([Field("a", "w7"), Field("b", "w3")])]
    dense = [(frame["a"].array.score("w1") + frame["b"].array.score("w1")).astype(np.float32),
             (frame["a"].array.score("w7") + frame["b"].array.score("w3")).astype(np.float32)]
    for k in (33, 1000):
        docs, scores = fields_topk(frame, queries, k=k)
        for i in range(len(queries)):
            assert_topk(docs[i], scores[i], dense[i], ("fields", i, k))
    d1024, s1024 = fields_topk(frame, queries, k=1024)
    for kp in (1, 10, 32):
        d, s = fields_topk(frame, queries, k=kp)
        assert np.array_equal(d1024[:, :kp], d) and np.array_equal(s1024[:, :kp].view(np.uint32), s.view(np.uint32))


# --------------------------------------------------------------------------------------------- tile shapes
def test_tile_shapes():
    """Tiles with fewer than, exactly and more than k ranked docs; one tile holding the whole top k (a clustered
    corpus); thousands of docs tied at the bound in one tile; an index of fewer than k docs."""
    from searcharray_b200 import SearchArray
    k = 100
    docs = []
    for t in range(4):
        n_hit = {0: 50, 1: 100, 2: 3000, 3: 0}[t]
        docs += ["x filler"] * (TILE - n_hit) + ["x hit"] * n_hit
    docs += ["hit hit hit short"] * 300 + ["filler"] * 77            # the last tile holds the best docs
    arr = SearchArray.index(docs)
    for q in ("hit", "x", "filler"):
        dense = arr.score(q)
        for kk in (k, 1024):
            d, s = arr.search_topk([q], k=kk)
            assert_topk(d[0], s[0], dense, (q, kk))
    small = SearchArray.index(["a b", "b", "a a", "c"] * 10)
    d, s = small.search_topk(["a", "b", "zzz"], k=1024)
    for i, q in enumerate(["a", "b", "zzz"]):
        assert_topk(d[i], s[i], small.score(q), q)


def test_two_million_docs_at_k1000():
    """The 2M-doc synthetic corpus (bench.py's generator) at k = 1,000."""
    from searcharray_b200 import SearchArray, synth
    spec = synth.SynthSpec(2_000_000)
    host, _, _ = synth.generate_shard(spec)
    host.avg_doc_length = synth.global_avg_doc_length(spec)
    arr = SearchArray.from_host_index(host, avg_doc_length=host.avg_doc_length)
    queries = list(synth.stratified_term_queries(spec, 64))[::8]
    check_queries(arr, queries, oracle_dense(arr, queries), ks=(1000,), what="2M")


def test_k_range_refused(corpus):
    import pandas as pd
    from searcharray_b200 import classic_similarity
    from searcharray_b200.solr import edismax_topk
    for k in (0, 1025):
        with pytest.raises(ValueError, match=r"\[1, 1024\]"):
            corpus.search_topk(["w0"], k=k)
        with pytest.raises(ValueError, match=r"\[1, 1024\]"):
            corpus.search_topk(["w0"], k=k, similarity=classic_similarity())
        with pytest.raises(ValueError, match=r"\[1, 1024\]"):
            edismax_topk(pd.DataFrame({"body": corpus}), "w0", qf=["body"], k=k)


def test_feature_clauses(corpus):
    """The FEATURE instances of the deep boolean fold, with and without a mask, and the COUNT ones (facets=)."""
    from searcharray_b200 import Bool, Boost, Feature, Or
    f32 = np.float32
    rng = np.random.default_rng(12)
    pop = np.where(rng.random(len(corpus)) < 0.3, rng.integers(1, 500, len(corpus)), 0).astype(f32)
    corpus.set_feature("pop", pop)
    s1, s5 = corpus.score("w1"), corpus.score("w5")
    sat = np.where(pop > 0, pop / (pop + f32(50)), f32(0)).astype(f32)
    queries = [Or(["w1", Feature("pop")]), Bool(must=["w5"], should=[Boost(Feature("pop", "saturation", pivot=50), 2.0)])]
    dense = [(s1 + pop).astype(f32),
             np.where(s5 > 0, s5 + (f32(2) * sat).astype(f32), f32(0)).astype(f32)]
    check_queries(corpus, queries, dense, what="feature")
    check_prefix(corpus, queries, what="feature")
    mask = np.random.default_rng(13).random(len(corpus)) < 0.5
    check_queries(corpus, queries, [np.where(mask, d, f32(0)) for d in dense], ks=(64, 1024), what="feature where",
                  where=mask)
    corpus.set_facet("mod3", (np.arange(len(corpus)) % 3).astype(np.int32))
    d, s, h = corpus.search_topk(queries, k=1000, facets=["mod3"])
    for i in range(len(queries)):
        assert_topk(d[i], s[i], dense[i], ("feature facets", i))
        assert h.total[i] == np.count_nonzero(dense[i] > 0)


@pytest.mark.parametrize("view", [None, "mask", "stepped"])
def test_classic_similarity(corpus, view):
    from searcharray_b200 import classic_similarity
    sim = classic_similarity()
    rng = np.random.default_rng(14)
    v = corpus if view is None else {"mask": lambda a: a[rng.random(len(a)) < 0.5], "stepped": lambda a: a[1::3]}[view](corpus)
    queries = TERMS + PHRASES
    dense = [np.asarray(v.score(q, similarity=sim), dtype=np.float64) for q in queries]
    check_queries(v, queries, dense, what=("classic", view), similarity=sim)
    check_prefix(v, queries, what=("classic", view), similarity=sim)


def test_edismax_topk(corpus):
    import pandas as pd
    from searcharray_b200 import SearchArray
    from searcharray_b200.solr import edismax, edismax_topk
    rng = np.random.default_rng(15)
    n = 3 * TILE + 77
    frame = pd.DataFrame({"title": SearchArray.index(random_corpus(rng, n, 150, mean_len=4)),
                          "body": SearchArray.index(random_corpus(rng, n, 300))})
    for q, kw in (("w1 w2", {}), ("w0 w3 w7", {"mm": 2, "pf": ["body"], "tie": 0.3})):
        dense = np.asarray(edismax(frame, q, qf=["title^2", "body"], **kw)[0], dtype=np.float64)
        first = {}
        for k in KS + (1, 10, 32):
            docs, scores = edismax_topk(frame, q, qf=["title^2", "body"], k=k, **kw)
            assert_topk(docs, scores, dense, ("edismax", q, k))
            first[k] = (docs, scores)
        for kp in (1, 10, 32):
            assert np.array_equal(first[1024][0][:kp], first[kp][0])
            assert np.array_equal(first[1024][1][:kp].view(np.uint64), first[kp][1].view(np.uint64))


@pytest.mark.parametrize("world", [1, 2, 5, 8])
def test_device_merge_of_rank_lists(corpus, world):
    """sa_topk_merge: the device merge of the all-gather (topk_merge_kernel, and topk_merge_ranked_kernel above
    4,096 keys) over synthetic per-rank lists -- sorted, 0-padded, disjoint doc ranges, ties in score across ranks."""
    from searcharray_b200 import _lib
    rng = np.random.default_rng(world)
    nq = 3
    for k in (10, 100, 1000, 1024):
        lists = np.zeros((world, nq, k), dtype=np.uint64)
        for r in range(world):
            for q in range(nq):
                m = int(rng.integers(0, k + 1))
                docs = r * 1_000_000 + rng.choice(1_000_000, size=m, replace=False)
                bits = np.float32(rng.integers(1, 40, m) / 8).view(np.uint32).astype(np.uint64)
                keys = (bits << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - docs.astype(np.uint64))
                lists[r, q, :m] = np.sort(keys)[::-1]
        out = np.empty((nq, k), dtype=np.uint64)
        _lib.check(_lib.lib().sa_topk_merge(corpus._device().handle, _lib.p_u64(lists.reshape(-1)), world, nq, k,
                                            _lib.p_u64(out)))
        for q in range(nq):
            want = np.sort(lists[:, q, :].reshape(-1))[::-1][:k]
            assert np.array_equal(out[q], want), (world, k, q)
