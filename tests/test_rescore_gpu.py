"""GPU: scoring at given documents (SearchArray.score_docs, solr.fields_score_docs; bool_docs_kernel in sa_bool.cu)
and window rescoring (query.Rescore).

The invariant: score_docs(queries, search_topk(queries, k)[0]) equals search_topk's scores bit for bit, for every
query form, on a random Zipf corpus of three tiles and a partial fourth (empty docs included) and on the TMDB fixture.
Dense parity: at random docs, ranked and not, at tile edges, duplicated and NO_DOC, score_docs equals the dense vector
composed from .score (compose_nested), also under BM25 parameters that are not sparse-safe.  Then fields, a shard, the
device memory and launches of a term-and-feature call (no dense row), Rescore against its numpy composition, and the
invariant at scale on a 2M-doc synthetic corpus."""
import ctypes
import os

import numpy as np
import pandas as pd
import pytest

from _nested_compose import compose_nested
from _tmdb_index import load_field
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

TILE = 8192
N = 3 * TILE + 1234
NO_DOC = 0xFFFFFFFF
K = 1024


def zipf_array(n=N, seed=3, vocab=3000):
    """Random Zipf text: w0 the most frequent token (a tf-table list), w1000+ rare ones (binary search over words);
    about 3 % of the docs are empty."""
    from searcharray_b200 import SearchArray
    rng = np.random.default_rng(seed)
    lens = np.where(rng.random(n) < 0.03, 0, rng.integers(1, 40, n))
    toks = np.minimum(rng.zipf(1.3, int(lens.sum())), vocab) - 1
    ends = np.cumsum(lens)
    docs = [" ".join(f"w{t}" for t in toks[e - ln:e]) for e, ln in zip(ends, lens)]
    return SearchArray.index(docs)


def add_features(arr, seed=4):
    rng = np.random.default_rng(seed)
    n = len(arr)
    arr.set_feature("pop", np.where(rng.random(n) < 0.7, rng.integers(1, 500, n), 0).astype(np.float32))
    frac = np.zeros(n, dtype=np.float32)
    frac[TILE:] = rng.random(n - TILE) * 10                 # tile 0 without a value
    arr.set_feature("frac", frac)
    arr.set_facet("lang", rng.integers(-1, 5, n))


@pytest.fixture(scope="module")
def zipf():
    arr = zipf_array()
    add_features(arr)
    return arr


def scorer(arr):
    from searcharray_b200 import Feature, Field

    def score(c):
        if isinstance(c, Field):
            return scorer(frame_arrays[c.field])(c.clause)
        if isinstance(c, Feature):
            return c.apply(arr.host.features[c.name])
        return arr.score(c)
    return score


frame_arrays = {}


def dense_of(score, q):
    """S_q: what search_topk ranks query q from, +0 where a doc does not rank."""
    from searcharray_b200 import Or
    from searcharray_b200.query import is_boolean
    return compose_nested(score, q if is_boolean(q) else Or([q]))


def forms():
    """{name: (queries, slop)}: every form the boolean path takes, and plain terms and phrases."""
    from searcharray_b200 import And, Bool, Boost, DisMax, Feature, Or
    return {
        "terms": (["w0", "w3", "w40", "w1500", "nope"], 0),
        "phrase0": ([["w0", "w1"], ["w1", "w0"], ["w0", "w0"], ["w2", "w1", "w0"]], 0),
        "phrase2": ([["w0", "w2"], ["w3", "w1", "w0"]], 2),
        "or_and": ([Or(["w0", "w5", "w9"], mm=2), And(["w1", "w2"]), Or(["w4", ["w0", "w1"], "nope"])], 0),
        "bool": ([Bool(must=["w0"], should=[Boost("w3", 2.5), "w8"], filter=["w1"], must_not=["w12"], mm=1),
                  Bool(should=[Boost("w2", 0.5), "w40", ["w0", "w1"]], must_not=["w0"]),
                  Bool(must=[Boost("w6", 0.0)], should=["w7"])], 0),
        "dismax": ([Or([DisMax(["w1", Boost("w2", 2.0)], tie=0.3), "w5"]), DisMax(["w3", "w6", "w9"], tie=0.1),
                    Bool(must=[DisMax([["w0", "w1"], "w11"])], must_not=[DisMax(["w20", "w21"])])], 0),
        "nested": ([Or([And(["w0", Or(["w1", Bool(must=["w2"], should=["w3"])])]), "w7"]),
                    Bool(must=[Or(["w4", "w5"])], should=[Boost(And(["w0", "w1"]), 1.5)], must_not=[And(["w0", "w6"])]),
                    Or([Or([Or(["w8", DisMax(["w9", "w10"], tie=0.5)])]), Feature("pop", "log", scaling_factor=2)])], 0),
        "features": ([Bool(should=["w0", Feature("pop")]), Or(["w1", Feature("frac", "saturation", pivot=2.0)]),
                      Bool(must=["w2"], should=[Boost(Feature("pop", "log", scaling_factor=2), 0.7)]),
                      Bool(filter=[Feature("frac")], should=["w3"]), Bool(should=[Feature("frac", "log",
                                                                                          scaling_factor=1.5)])], 0),
    }


def bits(a):
    return np.asarray(a, dtype=np.float32).view(np.uint32)


def assert_invariant(arr, queries, slop, what, k=K, similarity=None):
    from searcharray_b200 import bm25_similarity
    sim = similarity or bm25_similarity()
    docs, scores = arr.search_topk(queries, k=k, slop=slop, similarity=sim)
    got = arr.score_docs(queries, docs, slop=slop, similarity=sim)
    assert got.shape == docs.shape and got.dtype == np.float32
    assert np.array_equal(bits(got), bits(scores)), what
    assert (docs != NO_DOC).any(), what
    return docs, scores


@pytest.mark.parametrize("form", list(forms()))
def test_invariant_zipf(zipf, form):
    queries, slop = forms()[form]
    assert_invariant(zipf, queries, slop, form)


def test_invariant_mixed_batch(zipf):
    """Every form of slop 0 in one score_docs call, flattened at its heaviest form (search_topk runs one call per
    form): the same scores."""
    queries = [q for name, (qs, slop) in forms().items() if slop == 0 for q in qs]
    assert_invariant(zipf, queries, 0, "mixed")


def test_paths_are_exercised(zipf):
    """w0 has a tf table (long list), w1500 is read by binary search over its words."""
    host = zipf.host
    t0, t1 = zipf._term_id("w0"), zipf._term_id("w1500")
    assert host.term_lengths[t0] > 20 * host.term_lengths[t1] > 0


@pytest.fixture(scope="module")
def tmdb():
    from searcharray_b200 import SearchArray
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    return pd.DataFrame({name: SearchArray.from_host_index(load_field(z, name))
                         for name in ("title_tokens", "overview_tokens")})


def test_invariant_tmdb(tmdb):
    from searcharray_b200 import And, Bool, Boost, DisMax, Or
    arr = tmdb["overview_tokens"].array
    qs = ["war", "love", "zzzz", ["star", "wars"], Or(["alien", "space", "ship"], mm=2), And(["young", "man"]),
          Bool(must=["life"], should=[Boost("family", 2.0)], must_not=["war"]),
          Or([DisMax(["film", "movie"], tie=0.1), And(["new", Or(["york", "city"])])])]
    assert_invariant(arr, qs, 0, "tmdb")
    assert_invariant(arr, [["star", "wars"], ["world", "war"]], 2, "tmdb slop 2")


def test_dense_parity(zipf):
    """Random docs, ranked and not, the tile edges, duplicates and NO_DOC: S_q gathered from the .score
    composition, bit for bit."""
    rng = np.random.default_rng(7)
    queries = [q for qs, slop in forms().values() if slop == 0 for q in qs]
    top, _ = zipf.search_topk(queries, k=16)
    n = len(zipf)
    docs = rng.integers(0, n, (len(queries), 96)).astype(np.uint32)
    docs[:, :4] = [0, TILE - 1, TILE, n - 1]
    docs[:, 4:20] = top
    docs[:, 20:24] = docs[:, 4:8]                            # duplicates
    docs[:, 24] = NO_DOC
    got = zipf.score_docs(queries, docs)
    score = scorer(zipf)
    for i, q in enumerate(queries):
        dense = dense_of(score, q)
        want = np.where(docs[i] == NO_DOC, np.float32(0), dense[np.minimum(docs[i], n - 1)])
        assert np.array_equal(bits(got[i]), bits(want)), q
    assert (got > 0).any() and (got == 0).any()


@pytest.mark.parametrize("k1,b", [(1.2, 1.0), (1.2, 1.5), (-0.5, 0.75)])
def test_dense_parity_not_sparse_safe(zipf, k1, b):
    """Parameters under which a doc without the term does not score +0 under .score (NaN at empty docs, -0 or
    negative norms): every doc is evaluated with bm25_one, as the tile fold does."""
    from searcharray_b200 import Or, bm25_similarity
    sim = bm25_similarity(k1=k1, b=b)
    queries = ["w0", "w7", "w1500", Or(["w0", "w2"]), Or(["w1", "w3", "w40"], mm=2)]
    n = len(zipf)
    rng = np.random.default_rng(8)
    docs = rng.integers(0, n, (len(queries), 200)).astype(np.uint32)
    docs[:, :4] = [0, TILE - 1, TILE, n - 1]
    empty = np.flatnonzero(zipf.doc_lens == 0)[:8]
    docs[:, 4:4 + len(empty)] = empty
    got = zipf.score_docs(queries, docs, similarity=sim)
    for i, q in enumerate(queries):
        dense = dense_of(lambda c: zipf.score(c, similarity=sim), q)
        assert np.array_equal(bits(got[i]), bits(dense[docs[i]])), q
    assert_invariant(zipf, queries, 0, f"k1={k1} b={b}", similarity=sim)


@pytest.fixture(scope="module")
def frame(zipf):
    other = zipf_array(seed=9)
    add_features(other, seed=10)
    f = pd.DataFrame({"t": zipf, "o": other})
    f["t2"] = f["t"]                                        # one device index under two names
    frame_arrays.update({"t": zipf, "o": other, "t2": zipf})
    return f


def test_fields(frame):
    from searcharray_b200 import Bool, Boost, DisMax, Feature, Field, Or, fields_score_docs, fields_topk
    qs = [Bool(should=[Field("t", "w0"), Field("o", "w1")]),
          Bool(must=[Field("t2", "w2")], should=[Field("t", "w3"), Field("o", ["w0", "w1"])]),
          Or([DisMax([Field("t", "w1"), Boost(Field("o", "w1"), 2.0), Field("t2", "w4")], tie=0.2),
              Field("o", Feature("pop"))]),
          Bool(must=[Or([Field("o", "w5"), Field("t", "w6")])], must_not=[Field("t2", "w0")])]
    docs, scores = fields_topk(frame, qs, k=K)
    got = fields_score_docs(frame, qs, docs)
    assert np.array_equal(bits(got), bits(scores)) and (docs != NO_DOC).any()
    rng = np.random.default_rng(3)
    rows = rng.integers(0, len(frame), (len(qs), 64)).astype(np.uint32)
    rows[:, 0] = NO_DOC
    got = fields_score_docs(frame, qs, rows)
    for i, q in enumerate(qs):
        dense = dense_of(scorer(frame_arrays["t"]), q)
        want = np.where(rows[i] == NO_DOC, np.float32(0), dense[np.minimum(rows[i], len(frame) - 1)])
        assert np.array_equal(bits(got[i]), bits(want)), q


def test_shard_doc_base():
    """Global ids on a shard: accepted through the public call, others refused by it and by the C entry point."""
    from searcharray_b200 import Or, SearchArray, bm25_similarity
    from searcharray_b200._lib import SearchArrayB200Error
    from test_bool_topk_gpu import synth_corpus
    base = 1_000_003
    host, _ = synth_corpus(doc_base=base)
    shard = SearchArray.from_host_index(host, doc_base=base)
    qs = ["w0", "s2", Or(["w1", "t3"]), ["pa", "pb"]]
    docs, scores = assert_invariant(shard, qs, 0, "shard")
    assert docs[docs != NO_DOC].min() >= base
    for bad in (base - 1, base + len(shard), 0):
        d = docs.copy()
        d[0, 0] = bad
        with pytest.raises(ValueError):
            shard.score_docs(qs, d)
        with shard._shared["lock"]:
            prep = shard._prepare_bool([q if not isinstance(q, (str, list)) else Or([q]) for q in qs],
                                       bm25_similarity())
            with pytest.raises(SearchArrayB200Error, match="error 2"):
                prep.score_docs(np.ascontiguousarray(d, dtype=np.uint32), 0)


def stats(arr):
    from searcharray_b200 import _lib
    st = _lib.SaStats()
    _lib.check(_lib.lib().sa_stats_get(arr._device().handle, ctypes.byref(st)))
    return st


def live_bytes():
    from searcharray_b200 import _lib
    nbuf, nbytes = ctypes.c_uint64(0), ctypes.c_uint64(0)
    _lib.check(_lib.lib().sa_device_allocations(ctypes.byref(nbuf), ctypes.byref(nbytes)))
    return nbytes.value


def test_no_dense_rows():
    """A term-and-feature batch: no term, phrase or tile-fold launch, and less device memory than one score row."""
    from searcharray_b200 import Bool, Feature, Or
    arr = zipf_array(seed=21)
    add_features(arr)
    arr._device()
    before, st0 = live_bytes(), stats(arr)
    qs = ["w0", Or(["w1", "w1500"], mm=1), Bool(should=["w2", Feature("pop")]),
          Bool(must=[Feature("frac", "saturation", pivot=1.0)], should=["w3"])]
    docs = np.tile(np.arange(K, dtype=np.uint32) * 7 % len(arr), (len(qs), 1))
    arr.score_docs(qs, docs)
    grown, st1 = live_bytes() - before, stats(arr)
    padded = -(-len(arr) // TILE) * TILE
    assert grown < 8 * padded, (grown, padded)
    for f in ("term_kernel_launches", "bool_instances", "phrase_kernel_launches"):
        assert getattr(st1, f) == getattr(st0, f), f
    assert st1.total_launches > st0.total_launches


@pytest.fixture(scope="module")
def rescore_case(zipf):
    from searcharray_b200 import And, Bool, Boost, DisMax, Feature, Or
    qs = [Or(["w1", "w2"]), "w3", Bool(must=["w4"], should=["w0"]), "w1500", And(["w0", "w1"])]
    rq = [Bool(should=[Or(["w1", "w2", "w5"]), Feature("pop", "saturation", pivot=100)]), ["w3", "w0"],
          Or([Boost("w0", 2.0), "w7"]), "w1", DisMax(["w0", "w1"], tie=0.25)]
    return qs, rq


def window_dense(arr, q, rq, window, qw, rw, k):
    """The fully dense composition of one rescored query: the top window of S_q, then c over it."""
    score = scorer(arr)
    d1 = dense_of(score, q)
    order = np.lexsort((np.arange(len(d1)), -d1.astype(np.float64)))[:window]
    order = order[d1[order] > 0]
    d2 = dense_of(score, rq)
    c = (np.float32(qw) * d1[order]).astype(np.float32) + (np.float32(rw) * d2[order]).astype(np.float32)
    o2 = np.lexsort((order, -c.astype(np.float64)))[:k]
    docs = np.full(k, NO_DOC, dtype=np.uint32)
    sc = np.zeros(k, dtype=np.float32)
    docs[:len(o2)], sc[:len(o2)] = order[o2], c[o2]
    return docs, sc


@pytest.mark.parametrize("window,k,qw,rw", [(100, 10, 1.0, 1.0), (50, 50, 0.5, 2.0), (1024, 20, 1.0, 0.3)])
def test_rescore(zipf, rescore_case, window, k, qw, rw):
    from searcharray_b200 import Rescore
    from searcharray_b200.query import rescore_window
    qs, rq = rescore_case
    r = Rescore(rq, window=window, query_weight=qw, rescore_weight=rw)
    docs, scores = zipf.search_topk(qs, k=k, rescore=r)
    d1, s1 = zipf.search_topk(qs, k=window)
    s2 = zipf.score_docs(rq, d1)
    wd, ws = rescore_window(d1, s1, s2, qw, rw, k)
    assert np.array_equal(docs, wd) and np.array_equal(bits(scores), bits(ws))
    # a window below the match count of some queries and above that of w1500's
    n_match = (d1 != NO_DOC).sum(axis=1)
    assert window == 1024 or n_match.max() == window
    assert n_match[3] < window
    for i in range(len(qs)):
        dd, ds = window_dense(zipf, qs[i], rq[i], window, qw, rw, k)
        assert np.array_equal(docs[i], dd) and np.array_equal(bits(scores[i]), bits(ds)), qs[i]


def test_rescore_zero_weight_is_pass_one(zipf, rescore_case):
    from searcharray_b200 import Rescore
    qs, rq = rescore_case
    docs, scores = zipf.search_topk(qs, k=30, rescore=Rescore(rq, window=200, rescore_weight=0.0))
    d1, s1 = zipf.search_topk(qs, k=30)
    assert np.array_equal(docs, d1) and np.array_equal(bits(scores), bits(s1))


def test_rescore_where_and_facets(zipf, rescore_case):
    from searcharray_b200 import Rescore
    from searcharray_b200.query import rescore_window
    qs, rq = rescore_case
    m = np.random.default_rng(2).random(len(zipf)) < 0.5
    r = Rescore(rq, window=64)
    docs, scores, hits = zipf.search_topk(qs, k=16, where=m, facets=["lang"], rescore=r)
    d1, s1, h1 = zipf.search_topk(qs, k=64, where=m, facets=["lang"])
    assert np.array_equal(hits.total, h1.total) and np.array_equal(hits.facets["lang"], h1.facets["lang"])
    wd, ws = rescore_window(d1, s1, zipf.score_docs(rq, d1), 1.0, 1.0, 16)
    assert np.array_equal(docs, wd) and np.array_equal(bits(scores), bits(ws))
    assert m[docs[docs != NO_DOC]].all()


def test_rescore_fields(frame):
    from searcharray_b200 import Bool, Field, Rescore, fields_score_docs, fields_topk
    from searcharray_b200.query import rescore_window
    qs = [Bool(should=[Field("t", "w1"), Field("o", "w1")]), Bool(must=[Field("o", "w2")])]
    rq = [Bool(should=[Field("t", ["w0", "w1"]), Field("o", "w0")]), Bool(should=[Field("t2", "w3")])]
    r = Rescore(rq, window=200, query_weight=2.0, rescore_weight=0.5, slop=1)
    docs, scores = fields_topk(frame, qs, k=25, rescore=r)
    d1, s1 = fields_topk(frame, qs, k=200)
    wd, ws = rescore_window(d1, s1, fields_score_docs(frame, rq, d1, slop=1), 2.0, 0.5, 25)
    assert np.array_equal(docs, wd) and np.array_equal(bits(scores), bits(ws))


def test_scale_2m():
    """64 queries on a 2M-doc synthetic corpus, whose long lists take the tf table: the invariant at k = 1,024."""
    from searcharray_b200 import Or, SearchArray, synth
    spec = synth.SynthSpec(2_000_000)
    host, lo, _ = synth.generate_shard(spec)
    arr = SearchArray.from_host_index(host, avg_doc_length=synth.global_avg_doc_length(spec))
    terms = synth.stratified_term_queries(spec, 56)
    qs = terms[:40] + [Or([a, b]) for a, b in zip(terms[40:48], terms[48:56])] + synth.phrase_queries(spec, 8) + \
        [Or(terms[i:i + 3], mm=2) for i in range(0, 24, 3)]
    assert len(qs) == 64
    assert_invariant(arr, qs, 0, "2M")
