"""GPU: feature clauses (query.Feature over SearchArray.set_feature columns; the FEATURE instances of bool_tile in
sa_bool.cu and sa_index_set_feature in sa_feature.cu) against compose_nested with each text clause scored by this
library's .score and each feature clause by Feature.apply over the registered values: ids and float32 score bits
must be equal.

The corpus is tests/test_bool_topk_gpu.py's five-tile synthetic one (plus its second column for fields_topk).  Its
feature columns: `pop` (integers, ~80 % of docs non-zero), `frac` (floats, every doc), `range` (non-zero in tiles 1-2
only: whole tiles absent), `tail` (non-zero in the last, partial tile only), `zero` (no non-zero value), `tiny`
(values whose log(1 + x) or saturation underflows to 0), and `ties` (320 docs of tile 1, owned by ten threads, at one
integer value: more exact ties than candidate slots)."""

import numpy as np
import pandas as pd
import pytest

from _nested_compose import compose_nested
from test_bool_fields_gpu import A, B, fb_corpus
from test_bool_topk_gpu import KS, TILE, assert_topk, synth_corpus

pytestmark = pytest.mark.gpu

N = 5 * TILE + 300


def feature_columns(n=N, seed=5):
    rng = np.random.default_rng(seed)
    pop = np.where(rng.random(n) < 0.8, rng.integers(1, 1000, n), 0).astype(np.float32)
    frac = (rng.random(n) * 100).astype(np.float32)
    rng_col = np.zeros(n, dtype=np.float32)
    rng_col[TILE:3 * TILE] = np.where(rng.random(2 * TILE) < 0.5, rng.random(2 * TILE) * 10, 0)
    tail = np.zeros(n, dtype=np.float32)
    tail[5 * TILE:] = rng.integers(1, 50, n - 5 * TILE)
    tiny = np.zeros(n, dtype=np.float32)
    tiny[::7] = 1e-45                                        # log(1 + x) == 0 in double; saturation underflows
    tiny[3::7] = 1e-38
    tiny[5::7] = rng.random(len(tiny[5::7])) * 3
    ties = np.zeros(n, dtype=np.float32)              # tile 1: the 320 docs threads 10-19 own, one integer value
    ties[[TILE + 4 * t + 1024 * j + e for t in range(10, 20) for j in range(8) for e in range(4)]] = 7
    return {"pop": pop, "frac": frac, "range": rng_col, "tail": tail, "zero": np.zeros(n, dtype=np.float32),
            "tiny": tiny, "ties": ties}


class Corpus:
    def __init__(self):
        from searcharray_b200 import SearchArray
        self.host, _ = synth_corpus()
        self.arr = SearchArray.from_host_index(self.host)
        self.cols = feature_columns()
        for name, v in self.cols.items():
            self.arr.set_feature(name, v)


@pytest.fixture(scope="module")
def corpus():
    return Corpus()


def scorer(arr):
    """score(clause) for compose_nested on one column: .score for text, Feature.apply over the registered values."""
    from searcharray_b200 import Feature

    def score(c):
        if isinstance(c, Feature):
            return c.apply(arr.host.features[c.name])
        return arr.score(c)
    return score


def check(arr, queries, k, what, where=None):
    docs, scores = arr.search_topk(queries, k=k, where=where)
    assert docs.shape == (len(queries), k) and scores.dtype == np.float32
    score = scorer(arr)
    for i, q in enumerate(queries):
        dense = compose_nested(score, q)
        if where is not None:
            m = np.asarray(where)
            dense = np.where(m if m.ndim == 1 else m[i], dense, np.float32(0))
        assert_topk(docs[i], scores[i], dense, k, f"{what} {q!r} k={k}")
    return docs, scores


def functions():
    from searcharray_b200 import Feature
    return [Feature("pop"), Feature("pop", "saturation", pivot=50), Feature("frac", "log", scaling_factor=1),
            Feature("frac", "saturation", pivot=0.5), Feature("pop", "log", scaling_factor=3.5)]


@pytest.mark.parametrize("k", KS)
def test_functions_roles_boosts(corpus, k):
    """Every function in every role, boosted and not, mm counting a feature, and Or / And holding one."""
    from searcharray_b200 import And, Bool, Boost, Or
    qs = []
    for f in functions():
        qs += [Or(["w1", f]), And(["s1", f]), Or(["w0", "w2", f], mm=2), Or([Boost(f, 0.25), "w2"]),
               Bool(must=[Or(["w0", "w1"])], should=[Boost(f, 2.0)]),
               Bool(must=[f], should=["w2", "s2"]),
               Bool(should=["w1", "w2", f], mm=2),
               Bool(should=["w1"], filter=[f]), Bool(should=["w0"], must_not=[f]),
               Bool(must=[Boost(f, 0)], should=["s1"]),
               Bool(should=[f])]
    check(corpus.arr, qs, k, "roles")


def test_or_and_promotion_is_the_roles_result(corpus):
    """An Or / And with a feature runs as the roles form; Bool(should=...) with the same clauses ranks the same."""
    from searcharray_b200 import Bool, Feature, Or
    f = Feature("pop", "saturation", pivot=50)
    d1, s1 = corpus.arr.search_topk([Or(["w1", f, "s2"], mm=2)], k=20)
    d2, s2 = corpus.arr.search_topk([Bool(should=["w1", f, "s2"], mm=2)], k=20)
    assert np.array_equal(d1, d2) and np.array_equal(s1.view(np.uint32), s2.view(np.uint32))


def test_nested_and_dismax_forms(corpus):
    from searcharray_b200 import And, Bool, Boost, DisMax, Feature, Or
    f, g = Feature("pop", "log", scaling_factor=1), Feature("range", "saturation", pivot=2)
    qs = [Or([And(["w0", f]), And(["w1", g])]),
          Bool(must=[Or(["s1", f], mm=2)], should=[Boost(g, 3)]),
          Bool(should=["w0", Bool(must=[g], should=[f])], must_not=[And(["t3", f])]),
          Or([Or([Or([f])]), "t0"]),
          Bool(must=[DisMax(["w0", "w1"], tie=0.2)], should=[Boost(f, 1.5)]),     # DisMax form, feature plain
          Or([DisMax(["s1", "s2"], tie=0.5), g, "t3"], mm=2)]
    for k in (1, 10, 32):
        check(corpus.arr, qs, k, "nested / dismax")


def test_where(corpus):
    from searcharray_b200 import Bool, Feature, Or
    f = Feature("pop", "saturation", pivot=50)
    qs = [Bool(must=["w0"], should=[f]), Or(["w2", Feature("frac")]), Bool(should=[f])]
    rng = np.random.default_rng(3)
    one = rng.random(N) < 0.3
    per = rng.random((len(qs), N)) < 0.5
    per[2, :2 * TILE] = False
    for k in (1, 10, 17):
        check(corpus.arr, qs, k, "where one", where=one)
        check(corpus.arr, qs, k, "where per query", where=per)


def test_tile_ranges_and_empty_features(corpus):
    """range: whole tiles absent (MUST pruning); tail: only the last partial tile; zero: no non-zero value; tiny:
    values whose function underflows to 0 do not match."""
    from searcharray_b200 import Bool, Feature, Or
    qs = [Bool(must=[Feature("range")], should=["w0"]), Bool(must=[Feature("range", "log", scaling_factor=1)]),
          Or(["t3", Feature("range")], mm=2), Bool(should=[Feature("tail")], filter=["w0"]),
          Bool(should=[Feature("tail", "saturation", pivot=10)]), Bool(should=["w1", Feature("zero")], mm=2),
          Bool(must=[Feature("zero")], should=["w0"]), Bool(should=["w2"], must_not=[Feature("zero")]),
          Bool(should=[Feature("tiny", "log", scaling_factor=1)]), Bool(should=[Feature("tiny", "saturation", pivot=1e30)]),
          Bool(should=[Feature("tiny")]), Or(["w0", Feature("tiny", "log", scaling_factor=1)], mm=2)]
    docs, scores = check(corpus.arr, qs, 32, "ranges")
    assert (docs[0] >= TILE).all() and (docs[0] < 3 * TILE).all()
    assert (docs[3][docs[3] != 0xFFFFFFFF] >= 5 * TILE).all() and (docs[3] != 0xFFFFFFFF).any()
    assert (docs[5] == 0xFFFFFFFF).all() and (docs[6] == 0xFFFFFFFF).all()
    tiny = corpus.cols["tiny"]
    for i in (8, 9):     # no doc with the underflowing values ranks
        got = docs[i][docs[i] != 0xFFFFFFFF]
        assert len(got) and not np.isin(tiny[got], [np.float32(1e-45)]).any()


def test_exact_ties_rerun(corpus):
    """320 docs of tile 1 tie at one feature score.  With fewer threads holding a tie than k = 32 the tile keeps
    every tie, more than its candidate slots, and the query is re-run exactly (n_redone)."""
    from searcharray_b200 import Bool, Feature, bm25_similarity
    qs = [Bool(should=[Feature("ties")]), Bool(should=[Feature("ties", "log", scaling_factor=1)], filter=["w0"])]
    for k in (10, 32):
        docs, scores, n_redone = corpus.arr._search_topk_bool(qs, k, bm25_similarity(), 0)
        assert k == 10 or n_redone >= 1
        score = scorer(corpus.arr)
        for i, q in enumerate(qs):
            assert_topk(docs[i], scores[i], compose_nested(score, q), k, f"ties {q!r}")
        assert (scores[0] == np.float32(7)).all()


def test_mixed_batch(corpus):
    """Plain terms, phrases, feature-free boolean queries and feature queries in one batch: the feature-free ones
    rank exactly as a batch without any feature."""
    from searcharray_b200 import And, Bool, Boost, Feature, Or
    plain = ["w1", ["pa", "pb"], Or(["w0", "s1"]), Bool(must=["w2"], should=[Boost("w1", 2)]),
             Or([And(["w0", "w1"]), "t0"])]
    feat = [Bool(must=["w1"], should=[Feature("pop")]), Or([["pa", "pb"], Feature("frac", "log", scaling_factor=1)])]
    mixed = [plain[0], feat[0], plain[1], plain[2], feat[1], plain[3], plain[4]]
    dm, sm = corpus.arr.search_topk(mixed, k=10)
    dp, sp = corpus.arr.search_topk(plain, k=10)
    for i, j in ((0, 0), (2, 1), (3, 2), (5, 3), (6, 4)):
        assert np.array_equal(dm[i], dp[j]) and np.array_equal(sm[i].view(np.uint32), sp[j].view(np.uint32)), i
    score = scorer(corpus.arr)
    for i in (1, 4):
        assert_topk(dm[i], sm[i], compose_nested(score, mixed[i]), 10, f"mixed {mixed[i]!r}")


def test_reregister_and_set_after_device():
    """A name set again replaces its values on the device; a name set after the device index exists is uploaded."""
    from searcharray_b200 import Bool, Feature, SearchArray
    host, _ = synth_corpus()
    arr = SearchArray.from_host_index(host)
    arr.search_topk(["w0"], k=5)                          # the device index exists
    cols = feature_columns()
    arr.set_feature("pop", cols["pop"])
    q = [Bool(must=["w1"], should=[Feature("pop", "saturation", pivot=50)])]
    check(arr, q, 10, "set after device")
    arr.set_feature("pop", cols["frac"])
    check(arr, q, 10, "re-registered")
    assert np.array_equal(arr.host.features["pop"], cols["frac"])


def test_fields_topk():
    """Field(column, Feature) on the column whose index holds it, and on a second name of that column."""
    from searcharray_b200 import And, Bool, Boost, DisMax, Feature, Field, Or, SearchArray, fields_topk
    ha, _ = synth_corpus()
    hb, _ = fb_corpus()
    frame = pd.DataFrame({A: SearchArray.from_host_index(ha), B: SearchArray.from_host_index(hb)})
    frame["fa2"] = frame[A]
    cols = feature_columns()
    frame[A].array.set_feature("pop", cols["pop"])
    frame[B].array.set_feature("votes", cols["range"])

    def score(c):
        arr = frame[c.field].array
        if isinstance(c.clause, Feature):
            return c.clause.apply(arr.host.features[c.clause.name])
        return arr.score(c.clause)
    pop, votes = Feature("pop", "saturation", pivot=50), Feature("votes", "log", scaling_factor=1)
    qs = [Bool(must=[Field(A, "w0")], should=[Field(A, pop)]),
          Bool(must=[Field(B, "b1")], should=[Boost(Field("fa2", pop), 2), Field(B, votes)]),
          Or([Field(A, "w1"), Field(B, votes), Field("fa2", Feature("pop"))], mm=2),
          Bool(should=[DisMax([Field(A, "w0"), Field(B, "b1")], tie=0.3), Field(B, votes)]),
          Or([And([Field(A, "s1"), Field(A, pop)]), Field(B, "b2")])]
    for k in (1, 10, 32):
        docs, scores = fields_topk(frame, qs, k=k)
        for i, q in enumerate(qs):
            assert_topk(docs[i], scores[i], compose_nested(score, q), k, f"fields {q!r} k={k}")
    where = np.random.default_rng(9).random(N) < 0.4
    docs, scores = fields_topk(frame, qs, k=10, where=where)
    for i, q in enumerate(qs):
        assert_topk(docs[i], scores[i], np.where(where, compose_nested(score, q), np.float32(0)), 10, f"fields where {q!r}")


def _c_call(arr, clauses, starts, terms, term_starts, idf, weights=None, occurs=None, groups=None, ties=None,
            mm=None, k=10):
    """sa_score_batch_topk_bool on one array: (rc, docs, scores)."""
    from searcharray_b200 import _lib
    u32 = lambda x: np.asarray(x, dtype=np.uint32)      # noqa: E731
    f32 = lambda x: np.asarray(x, dtype=np.float32)     # noqa: E731
    starts, terms, term_starts, idf = u32(starts), u32(terms), u32(term_starts), f32(idf)
    nq = len(starts) - 1
    mm = u32(mm if mm is not None else [1] * nq)
    docs = np.empty((nq, k), dtype=np.uint32)
    scores = np.empty((nq, k), dtype=np.float32)
    w, o = (None, None) if weights is None else (f32(weights), np.asarray(occurs, dtype=np.uint8))
    g, t = (None, None) if groups is None else (u32(groups), f32(ties))
    opt = lambda a, p: None if a is None else p(a)      # noqa: E731
    dev = arr._device()
    with arr._shared["lock"]:
        dev.sync_features(arr.host)
        rc = _lib.lib().sa_score_batch_topk_bool(
            dev.handle, nq, _lib.p_u32(starts), None, _lib.p_u32(terms), _lib.p_u32(term_starts), _lib.p_f32(idf),
            opt(w, _lib.p_f32), opt(o, _lib.p_u8), opt(g, _lib.p_u32), opt(t, _lib.p_f32), _lib.p_u32(mm), nq, 0,
            arr.avg_doc_length, 1.2, 0.75, k, None, 0, 0, _lib.p_u32(docs), _lib.p_f32(scores), None,
            0, None, None, None, None)
    return rc, docs, scores


def test_c_abi_errors_leave_the_index_usable():
    from searcharray_b200 import Bool, Feature, SearchArray, _lib
    from searcharray_b200.similarity import compute_idf
    host, names = synth_corpus()
    arr = SearchArray.from_host_index(host)
    cols = feature_columns()
    arr.set_feature("pop", cols["pop"])            # slot 0
    w1 = host.term_dict.get_term_id("w1")
    idf_w1 = np.float32(compute_idf(arr.corpus_size, np.asarray([arr.docfreq("w1")])))
    base = 0xFF000000

    def good():
        rc, docs, scores = _c_call(arr, None, [0, 2], [w1, base | 1 << 8], [0, 1, 2], [idf_w1, 50.0])
        assert rc == 0, _lib.lib().sa_last_error()
        want = arr.search_topk([Bool(should=["w1", Feature("pop", "saturation", pivot=50)])], k=10)
        assert np.array_equal(docs, want[0]) and np.array_equal(scores.view(np.uint32), want[1].view(np.uint32))
    good()                                          # Or / And arrays (NULL roles): the promotion
    bad = [([w1, base | 3], [0, 1, 2], [idf_w1, 0.0]),                   # slot 3 is not set
           ([w1, base | 3 << 8], [0, 1, 2], [idf_w1, 1.0]),              # no function 3
           ([w1, base | 0xFF << 8], [0, 1, 2], [idf_w1, 1.0]),
           ([w1, w1, base], [0, 2, 3], [idf_w1, 0.0]),                   # fine, then a phrase holding a feature:
           ([w1, base, w1], [0, 1, 3], [idf_w1, 0.0]),
           ([w1, base], [0, 1, 2], [idf_w1, 1.0]),                       # linear takes no parameter
           ([w1, base | 1 << 8], [0, 1, 2], [idf_w1, 0.0]),              # saturation pivot 0
           ([w1, base | 1 << 8], [0, 1, 2], [idf_w1, np.inf]),
           ([w1, base | 2 << 8], [0, 1, 2], [idf_w1, 0.5]),              # log scaling factor < 1
           ([w1, base | 2 << 8], [0, 1, 2], [idf_w1, np.nan])]
    rc, _, _ = _c_call(arr, None, [0, 2], *bad[3])
    assert rc == 0
    for i, args in enumerate(bad):
        if i == 3:
            continue
        rc, _, _ = _c_call(arr, None, [0, 2], *args)
        assert rc == 2, (i, args)
        good()
    # a feature as a member of a DisMax group of two
    rc, _, _ = _c_call(arr, None, [0, 2], [w1, base], [0, 1, 2], [idf_w1, 0.0], weights=[1, 1], occurs=[0, 0],
                       groups=[0, 0], ties=[0.1, 0.1])
    assert rc == 2
    good()
    # sa_index_set_feature: slot, length, NaN, inf, negative
    dev = arr._device()
    v = cols["frac"].copy()
    for slot, vals in ((16, v), (1, v[:-1]), (1, np.append(v, 1).astype(np.float32))):
        assert _lib.lib().sa_index_set_feature(dev.handle, slot, _lib.p_f32(vals), len(vals)) == 2
        good()
    for x in (np.nan, np.inf, -1.0):
        vals = v.copy()
        vals[123] = x
        assert _lib.lib().sa_index_set_feature(dev.handle, 0, _lib.p_f32(vals), len(vals)) == 2
        good()                                      # slot 0 still holds pop
    # the other entry points treat a reserved id as the out-of-range id it is
    out = np.empty(arr.corpus_size, dtype=np.float32)
    assert _lib.lib().sa_score_term(dev.handle, base, 1.0, arr.avg_doc_length, 1.2, 0.75, 0, _lib.ALL_BITS,
                                    _lib.p_f32(out)) == 2


def test_two_million_docs():
    """A 2M-doc seeded corpus (many tiles, a feature with ~80 % of docs non-zero) for a handful of queries."""
    from searcharray_b200 import And, Bool, Boost, Feature, Or, SearchArray
    from searcharray_b200.indexing import index_from_term_postings
    from searcharray_b200.roaringish import encode_postings
    n = 2_000_000
    rng = np.random.default_rng(2024)
    names, words = [], []
    for name, p in (("a", 0.2), ("b", 0.05), ("c", 0.01), ("d", 0.3)):
        docs = np.flatnonzero(rng.random(n) < p)
        posns = rng.integers(0, 50, len(docs))
        names.append(name)
        words.append(encode_postings(docs, posns))
    host = index_from_term_postings(names, words, rng.integers(5, 80, n).astype(np.float32))
    arr = SearchArray.from_host_index(host)
    arr.set_feature("pop", np.where(rng.random(n) < 0.8, rng.integers(1, 10000, n), 0).astype(np.float32))
    arr.set_feature("rank", (rng.random(n) * 3).astype(np.float32))
    qs = [Bool(must=[Or(["a", "b"])], should=[Boost(Feature("pop", "saturation", pivot=500), 2)]),
          Or(["c", Feature("pop", "log", scaling_factor=1)]),
          Bool(must=["b"], should=[Feature("rank"), Feature("pop", "log", scaling_factor=4)]),
          Or([And(["a", "d"]), Feature("rank", "saturation", pivot=1)], mm=2)]
    check(arr, qs, 10, "2M")
    check(arr, qs, 10, "2M where", where=rng.random(n) < 0.1)
