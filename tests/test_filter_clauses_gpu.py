"""GPU: range and code-set filter clauses (query.Range over feature columns, query.In over facet columns; the range
and In paths of bool_tile's FEATURE instances and bool_docs_kernel in sa_bool.cu, and the tile bounds and code sets of
sa_feature.cu).

The main check is equivalence with `where=`: Bool(must=[q], filter=[Range(...)]) must return, bit for bit, the docs
and score bits of Bool(must=[q]) with the mask Range.match(column) -- a filter adds nothing to a score, so the two
are the same query.  must_not is checked against the complement mask, In against np.isin masks, and the scoring roles
(should / must with Boost, mm, nested) against compose_nested with the clause scored as a constant 1 where it matches.

The corpus is tests/test_bool_topk_gpu.py's five-tile synthetic one.  Its columns: `year` (integers 1950-2020,
~85 % of docs, shuffled), `clus` (increasing with doc id, so whole tiles lie outside a range: presence pruning),
`zero` (no value), `lang` (a facet of 32 codes, ~90 % of docs, shuffled, code 31 present) and `lclus` (codes
clustered by tile)."""

import os

import numpy as np
import pandas as pd
import pytest

from _nested_compose import compose_nested
from _tmdb_index import load_field
from conftest import GOLDEN
from test_bool_fields_gpu import A, B, fb_corpus
from test_bool_topk_gpu import TILE, assert_topk, synth_corpus

pytestmark = pytest.mark.gpu

N = 5 * TILE + 300
KS = (1, 10, 32, 33, 1000, 1024)


def columns(n=N, seed=21):
    rng = np.random.default_rng(seed)
    year = np.where(rng.random(n) < 0.85, rng.integers(1950, 2021, n), 0).astype(np.float32)
    clus = (1 + np.arange(n) // 64).astype(np.float32)          # 1 .. 645, increasing: 128 values per tile
    lang = np.where(rng.random(n) < 0.9, rng.integers(0, 32, n), -1).astype(np.int32)
    lclus = np.minimum(np.arange(n) // TILE, 5).astype(np.int32) * 4 + rng.integers(0, 4, n).astype(np.int32)
    lclus[::97] = -1
    return {"year": year, "clus": clus, "zero": np.zeros(n, dtype=np.float32)}, {"lang": lang, "lclus": lclus}


def setup(arr, n=N, seed=21):
    feats, facets = columns(n, seed)
    for name, v in feats.items():
        arr.set_feature(name, v)
    arr.set_facet("lang", facets["lang"], 32)
    arr.set_facet("lclus", facets["lclus"], 24)
    return feats, facets


class Corpus:
    def __init__(self):
        from searcharray_b200 import SearchArray
        self.host, _ = synth_corpus()
        self.arr = SearchArray.from_host_index(self.host)
        self.feats, self.facets = setup(self.arr)

    def mask(self, c):
        from searcharray_b200 import Range
        return c.match(self.feats[c.name]) if isinstance(c, Range) else c.match(self.facets[c.name])


@pytest.fixture(scope="module")
def corpus():
    return Corpus()


def scorer(arr, feats, facets):
    """score(clause) for compose_nested: .score for text, Feature.apply, and 1 where a Range / In matches."""
    from searcharray_b200 import Feature, In, Range

    def score(c):
        if isinstance(c, Feature):
            return c.apply(feats[c.name])
        if isinstance(c, Range):
            return c.match(feats[c.name]).astype(np.float32)
        if isinstance(c, In):
            return c.match(facets[c.name]).astype(np.float32)
        return arr.score(c)
    return score


def same(a, b, what):
    assert np.array_equal(a[0], b[0]), f"{what}: ids differ"
    assert np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32)), f"{what}: score bits differ"


def base_queries():
    """Every form as the query a filter is added to."""
    from searcharray_b200 import And, Bool, Boost, DisMax, Feature, Or
    return [Or(["w0", "w1", "s1"], mm=2), And(["w0", "w1"]), Or([Boost("w1", 2.5), "w2", "s2"]),
            Bool(must=["w0"], should=[Boost("w1", 0.5)], must_not=["t0"]),
            DisMax(["w0", "w1", "w2"], tie=0.3), Or([And(["w0", "w1"]), Or(["s1", "t3"])]),
            Bool(should=["w1", Feature("year", "saturation", pivot=1990)]),
            Or([["pa", "pb"], "w2"]), Bool(must=[Or(["w1", "s2"])], should=[["pa", "pb"]])]


def filtered(q, filt, role="filter"):
    from searcharray_b200 import Bool
    return Bool(must=[q], **{role: filt})


def test_where_equivalence_every_form(corpus):
    """One filter for the batch and one range per query, against the same masks, for every k."""
    from searcharray_b200 import Bool, Range
    qs = base_queries()
    one = Range("year", gte=1977, lt=1990)
    per = [Range("year", gte=1950 + 5 * i, lte=1960 + 7 * i) for i in range(len(qs))]
    m_one = corpus.mask(one)
    m_per = np.stack([corpus.mask(r) for r in per])
    plain = [Bool(must=[q]) for q in qs]
    for k in KS:
        same(corpus.arr.search_topk([filtered(q, [one]) for q in qs], k=k),
             corpus.arr.search_topk(plain, k=k, where=m_one), f"shared k={k}")
        same(corpus.arr.search_topk([filtered(q, [r]) for q, r in zip(qs, per)], k=k),
             corpus.arr.search_topk(plain, k=k, where=m_per), f"per query k={k}")


@pytest.mark.parametrize("slop", [0, 2])
def test_where_equivalence_in_and_must_not(corpus, slop):
    from searcharray_b200 import Bool, In, Range
    qs = base_queries()
    plain = [Bool(must=[q]) for q in qs]
    ins = [In("lang", [0, 31]), In("lang", [5, 5, 7, 9, 31]), In("lclus", [0, 1, 23]), In("lclus", [9])]
    for i in ins:
        for k in (10, 33):
            same(corpus.arr.search_topk([filtered(q, [i]) for q in qs], k=k, slop=slop),
                 corpus.arr.search_topk(plain, k=k, where=corpus.mask(i), slop=slop), f"{i!r} k={k}")
    for c in (Range("year", gt=1990), In("lang", list(range(0, 32, 2))), Range("clus", lte=300)):
        same(corpus.arr.search_topk([filtered(q, [c], "must_not") for q in qs], k=32, slop=slop),
             corpus.arr.search_topk(plain, k=32, where=~corpus.mask(c), slop=slop), f"must_not {c!r}")
    # two filters and a must_not together
    r, i, x = Range("year", gte=1960, lt=2000), In("lang", list(range(20))), Range("clus", gt=100, lt=400)
    want = corpus.mask(r) & corpus.mask(i) & ~corpus.mask(x)
    got = corpus.arr.search_topk([Bool(must=[q], filter=[r, i], must_not=[x]) for q in qs], k=17, slop=slop)
    same(got, corpus.arr.search_topk(plain, k=17, where=want, slop=slop), "combined")


def test_facets_under_a_filter(corpus):
    from searcharray_b200 import Bool, In, Range
    qs = base_queries()
    plain = [Bool(must=[q]) for q in qs]
    for c in (Range("year", gte=1980, lte=1999), In("lang", [3, 4, 31])):
        d1, s1, h1 = corpus.arr.search_topk([filtered(q, [c]) for q in qs], k=10, facets=["lang", "lclus"])
        d2, s2, h2 = corpus.arr.search_topk(plain, k=10, where=corpus.mask(c), facets=["lang", "lclus"])
        same((d1, s1), (d2, s2), f"facets {c!r}")
        assert np.array_equal(h1.total, h2.total)
        for f in ("lang", "lclus"):
            assert np.array_equal(h1.facets[f], h2.facets[f])


def test_scoring_roles(corpus):
    """Range / In as scoring leaves: 1 where they match, boosted under should / must, counted once by mm, in nested
    queries, against compose_nested."""
    from searcharray_b200 import And, Bool, Boost, In, Or, Range
    r, i = Range("year", gte=1990), In("lang", [1, 2, 3, 30, 31])
    qs = [Bool(should=["w1", Boost(r, 2.0)]), Bool(must=[Boost(i, 0.75)], should=["w2", "s1"]),
          Bool(should=["w1", r, i], mm=2), Or(["w0", r], mm=2), Or([Boost(i, 3), "w2"]),
          Or([And(["w1", r]), Or([i, "t3"], mm=2)]), Bool(must=[Or(["s1", r])], should=[Boost(i, 0.5)]),
          Bool(should=[r]), Bool(must=[Boost(r, 0)], should=["s2"]), Bool(should=[Or([Range("clus", lt=50), "w2"])])]
    score = scorer(corpus.arr, corpus.feats, corpus.facets)
    for k in (1, 10, 32, 100):
        docs, scores = corpus.arr.search_topk(qs, k=k)
        for j, q in enumerate(qs):
            assert_topk(docs[j], scores[j], compose_nested(score, q), k, f"roles {q!r} k={k}")


def test_edges(corpus):
    """0 never matches, even under lte; bounds at stored values; an all-zero column; an empty range."""
    from searcharray_b200 import Bool, Range
    year = corpus.feats["year"]
    q = Bool(should=[Range("year", lte=1960)])
    docs, scores = corpus.arr.search_topk([q], k=1024)
    got = docs[0][docs[0] != 0xFFFFFFFF]
    assert len(got) and (year[got] > 0).all() and (year[got] <= 1960).all() and (scores[0][:len(got)] == 1).all()
    assert len(got) == min(1024, int(((year > 0) & (year <= 1960)).sum()))
    score = scorer(corpus.arr, corpus.feats, corpus.facets)
    edge = [Range("year", gte=1977, lte=1977), Range("year", gt=1977, lt=1979), Range("year", gte=2020),
            Range("year", lt=1951), Range("zero", lte=5), Range("zero", gte=0), Range("year", gte=5, lt=5),
            Range("year", gt=2020), Range("clus", gte=645)]
    qs = [Bool(must=["w0"], filter=[c]) for c in edge] + [Bool(should=[c]) for c in edge]
    docs, scores = corpus.arr.search_topk(qs, k=32)
    for j, q in enumerate(qs):
        assert_topk(docs[j], scores[j], compose_nested(score, q), 32, f"edge {q!r}")
    for j in (4, 5, 6, 7 + len(edge) - 2):
        assert (docs[j] == 0xFFFFFFFF).all(), edge[j % len(edge)]


def test_presence_pruning(corpus):
    """A clustered column lets whole tiles go without reading a list (sa_stats.filter_tiles > 0); a shuffled one
    prunes nothing, and both rank as the mask does."""
    from searcharray_b200 import Bool, In, Range, _lib
    qs = base_queries()
    plain = [Bool(must=[q]) for q in qs]
    handle = corpus.arr._device().handle

    def run(c):
        _lib.check(_lib.lib().sa_stats_reset(handle))
        got = corpus.arr.search_topk([filtered(q, [c]) for q in qs], k=10)
        st = _lib.SaStats()
        _lib.check(_lib.lib().sa_stats_get(handle, st))
        same(got, corpus.arr.search_topk(plain, k=10, where=corpus.mask(c)), repr(c))
        return st.filter_tiles
    assert run(Range("clus", gte=200, lt=300)) > 0            # tiles 1-2 hold clus 129-384
    assert run(In("lclus", [0, 1, 2])) > 0                     # tile 0 only
    assert run(Range("year", gte=1990)) == 0                   # present in every tile
    assert run(In("lang", [7])) == 0


def test_score_docs(corpus):
    from searcharray_b200 import Bool, Boost, In, Or, Range, Rescore
    r, i = Range("year", gte=1970, lt=2001), In("lang", [0, 1, 2, 3, 4, 5, 31])
    qs = [filtered(q, [r]) for q in base_queries()] + [Bool(should=["w1", Boost(r, 2)], must_not=[i]),
                                                      Or([Or(["w0", i], mm=2), "s2"])]
    for k in (10, 1000):
        docs, scores = corpus.arr.search_topk(qs, k=k)
        got = corpus.arr.score_docs(qs, docs)
        assert np.array_equal(got.view(np.uint32), scores.view(np.uint32)), k
    score = scorer(corpus.arr, corpus.feats, corpus.facets)
    rng = np.random.default_rng(4)
    at = rng.integers(0, N, (len(qs), 300)).astype(np.uint32)
    got = corpus.arr.score_docs(qs, at)
    for j, q in enumerate(qs):
        assert np.array_equal(got[j].view(np.uint32), compose_nested(score, q)[at[j]].view(np.uint32)), q
    # a range in the rescore query
    resc = Rescore([Bool(should=[Range("year", gte=2000)], must=["w0"]) for _ in qs[:3]], window=50, rescore_weight=3)
    d, s = corpus.arr.search_topk(qs[:3], k=10, rescore=resc)
    d1, s1 = corpus.arr.search_topk(qs[:3], k=50)
    s2 = corpus.arr.score_docs(resc.queries, d1)
    from searcharray_b200.query import rescore_window
    wd, ws = rescore_window(d1, s1, s2, resc.query_weight, resc.rescore_weight, 10)
    assert np.array_equal(d, wd) and np.array_equal(s.view(np.uint32), ws.view(np.uint32))


def test_fields():
    """Field(column, Range / In) on two columns' indexes, and on a second name of one column."""
    from searcharray_b200 import Bool, Boost, Field, In, Or, Range, SearchArray, fields_score_docs, fields_topk
    ha, _ = synth_corpus()
    hb, _ = fb_corpus()
    frame = pd.DataFrame({A: SearchArray.from_host_index(ha), B: SearchArray.from_host_index(hb)})
    frame["fa2"] = frame[A]
    fa, ca = setup(frame[A].array)
    fb, cb = setup(frame[B].array, seed=22)
    cols = {A: (fa, ca), "fa2": (fa, ca), B: (fb, cb)}

    def score(c):
        feats, facets = cols[c.field]
        if isinstance(c.clause, Range):
            return c.clause.match(feats[c.clause.name]).astype(np.float32)
        if isinstance(c.clause, In):
            return c.clause.match(facets[c.clause.name]).astype(np.float32)
        return frame[c.field].array.score(c.clause)
    r, i = Range("year", gte=1980), In("lang", [2, 3, 31])
    qs = [Bool(must=[Field(A, "w0")], filter=[Field(B, r)]),
          Bool(must=[Field(B, "b1")], filter=[Field("fa2", i)], should=[Boost(Field(A, r), 2)]),
          Or([Field(A, "w1"), Field(B, i), Field("fa2", Range("clus", lt=200))], mm=2),
          Bool(should=[Field(A, "w2"), Field(B, "b2")], must_not=[Field(A, i), Field(B, r)]),
          Or([Bool(must=[Field(A, "s1")], filter=[Field(A, i)]), Field(B, "b2")])]
    for k in (1, 10, 33):
        docs, scores = fields_topk(frame, qs, k=k)
        for j, q in enumerate(qs):
            assert_topk(docs[j], scores[j], compose_nested(score, q), k, f"fields {q!r} k={k}")
        got = fields_score_docs(frame, qs, docs)
        assert np.array_equal(got.view(np.uint32), scores.view(np.uint32))
    at = np.random.default_rng(5).integers(0, N, (len(qs), 200)).astype(np.uint32)
    got = fields_score_docs(frame, qs, at)
    for j, q in enumerate(qs):
        assert np.array_equal(got[j].view(np.uint32), compose_nested(score, q)[at[j]].view(np.uint32)), q


def test_shard_doc_base():
    from searcharray_b200 import Bool, In, Or, Range, SearchArray
    base = 1_000_003
    host, _ = synth_corpus(doc_base=base)
    arr = SearchArray.from_host_index(host, doc_base=base, corpus_size=3_000_000, avg_doc_length=31.5,
                                      global_df=np.asarray([int(host.term_lengths[t]) + 500 for t in range(host.n_terms)],
                                                           dtype=np.uint64))
    feats, facets = setup(arr)
    r, i = Range("clus", gt=150, lte=420), In("lclus", [5, 6, 7, 13])
    qs = [Bool(must=[Or(["w0", "w1"])], filter=[r]), Bool(must=["w0"], filter=[i]), Bool(should=["w2", r, i], mm=2)]
    score = scorer(arr, feats, facets)
    for k in (10, 33):
        docs, scores = arr.search_topk(qs, k=k)
        for j, q in enumerate(qs):
            assert_topk(docs[j], scores[j], compose_nested(score, q), k, f"shard {q!r}", doc_base=base)
        assert np.array_equal(arr.score_docs(qs, docs).view(np.uint32), scores.view(np.uint32))


def test_tmdb():
    """Title and overview queries on the TMDB corpus, filtered by a release year and an original language."""
    from searcharray_b200 import Bool, In, Or, Range, SearchArray
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    fz = np.load(os.path.join(GOLDEN, "tmdb_facets.npz"))
    lang, decade = fz["original_language"], fz["decade"]
    rng = np.random.default_rng(7)
    year = np.where(decade >= 0, int(fz["decade.first"]) + 10 * decade + rng.integers(0, 10, len(decade)), 0)
    year = year.astype(np.float32)
    top = np.bincount(lang[lang >= 0]).argsort()[::-1]
    filters = [Range("year", gte=1977, lt=1990), In("lang", top[:2].tolist()), Range("year", gt=2005),
               In("lang", top[5:40].tolist())]
    for field, terms in (("title_tokens", ["Star", "Wars", "the", "of"]), ("overview_tokens", ["love", "war", "young", "family"])):
        arr = SearchArray.from_host_index(load_field(z, field))
        arr.set_feature("year", year)
        arr.set_facet("lang", lang, int(lang.max()) + 1)
        qs = [Or(terms[:2]), Or(terms), Bool(must=[terms[2]], should=[terms[0]])]
        for c in filters:
            m = c.match(year) if isinstance(c, Range) else c.match(lang)
            for k in (10, 100):
                same(arr.search_topk([filtered(q, [c]) for q in qs], k=k),
                     arr.search_topk([Bool(must=[q]) for q in qs], k=k, where=m), f"tmdb {field} {c!r} k={k}")


def test_two_million_docs():
    from searcharray_b200 import Bool, In, Or, Range, SearchArray
    from searcharray_b200.indexing import index_from_term_postings
    from searcharray_b200.roaringish import encode_postings
    n = 2_000_000
    rng = np.random.default_rng(2025)
    names, words = [], []
    for name, p in (("a", 0.2), ("b", 0.05), ("c", 0.01)):
        docs = np.flatnonzero(rng.random(n) < p)
        names.append(name)
        words.append(encode_postings(docs, rng.integers(0, 50, len(docs))))
    arr = SearchArray.from_host_index(index_from_term_postings(names, words, rng.integers(5, 80, n).astype(np.float32)))
    year = np.where(rng.random(n) < 0.9, rng.integers(1900, 2025, n), 0).astype(np.float32)
    clus = (1 + np.arange(n) // 1000).astype(np.float32)
    lang = rng.integers(-1, 32, n).astype(np.int32)
    arr.set_feature("year", year)
    arr.set_feature("clus", clus)
    arr.set_facet("lang", lang, 32)
    qs = [Or(["a", "b"]), Or(["a", "c"], mm=2), Bool(must=["b"], should=["c"])]
    for c in (Range("year", gte=1977, lt=1990), Range("clus", gt=500, lte=700), In("lang", [0, 5, 31])):
        m = c.match(year if c.name == "year" else clus) if isinstance(c, Range) else c.match(lang)
        for k in (10, 1000):
            same(arr.search_topk([filtered(q, [c]) for q in qs], k=k),
                 arr.search_topk([Bool(must=[q]) for q in qs], k=k, where=m), f"2M {c!r} k={k}")


def _c_call(arr, terms, term_starts, idf, k=10):
    """sa_score_batch_topk_bool on one array, one Or query: (rc, docs, scores)."""
    from searcharray_b200 import _lib
    u32 = lambda x: np.asarray(x, dtype=np.uint32)      # noqa: E731
    starts, terms, term_starts, idf = u32([0, len(term_starts) - 1]), u32(terms), u32(term_starts), \
        np.asarray(idf, dtype=np.float32)
    docs = np.empty((1, k), dtype=np.uint32)
    scores = np.empty((1, k), dtype=np.float32)
    dev = arr._device()
    with arr._shared["lock"]:
        dev.sync_features(arr.host)
        dev.sync_facets(arr.host)
        rc = _lib.lib().sa_score_batch_topk_bool(
            dev.handle, 1, _lib.p_u32(starts), None, _lib.p_u32(terms), _lib.p_u32(term_starts), _lib.p_f32(idf),
            None, None, None, None, _lib.p_u32(u32([1])), 1, 0, arr.avg_doc_length, 1.2, 0.75, k, None, 0, 0,
            _lib.p_u32(docs), _lib.p_f32(scores), None, 0, None, None, None, None)
    return rc, docs, scores


def test_c_abi_errors_leave_the_index_usable():
    from searcharray_b200 import Bool, In, Range, SearchArray, _lib
    from searcharray_b200.similarity import compute_idf
    host, _ = synth_corpus()
    arr = SearchArray.from_host_index(host)
    feats, facets = setup(arr)                     # features year 0, clus 1, zero 2; facets lang 0 (32), lclus 1
    w1 = host.term_dict.get_term_id("w1")
    idf = np.float32(compute_idf(arr.corpus_size, np.asarray([arr.docfreq("w1")])))
    rng_id, in_id = 0xFF001000, 0xFF001100
    bits = lambda x: int(np.float32(x).view(np.uint32))     # noqa: E731
    nan = int(np.float32(np.nan).view(np.uint32))

    def good():
        rc, docs, scores = _c_call(arr, [w1, rng_id, bits(1990), bits(np.inf), in_id, 3, 31], [0, 1, 4, 7],
                                   [idf, 0, 0])
        assert rc == 0, _lib.lib().sa_last_error()
        want = arr.search_topk([Bool(should=["w1", Range("year", gte=1990), In("lang", [3, 31])])], k=10)
        assert np.array_equal(docs, want[0]) and np.array_equal(scores.view(np.uint32), want[1].view(np.uint32))
    good()
    bad = [([w1, rng_id, bits(1)], [0, 1, 3], [idf, 0]),                       # two entries
           ([w1, rng_id, bits(1), bits(2), bits(3)], [0, 1, 5], [idf, 0]),     # four
           ([w1, rng_id], [0, 1, 2], [idf, 0]),                                # one
           ([w1, rng_id, nan, bits(2)], [0, 1, 4], [idf, 0]),                  # NaN bits
           ([w1, rng_id, bits(1), nan], [0, 1, 4], [idf, 0]),
           ([w1, rng_id | 5, bits(1), bits(2)], [0, 1, 4], [idf, 0]),          # feature slot 5 not set
           ([w1, rng_id, bits(1), bits(2)], [0, 1, 4], [idf, 1.0]),            # a parameter
           ([w1, in_id, 32], [0, 1, 3], [idf, 0]),                             # code 32 of 32 buckets
           ([w1, in_id | 1, 3, 24], [0, 1, 4], [idf, 0]),                      # 24 of lclus' 24
           ([w1, in_id], [0, 1, 2], [idf, 0]),                                 # no code
           ([w1, in_id | 2, 0], [0, 1, 3], [idf, 0]),                          # facet slot 2 not set
           ([w1, in_id, 1], [0, 1, 3], [idf, 0.5]),                            # a parameter
           ([w1, 0xFF000000, w1], [0, 1, 3], [idf, 0]),                        # a feature id in a phrase
           ([w1, w1, rng_id, bits(1), bits(2)], [0, 1, 5], [idf, 0])]          # a range id inside a phrase
    for j, args in enumerate(bad):
        rc, _, _ = _c_call(arr, *args)
        assert rc == 2, (j, args)
        good()
