"""GPU: boolean queries in search_topk (sa_score_batch_topk_bool, bool_tile_kernel in sa_bool.cu) against the
composition of the reference's tests (tests/_bool_compose.py): ids and float32 score bits must be equal.

The synthetic corpus spans five 8192-doc tiles and places clause terms on every path of the kernel: terms with
>= 1,024 words have a tile directory and a tf table (records), shorter ones are found by binary search over their
words; `t0` and `t3` live in one tile each, so And / mm > 1 tiles fall on both sides of the pruning test; `pa` /
`pb` make phrases at slop 0 and 2 and a same-term phrase; `hot` / `cold` crowd one tile's best scores into four
threads so that its candidates overflow and the query is re-run exactly."""
import ctypes
import json
import os

import numpy as np
import pytest

from _bool_compose import compose, expand, oracle_score, topk
from _tmdb_index import load_field
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

TILE = 8192
KS = (1, 10, 16, 17, 32)


def assert_topk(docs, scores, dense, k, what, doc_base=0):
    wd, ws = topk(dense, k, doc_base)
    assert np.array_equal(np.asarray(docs, dtype=np.uint32), wd), f"{what}: ids {docs} want {wd}"
    assert np.array_equal(np.asarray(scores, dtype=np.float32).view(np.uint32), ws.view(np.uint32)), \
        f"{what}: score bits {scores} want {ws}"


def synth_corpus(n=5 * TILE + 300, doc_base=0, seed=11):
    from searcharray_b200.indexing import index_from_term_postings
    from searcharray_b200.roaringish import encode_postings
    rng = np.random.default_rng(seed)
    doc_lens = rng.integers(1, 60, n).astype(np.float32)
    postings = {}

    def add(name, docs, posns_of):
        docs = np.sort(np.unique(np.asarray(docs, dtype=np.int64)))
        d, p = [], []
        for doc in docs:
            ps = sorted(set(posns_of(doc)))
            d += [doc] * len(ps)
            p += ps
        postings[name] = (np.asarray(d, dtype=np.int64), np.asarray(p, dtype=np.int64))

    def rand_posns(doc):
        return rng.integers(30, 200, rng.integers(1, 4)).tolist()

    add("w0", np.flatnonzero(rng.random(n) < 0.45), rand_posns)             # tf table
    add("w1", np.flatnonzero(rng.random(n) < 0.2), rand_posns)
    add("w2", rng.choice(n, 1200, replace=False), rand_posns)
    add("s1", rng.choice(3 * TILE, 400, replace=False), rand_posns)         # binary search over words
    add("s2", np.concatenate([rng.choice(np.arange(TILE, 3 * TILE), 200, replace=False),
                              rng.choice(np.arange(4 * TILE, n), 100, replace=False)]), rand_posns)
    add("t0", rng.choice(TILE, 500, replace=False), rand_posns)             # tile 0 only
    add("t3", 3 * TILE + rng.choice(TILE, 600, replace=False), rand_posns)  # tile 3 only
    ph = rng.choice(n, 3000, replace=False)
    add("pa", ph, lambda doc: [10, 11] if doc % 5 == 0 else [10])
    add("pb", ph[: 2000], lambda doc: [11] if doc % 2 else [13])
    # four threads of tile 1 own its best docs (local 4 t + e + 1024 j, t < 4), many others hold lower scores
    hot = TILE + np.asarray([4 * t + e + 1024 * j for t in range(4) for e in range(4) for j in range(8)])
    add("hot", hot, lambda doc: list(range(40, 40 + 2 + doc % 5)))
    cold = np.setdiff1d(TILE + rng.choice(TILE, 1500, replace=False), hot)
    add("cold", cold, lambda doc: [40])
    names = list(postings)
    words = [encode_postings(d + doc_base, p) for d, p in (postings[t] for t in names)]
    return index_from_term_postings(names, words, doc_lens), names


class Synth:
    def __init__(self, **kw):
        from oracle import search as osearch
        from searcharray_b200 import SearchArray
        self.host, self.names = synth_corpus()
        self.arr = SearchArray.from_host_index(self.host, **kw)
        self.oidx = osearch.OracleIndex({t: self.host.term_words(t) for t in range(self.host.n_terms)},
                                        self.host.doc_lens, avg_doc_length=self.host.avg_doc_length)

    def oracle(self, **kw):
        return oracle_score(self.oidx, self.host.term_dict, **kw)


@pytest.fixture(scope="module")
def synth():
    return Synth()


def check_batch(arr, queries, k, score, what, doc_base=0, slop=0, similarity=None):
    """search_topk(queries) against the composition of score(clause) for every boolean query."""
    from searcharray_b200 import bm25_similarity
    sim = similarity or bm25_similarity()
    docs, scores = arr.search_topk(queries, k=k, similarity=sim, slop=slop)
    assert docs.shape == (len(queries), k) and scores.dtype == np.float32
    for i, q in enumerate(queries):
        s, _ = compose(score, q.clauses, q.mm)
        assert_topk(docs[i], scores[i], s, k, f"{what} {q!r} k={k}", doc_base)
    return docs, scores


SYNTH_QUERIES = [
    (["w0", "w1", "w2", "s1"], (0, 1, 2, 3, 4)),
    (["w2", "s1", "s2", "t0", "t3"], (1, 2, 3)),
    (["t0", "w0"], (2,)), (["t0", "t3"], (1, 2)), (["t3", "s2", "w2"], (3,)),
    (["w1", "w1", "s2"], (1, 2, 3)),                          # duplicates count twice
    (["zzz", "w2"], (1, 2)), (["zzz", "yyy"], (0, 1)),      # unknown tokens, a query of unknown tokens only
    (["s1", "w0", "w2", "w1", "s2", "t0"], (1, 4)),          # fold order over six clauses
]


@pytest.mark.parametrize("k", KS)
def test_synth_terms(synth, k):
    """Term clauses on the tf-table and words paths, mm 0 .. C and And, pruned and unpruned tiles, duplicates and
    unknown tokens, against the oracle."""
    from searcharray_b200 import And, Or
    queries = [Or(c, mm=m) for c, ms in SYNTH_QUERIES for m in ms] + [And(c) for c, _ in SYNTH_QUERIES]
    check_batch(synth.arr, queries, k, synth.oracle(), "synth")


@pytest.mark.parametrize("slop", [0, 2])
def test_synth_phrases(synth, slop):
    """Phrase clauses (count rows) next to term clauses, a same-term phrase, phrases with an unknown token."""
    from searcharray_b200 import And, Or
    queries = [Or([["pa", "pb"], "w2"]), Or([["pa", "pb"], "w2"], mm=2), And([["pa", "pa"], "w0"]),
               Or([["pa", "pa"], ["pa", "pb"], "s1"], mm=1), Or([["pa", "zzz"], "t0"]), Or([["pa", "pb"]]),
               And([["pa", "pb"], ["pb", "pa"]]), Or([["w0", "w1"], ["pa", "pb"], "w1", "t3"], mm=2)]
    for k in (1, 10, 32):
        check_batch(synth.arr, queries, k, synth.oracle(slop=slop), f"synth slop={slop}", slop=slop)


def test_overflow_rerun(synth):
    """A tile whose best docs sit in four threads overflows its candidate slots: the query is re-run exactly."""
    from searcharray_b200 import Or
    queries = [Or(["hot", "cold"]), Or(["hot", "cold", "w0"], mm=1), Or(["w2"])]
    for k in (10, 16):
        docs, scores, n_redone = synth.arr._search_topk_bool(queries, k, __import__("searcharray_b200").bm25_similarity(), 0)
        assert n_redone > 0
        for i, q in enumerate(queries):
            s, _ = compose(synth.oracle(), q.clauses, q.mm)
            assert_topk(docs[i], scores[i], s, k, f"overflow {q!r} k={k}")


def test_same_as_plain_queries(synth):
    """Or(["t"]) and Or([["a", "b"]]) give search_topk("t") / search_topk([["a", "b"]])'s bits; a mixed batch
    equals its parts answered separately."""
    from searcharray_b200 import And, Or
    arr = synth.arr
    plain = ["w0", "s1", ["pa", "pb"], "zzz", "t3"]
    for k in (1, 10, 32):
        want_d, want_s = arr.search_topk(plain, k=k)
        got_d, got_s = arr.search_topk([Or([p]) for p in plain], k=k)
        assert np.array_equal(got_d, want_d) and np.array_equal(got_s.view(np.uint32), want_s.view(np.uint32))
        mixed = ["w1", Or(["w0", "t0"], mm=2), ["pa", "pb"], And(["s1", "w2"]), "t3"]
        d, s = arr.search_topk(mixed, k=k)
        pd_, ps = arr.search_topk(["w1", ["pa", "pb"], "t3"], k=k)
        bd, bs = arr.search_topk([mixed[1], mixed[3]], k=k)
        assert np.array_equal(d[[0, 2, 4]], pd_) and np.array_equal(s[[0, 2, 4]].view(np.uint32), ps.view(np.uint32))
        assert np.array_equal(d[[1, 3]], bd) and np.array_equal(s[[1, 3]].view(np.uint32), bs.view(np.uint32))


def test_launches_do_not_depend_on_q(synth):
    """A term-only boolean batch is one tile launch and one select, whatever the number of queries."""
    from searcharray_b200 import Or, _lib
    arr = synth.arr
    h = arr._device().handle
    launches = []
    for nq in (1, 4, 64):
        queries = [Or(["w0", "w1", "s1"], mm=1 + i % 3) for i in range(nq)]
        arr.search_topk(queries, k=10)                      # warm: the norm table for these parameters
        _lib.check(_lib.lib().sa_stats_reset(h))
        arr.search_topk(queries, k=10)
        st = _lib.SaStats()
        _lib.check(_lib.lib().sa_stats_get(h, ctypes.byref(st)))
        launches.append(st.total_launches)
    assert launches[0] == launches[1] == launches[2] == 2, launches


def test_shard_doc_base_global_df():
    """A shard (doc_base, global corpus size, avgdl, dfs): global ids, each clause scored as the shard's .score."""
    from searcharray_b200 import And, Or, SearchArray
    base = 1_000_003
    local, names = synth_corpus()
    host, _ = synth_corpus(doc_base=base)
    gdf = np.asarray([int(local.term_lengths[i]) + 1000 * (i + 1) for i in range(len(names))], dtype=np.uint64)
    arr = SearchArray.from_host_index(host, doc_base=base, corpus_size=3_000_000, avg_doc_length=31.5, global_df=gdf)
    queries = [Or(["w0", "w2", "s1"]), Or(["w0", "w2", "s1"], mm=2), And(["t0", "w0"]), Or([["pa", "pb"], "s2"])]
    for k in (1, 10, 32):
        check_batch(arr, queries, k, lambda c: arr.score(c), "shard", doc_base=base)


def test_avg_doc_length_zero():
    from searcharray_b200 import Or, SearchArray
    host, _ = synth_corpus()
    arr = SearchArray.from_host_index(host, avg_doc_length=0)
    docs, scores = arr.search_topk([Or(["w0", "w1"]), Or([["pa", "pb"]])], k=10)
    assert np.all(docs == 0xFFFFFFFF) and np.all(scores == 0)


@pytest.mark.parametrize("k1, b", [(0.0, 0.75), (1.2, 1.0), (1.2, 1.5)])
def test_exotic_parameters(synth, k1, b):
    """Term-only queries under parameters that are not sparse-safe: every doc's BM25 is evaluated as the
    ALL_DOCS scan does; bits equal to the composition of .score, whose scores meet the oracle's under the 1e-5
    contract with the same NaN mask.  Phrase clauses are refused there."""
    from searcharray_b200 import Or, bm25_similarity, _lib
    sim = bm25_similarity(k1=k1, b=b)
    arr = synth.arr
    oracle = synth.oracle(k1=k1, b=b)
    for name in ("w0", "s1", "zzz"):
        got, want = arr.score(name, similarity=sim), oracle(name)
        assert np.array_equal(np.isnan(got), np.isnan(want))
        ok = ~np.isnan(want)
        np.testing.assert_allclose(got[ok], want[ok], rtol=1e-5, atol=0)
    queries = [Or(["w0", "s1"]), Or(["w0", "s1", "t0"], mm=2), Or(["zzz", "w2"]), Or(["s2"], mm=0)]
    for k in (1, 10, 32):
        check_batch(arr, queries, k, lambda c: arr.score(c, similarity=sim), f"k1={k1} b={b}", similarity=sim)
    with pytest.raises(_lib.SearchArrayB200Error, match="ordinary BM25 parameters"):
        arr.search_topk([Or([["pa", "pb"], "w0"])], k=10, similarity=sim)


def test_phrase_rows_span_two_groups():
    """~2M docs: a batch with more phrase clauses than one ~4 GB group of rows holds (512 rows of 8 MB)."""
    from searcharray_b200 import Or, SearchArray
    from searcharray_b200.indexing import index_from_term_postings
    from searcharray_b200.roaringish import encode_postings
    rng = np.random.default_rng(5)
    n = 2_000_000
    docs = np.sort(rng.choice(n, 20000, replace=False))
    pa = encode_postings(docs, np.full(len(docs), 3))
    pb_docs = docs[::2]
    pb = encode_postings(pb_docs, np.full(len(pb_docs), 4))
    x_docs = np.sort(rng.choice(n, 50000, replace=False))
    x = encode_postings(x_docs, np.full(len(x_docs), 7))
    host = index_from_term_postings(["pa", "pb", "x"], [pa, pb, x], rng.integers(1, 30, n).astype(np.float32))
    arr = SearchArray.from_host_index(host)
    queries = [Or([["pa", "pb"]] * 63 + ["x"], mm=1 + i % 2) for i in range(9)]   # 567 phrase rows
    check_batch(arr, queries, 10, lambda c: arr.score(c), "2M docs")


@pytest.fixture(scope="module")
def fixture():
    with open(os.path.join(GOLDEN, "bool_scenarios.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("kind", ["and", "or"])
def test_reference_scenarios(fixture, kind):
    """The reference's and/or scenarios: the top k of the composed scores, inside the expected mask, equal to the
    real reference's composed top 10."""
    from searcharray_b200 import Or, SearchArray
    for rec in fixture[kind]:
        arr = SearchArray.index(expand(rec["docs"]))
        expected = np.asarray(expand(rec["expected"]))
        q = Or(rec["clauses"], mm=rec["mm"])
        for k in KS:
            docs, scores = check_batch(arr, [q], k, lambda c: arr.score(c), rec["name"])
            got = docs[0][docs[0] != 0xFFFFFFFF]
            assert np.all(expected[got.astype(np.int64)]), rec["name"]
        docs, scores = arr.search_topk([q], k=10)
        n = len(rec["top_ids"])
        assert docs[0][:n].tolist() == rec["top_ids"] and scores[0][:n].view(np.uint32).tolist() == rec["top_bits"]


def test_tmdb(fixture):
    """The real reference's composed TMDB top 10, ids and score bits."""
    from searcharray_b200 import Or, SearchArray
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    arrs = {f: SearchArray.from_host_index(load_field(z, f)) for f in ("title_tokens", "overview_tokens")}
    for field in arrs:
        recs = [r for r in fixture["tmdb"] if r["field"] == field]
        docs, scores = arrs[field].search_topk([Or(r["clauses"], mm=r["mm"]) for r in recs], k=10)
        for i, r in enumerate(recs):
            n = len(r["top_ids"])
            what = f"{field} {r['clauses']} mm={r['mm']}"
            assert docs[i][:n].tolist() == r["top_ids"], what
            assert scores[i][:n].view(np.uint32).tolist() == r["top_bits"], what
            assert np.all(docs[i][n:] == 0xFFFFFFFF), what
