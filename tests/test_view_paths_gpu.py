"""GPU: every branch of the view and similarity top-k (sa_score_batch_topk_sim in sa_view.cu, through search_topk on
a view and under bm25_impact, bm25_legacy_similarity and classic_similarity) and of the view machinery of sa_filter.cu
(the row-filter compaction with and without the min/max-posn payload test, docfreq_rows_kernel) against the CPU oracle.

The expected vectors are composed from oracle.search and oracle.similarity alone, never from the library:
- counts: OracleIndex.sliced(key).termfreqs for views whose rows are sorted and distinct; for fancy and repeated-row
  keys the counts of the sorted distinct rows u, gathered per position with np.searchsorted(u, rows) (the oracle's
  np.isin assignment would misplace them on unsorted rows);
- document frequencies: the slice's docfreq (on repeated rows a doc counts once), a shard's global ones;
- scores: oracle.similarity with the view's own doc lengths, the parent's avgdl and corpus size; BM25 through
  OracleIndex.score, which carries the stepped-slice doc-length quirk;
- where=: the masked-out positions zeroed; ranking: the top k by (score desc, position asc) over scores > 0.
Ids and score bits are compared exactly, in the similarity's dtype (float32 BM25 and impact, float64 legacy and
classic).  sa_stats.sim_instances names the tile kernels a call launched (bit 2 * kind + masked) and every call asserts
the exact set; test_every_instance_ran asserts that the module's calls cover all 8.

The parent has 9 full tiles and a partial one, so docfreq_rows_kernel's records branch has a full 8-tile job and a
partial one.  tests/_view_paths_worker.py repeats the document-frequency and term checks with SA_NO_TF_TABLE=1, where
every list takes the words branch, including a 9,001-word list whose doc at list indices 4095 and 4096 straddles a
4,096-word job boundary."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TILE = 8192
N = 9 * TILE + 777
KS = (1, 2, 10, 11, 16, 17, 32)             # the candidate slots switch from 128 to 256 between 16 and 17
IMPACT, LEGACY, CLASSIC, BM25 = range(4)     # SA_SIM_*
KIND_NAMES = {IMPACT: "impact", LEGACY: "legacy", CLASSIC: "classic", BM25: "bm25"}
NO_DOC = 0xFFFFFFFF
RAN = set()                                  # sim_instances bits seen by this module's calls
STRADDLE_AT = 4095                           # the list index of the straddling doc's first word


def bit(kind, masked):
    return 1 << (2 * kind + masked)


# ------------------------------------------------------------------------------------------------------------ corpus
def _host(postings, doc_lens, doc_base=0):
    from searcharray_b200.indexing import index_from_term_postings
    from searcharray_b200.roaringish import encode_postings
    names = list(postings)
    words = [encode_postings(np.asarray(d, dtype=np.int64) + doc_base, np.asarray(p, dtype=np.int64))
             for d, p in (postings[t] for t in names)]
    return index_from_term_postings(names, words, np.asarray(doc_lens, dtype=np.float32))


def _add(postings, name, docs, posns_of):
    d, p = [], []
    for doc in np.unique(np.asarray(docs, dtype=np.int64)):
        ps = sorted(set(posns_of(int(doc))))
        d += [doc] * len(ps)
        p += ps
    postings[name] = (d, p)


def corpus_postings(n=N, seed=17):
    """(postings, doc lengths) of the parent.  r0 / r1 / edge: tf records; s0 / s1: short lists (binary search,
    no tf table); pa / pb: long phrase terms (several filter chunks each), pa twice in every fifth doc; qa / qb: a
    phrase in blocks 0-3 for the min / max-posn filter; fNNNN: exactly NNNN words, one per doc, in block doc % 3;
    straddle: 9,001 words, its 4,096th doc holding the words at list indices 4095 and 4096; edge: docs at 0,
    8191 / 8192, tile 7 and the last doc."""
    rng = np.random.default_rng(seed)
    doc_lens = rng.integers(1, 60, n).astype(np.float32)
    doc_lens[rng.random(n) < 0.03] = 0                              # counts > 0 at length 0: classic gives +inf
    post = {}

    def rand_posns(doc):
        return rng.integers(30, 200, rng.integers(1, 4)).tolist()
    _add(post, "r0", np.flatnonzero(rng.random(n) < 0.45), rand_posns)
    _add(post, "r1", np.flatnonzero(rng.random(n) < 0.12), rand_posns)
    _add(post, "s0", rng.choice(n, 300, replace=False), lambda d: [40 + d % 7])
    _add(post, "s1", rng.choice(n, 150, replace=False), lambda d: [50, 51 + d % 5])
    edges = [0, TILE - 1, TILE, 7 * TILE + 5, 8 * TILE - 1, n - 1]
    _add(post, "edge", np.concatenate([edges, rng.choice(n, 1500, replace=False)]), lambda d: [60 + d % 3])
    ph = rng.choice(n, 6000, replace=False)
    _add(post, "pa", ph, lambda d: [10, 11] if d % 5 == 0 else [10])
    _add(post, "pb", ph[:4000], lambda d: [11] if d % 2 else [12])
    qd = rng.choice(n, 3000, replace=False)
    blocks = {int(d): np.flatnonzero(rng.random(4) < 0.6).tolist() or [1] for d in qd}
    _add(post, "qa", qd, lambda d: [18 * b + 3 for b in blocks[d]])
    _add(post, "qb", qd, lambda d: [18 * b + 4 for b in blocks[d] if (b + d) % 3])
    for m in (2047, 2048, 2049, 5000):
        _add(post, f"f{m}", rng.choice(n, m, replace=False), lambda d: [18 * (d % 3) + d % 7])
    sd = np.sort(rng.choice(n, 9000, replace=False))
    _add(post, "straddle", sd, lambda d: [0, 18] if d == sd[STRADDLE_AT] else [5])
    return post, doc_lens


def view_keys(n=N):
    rng = np.random.default_rng(5)
    keys = {"unsliced": None}
    for length, start in ((0, 100), (1, 8191), (31, 8180), (32, 0), (33, n - 33), (8191, 1), (8192, 8192),
                          (8193, 5000), (16385, 3 * TILE + 7)):
        keys[f"len{length}"] = slice(start, start + length)
    keys.update({
        "stepped": slice(1, None, 3),
        "mask": rng.random(n) < 0.3,
        "fancy": rng.permutation(n)[:20_000],
        "repeats": rng.integers(0, n, 25_000),
        "view_of_view": (rng.random(n) < 0.5, slice(1_000, 30_000)),
        "edges": np.asarray([0, TILE - 1, TILE, 7 * TILE + 5, 8 * TILE - 1, n - 1, 3, 5 * TILE]),
    })
    return keys


VIEWS = view_keys()
UNSORTED = {"fancy", "repeats", "edges", "flood"}


def make_view(arr, key):
    if key is None:
        return arr
    if isinstance(key, tuple):
        return arr[key[0]][key[1]]
    return arr[key]


def view_rows(n, key):
    """The parent rows of a view's positions, in view order."""
    if key is None:
        return np.arange(n)
    if isinstance(key, tuple):
        return np.arange(n)[key[0]][key[1]]
    return np.arange(n)[key]


class Oracle:
    """Dense vectors of oracle.search / oracle.similarity over a parent's views.  shard: (corpus size, global dfs)."""

    def __init__(self, host, avgdl, shard=None):
        from oracle import search as osearch
        self.host, self.avgdl, self.shard = host, avgdl, shard
        self.n = host.n_docs
        self.corpus = self.n if shard is None else shard[0]
        self.oidx = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                                        avg_doc_length=avgdl, corpus_size=self.corpus, max_doc_id=self.n - 1)
        self.views, self.cache = {}, {}

    def tids(self, q):
        return [self.host.term_dict.term_to_ids.get(t) for t in ([q] if isinstance(q, str) else q)]

    def view(self, vname, key):
        """(oracle view to count on, gather index or None, the view's parent rows)."""
        if vname not in self.views:
            rows = view_rows(self.n, key)
            if vname in UNSORTED:
                u = np.unique(rows)
                self.views[vname] = (self.oidx.sliced(u), np.searchsorted(u, rows), rows)
            elif key is None:
                self.views[vname] = (self.oidx, None, rows)
            elif isinstance(key, tuple):
                self.views[vname] = (self.oidx.sliced(key[0]).sliced(key[1]), None, rows)
            else:
                self.views[vname] = (self.oidx.sliced(key), None, rows)
        return self.views[vname]

    def counts(self, vname, key, q, slop=0, min_posn=None, max_posn=None):
        ck = ("tf", vname, repr(q), slop, min_posn, max_posn)
        if ck not in self.cache:
            ov, gather, rows = self.view(vname, key)
            ids = self.tids(q)
            if len(rows) == 0:
                self.cache[ck] = np.zeros(0, dtype=np.float32)
                return self.cache[ck]
            c = ov.termfreqs(ids[0] if isinstance(q, str) else ids, slop=slop, min_posn=min_posn, max_posn=max_posn)
            self.cache[ck] = np.asarray(c if gather is None else c[gather], dtype=np.float32)
        return self.cache[ck]

    def dfs(self, vname, key, q):
        ov, _, _ = self.view(vname, key)
        if self.shard is not None:
            return [0 if t is None else int(self.shard[1][t]) for t in self.tids(q)]
        return [ov.docfreq(t) for t in self.tids(q)]

    def dense(self, vname, key, q, kind, sim, slop=0):
        """The vector .score(q, similarity=sim, slop=slop) returns on the view, composed from the oracle."""
        from oracle import search as osearch
        from oracle import similarity as osim
        ck = ("s", vname, repr(q), slop, kind, repr(sim))
        if ck in self.cache:
            return self.cache[ck]
        ov, gather, rows = self.view(vname, key)
        tf = self.counts(vname, key, q, slop)
        dfs = self.dfs(vname, key, q)
        dl = self.host.doc_lens[rows]
        if len(rows) == 0:
            v = np.zeros(0)
        elif kind == BM25:
            if gather is None:
                ids = self.tids(q)
                v = ov.score(ids[0] if isinstance(q, str) else ids, k1=sim.k1, b=sim.b, slop=slop)
            else:                                        # fancy keys: the view's own lengths (no stepped quirk)
                v = osearch.bm25(tf.copy(), dfs, dl, self.avgdl, self.corpus, sim.k1, sim.b)
        elif kind == IMPACT:
            v = osim.bm25_impact(tf, dfs, dl, self.avgdl, self.corpus, k1=sim.k1, b=sim.b)
        elif kind == LEGACY:
            v = osim.bm25_legacy(tf, dfs, dl, self.avgdl, self.corpus, k1=sim.k1, b=sim.b)
        else:
            v = osim.classic(tf, dfs, dl, self.avgdl, self.corpus)
        self.cache[ck] = np.asarray(v).astype(sim.out_dtype)
        return self.cache[ck]


def sim_of(kind, **kw):
    from searcharray_b200 import bm25_impact, bm25_legacy_similarity, bm25_similarity, classic_similarity
    return {IMPACT: bm25_impact, LEGACY: bm25_legacy_similarity, CLASSIC: lambda: classic_similarity(),
            BM25: bm25_similarity}[kind](**kw)


class Ctx:
    def __init__(self):
        from searcharray_b200 import SearchArray
        post, dl = corpus_postings()
        self.post, self.doc_lens = post, dl
        self.host = _host(post, dl)
        self.arr = SearchArray.from_host_index(self.host)
        self.oracle = Oracle(self.host, self.arr.avg_doc_length)


@pytest.fixture(scope="module")
def ctx():
    return Ctx()


# ------------------------------------------------------------------------------------------------------------ checks
def topk(dense, k, doc_base=0):
    """(ids, scores) of the top k of dense, in its dtype: (score desc, position asc) over the scores > 0."""
    dense = np.asarray(dense)
    nz = np.flatnonzero(dense > 0)
    order = nz[np.lexsort((nz, -dense[nz].astype(np.float64)))][:k]
    docs = np.full(k, NO_DOC, dtype=np.uint32)
    scores = np.zeros(k, dtype=dense.dtype)
    docs[:len(order)] = order + doc_base
    scores[:len(order)] = dense[order]
    return docs, scores


def bits_of(a):
    return np.asarray(a).view(np.uint64 if np.asarray(a).dtype == np.float64 else np.uint32)


def stats(arr):
    from searcharray_b200 import _lib
    st = _lib.SaStats()
    _lib.check(_lib.lib().sa_stats_get(arr._device().handle, ctypes.byref(st)))
    return st


def reset(arr):
    from searcharray_b200 import _lib
    _lib.check(_lib.lib().sa_stats_reset(arr._device().handle))


def run(view, queries, k, sim, slop=0, where=None):
    """(docs, scores, sa_stats) of one search_topk call."""
    reset(view)
    docs, scores = view.search_topk(queries, k=k, similarity=sim, slop=slop, where=where)
    st = stats(view)
    RAN.update(i for i in range(8) if st.sim_instances >> i & 1)
    return docs, scores, st


def check(view, queries, k, sim, kind, want_dense, what, slop=0, where=None, want_bits=None, doc_base=0):
    """One call against want_dense(i) per query: ids, score bits and dtype, and the exact sim_instances."""
    docs, scores, st = run(view, queries, k, sim, slop, where)
    assert docs.shape == (len(queries), k) and docs.dtype == np.uint32 and scores.dtype == sim.out_dtype, what
    if want_bits is None:
        masked = 0 if where is None else 1
        want_bits = 0 if len(view) == 0 else bit(kind, masked)
    assert st.sim_instances == want_bits, f"{what} k={k}: sim_instances {st.sim_instances:#x} want {want_bits:#x}"
    for i, q in enumerate(queries):
        dense = want_dense(i)
        if where is not None:
            m = np.asarray(where)
            dense = np.where(m[i] if m.ndim == 2 else m, dense, dense.dtype.type(0)).astype(dense.dtype)
        wd, ws = topk(dense, k, doc_base)
        tag = f"{what} #{i} {q!r} k={k}"
        assert np.array_equal(docs[i], wd), f"{tag}: ids {docs[i]} want {wd}"
        assert np.array_equal(bits_of(scores[i]), bits_of(ws)), f"{tag}: score bits {scores[i]} want {ws}"
    return st, docs


def query_masks(n_queries, n, seed):
    """Per-query masks: random docs; nothing; everything; every position past the first tile; a random 1 in 8."""
    rng = np.random.default_rng(seed)
    out = np.zeros((n_queries, n), dtype=bool)
    for i in range(n_queries):
        kind = i % 5
        if kind == 0:
            out[i] = rng.random(n) < 0.6
        elif kind == 2:
            out[i] = True
        elif kind == 3:
            out[i, TILE:] = True
        elif kind == 4:
            out[i] = rng.random(n) < 0.125
    return out


# a batch that mixes terms and phrases with a phrase first, so that the row order (terms, then phrases) differs from
# the query order: repeated terms, missing terms and a phrase whose terms are all missing
BATCH = [["pa", "pb"], "r0", ["pa", "pa", "pb"], "s0", ["qa", "qb"], "edge", ["pa", "zzz"], "r1", ["zzz", "yyy"],
         "s1", ["r0", "r1"], "zzz", "f5000"]
KIND_VIEWS = [(kind, v) for kind in (IMPACT, LEGACY, CLASSIC, BM25) for v in VIEWS if not (kind == BM25 and v == "unsliced")]


def check_kind_view(ctx, kind, vname, queries=BATCH, slops=(0, 2), ks=KS):
    key = VIEWS[vname]
    view = make_view(ctx.arr, key)
    sim = sim_of(kind)
    n = len(view)
    shared = np.random.default_rng(3).random(n) < 0.55
    per_query = query_masks(len(queries), n, 4)
    for slop in slops:
        def want(i, slop=slop):
            return ctx.oracle.dense(vname, key, queries[i], kind, sim, slop)
        wheres = (None, shared, per_query) if slop == 0 else (None, per_query)
        for where in wheres:
            for k in ks:
                check(view, queries, k, sim, kind, want, f"{KIND_NAMES[kind]} {vname} slop={slop} "
                      f"where={'none' if where is None else where.ndim}", slop, where)


@pytest.mark.parametrize("kind, vname", KIND_VIEWS)
def test_kind_view(ctx, kind, vname):
    """Each kind with and without where= (one mask, a mask per query) on every view shape, for terms with and without a
    tf table, phrases at slop 0 and 2 with repeated and missing terms."""
    check_kind_view(ctx, kind, vname)


def test_all_missing_phrases_skip_the_filter(ctx):
    """A batch whose phrases all miss a term filters no list: the only launches are a tile pass per query, the select
    and, when a phrase has a known term, the one document-frequency pass of the view."""
    view = ctx.arr[VIEWS["mask"]]
    for qs, df_pass in (([["zzz", "yyy"], ["qqq", "zzz", "qqq"]], 0), ([["zzz", "pa"], ["pb", "yyy"], ["zzz", "yyy"]], 1)):
        for kind in (IMPACT, BM25):
            sim = sim_of(kind)
            for k in KS:
                st, _ = check(view, qs, k, sim, kind, lambda i: np.zeros(len(view), dtype=sim.out_dtype), "all missing")
                assert st.topk_kernel_launches == len(qs) + 1 and st.total_launches == len(qs) + 1 + df_pass, \
                    (qs, st.total_launches, st.topk_kernel_launches)


@pytest.mark.parametrize("kind, k1, b", [(IMPACT, 0.0, 0.75), (IMPACT, -0.5, 0.75), (IMPACT, 1.2, 1.0),
                                         (LEGACY, 0.0, 1.0), (LEGACY, -1.5, 0.3), (BM25, 0.0, 0.75),
                                         (BM25, 1.2, 1.5)])
def test_exotic_parameters(ctx, kind, k1, b):
    """k1 / b where a zero count scores NaN or -0 in .score (never ranked), and negative or +inf scores."""
    sim = sim_of(kind, k1=k1, b=b)
    qs = ["r0", "s0", ["pa", "pb"], "edge", "zzz"]
    for vname in ("mask", "fancy", "stepped") + (() if kind == BM25 else ("unsliced",)):
        key = VIEWS[vname]
        view = make_view(ctx.arr, key)
        for k in KS:
            check(view, qs, k, sim, kind, lambda i: ctx.oracle.dense(vname, key, qs[i], kind, sim), f"exotic {vname}")
    if k1 == 0.0:
        assert np.isnan(ctx.oracle.dense("mask", VIEWS["mask"], "r0", kind, sim)).any()


def test_avgdl_zero_and_infinite_classic(ctx):
    """avg_doc_length == 0: legacy, impact and BM25 rank nothing (and launch no tile pass), classic ranks; a count > 0
    at doc length 0 scores +inf under classic."""
    from searcharray_b200 import SearchArray
    zero = SearchArray.from_host_index(ctx.host, avg_doc_length=0.0)
    oz = Oracle(ctx.host, 0.0)
    qs = ["r0", ["pa", "pb"], "s1"]
    for kind in (IMPACT, LEGACY, CLASSIC, BM25):
        sim = sim_of(kind)
        for vname in ("unsliced", "mask", "stepped"):
            if kind == BM25 and vname == "unsliced":
                continue
            key = VIEWS[vname]
            view = make_view(zero, key)
            for k in KS:
                check(view, qs, k, sim, kind, lambda i: oz.dense(vname, key, qs[i], kind, sim), f"avgdl 0 {vname}",
                      want_bits=bit(kind, 0) if kind == CLASSIC else 0)
    inf = ctx.oracle.dense("unsliced", None, "r0", CLASSIC, sim_of(CLASSIC))
    assert np.isposinf(inf).sum() > 32
    d, s, _ = run(ctx.arr, ["r0"], 32, sim_of(CLASSIC))
    assert np.all(np.isposinf(s[0]))


def test_shard_doc_base(ctx):
    """A shard (doc_base 1,000,003, corpus size 3,000,000, global dfs) under the three non-BM25 kinds, with and
    without where=: global ids, the shard's corpus size and global dfs."""
    from searcharray_b200 import SearchArray
    base, size = 1_000_003, 3_000_000
    gdf = np.asarray([int(ctx.host.term_lengths[i]) + 777 * (i + 1) for i in range(ctx.host.n_terms)], dtype=np.uint64)
    shard = SearchArray.from_host_index(_host(ctx.post, ctx.doc_lens, base), doc_base=base, corpus_size=size,
                                        global_df=gdf)
    o = Oracle(ctx.host, shard.avg_doc_length, shard=(size, gdf))
    mask = query_masks(len(BATCH), N, 8)
    for kind in (IMPACT, LEGACY, CLASSIC):
        sim = sim_of(kind)
        for where in (None, mask):
            for k in KS:
                check(shard, BATCH, k, sim, kind, lambda i: o.dense("unsliced", None, BATCH[i], kind, sim),
                      "shard", where=where, doc_base=base)


def test_legacy_idf_sign(ctx):
    """sa_score_batch_topk_sim with legacy idfs < 0, = 0 and > 0 in one batch: idf < 0 ranks by -sat, idf == 0 ranks
    nothing; the scores are idf * sat.  A non-finite idf is refused under legacy and classic."""
    from oracle import similarity as osim
    from searcharray_b200 import _lib
    arr = ctx.arr
    qs = ["r0", "r1", "edge", "r0", "s0", "r1"]
    idf = np.asarray([-2.5, 0.0, 1.75, 3.0, -0.3, -0.0], dtype=np.float64)
    tids = np.asarray([ctx.host.term_dict.term_to_ids[q] for q in qs], dtype=np.uint32)
    starts = np.arange(len(qs) + 1, dtype=np.uint32)
    dbl = ctypes.POINTER(ctypes.c_double)
    h = arr._device().handle
    avg = float(arr.avg_doc_length)
    for k1, b in ((1.2, 0.75), (-1.5, 0.3)):
        f32 = np.float32
        for k in KS:
            docs = np.full((len(qs), k), NO_DOC, dtype=np.uint32)
            scores = np.zeros((len(qs), k), dtype=np.float64)
            with arr._shared["lock"]:
                arr._apply_rows(arr._device())
                _lib.check(_lib.lib().sa_stats_reset(h))
                _lib.check(_lib.lib().sa_score_batch_topk_sim(
                    h, LEGACY, _lib.p_u32(tids), _lib.p_u32(starts), idf.ctypes.data_as(dbl), len(qs), 0, None, avg,
                    k1, b, k, None, N, 0, _lib.p_u32(docs), scores.ctypes.data_as(dbl)))
            st = stats(arr)
            RAN.update(i for i in range(8) if st.sim_instances >> i & 1)
            assert st.sim_instances == bit(LEGACY, 0), hex(st.sim_instances)
            for i, q in enumerate(qs):
                tf = ctx.oracle.counts("unsliced", None, q)
                # bm25_legacy derives its idf from the dfs and cannot take a negative one: the saturation is
                # rebuilt from the oracle's shared denominator, and the product formed as bm25_legacy forms it
                sat = (tf * f32(k1 + 1)) / osim._saturation_denominator(tf, ctx.host.doc_lens, avg, k1, b)
                dense = np.float64(idf[i]) * sat.astype(np.float64)
                wd, ws = topk(dense, k)
                tag = f"idf {idf[i]} k1={k1} {q} k={k}"
                assert np.array_equal(docs[i], wd), f"{tag}: ids {docs[i]} want {wd}"
                assert np.array_equal(bits_of(scores[i]), bits_of(ws)), f"{tag}: bits {scores[i]} want {ws}"
                if idf[i] == 0:
                    assert np.all(docs[i] == NO_DOC), tag
            assert np.any(docs[0] != NO_DOC) == (k1 < 0), "idf < 0 ranks where sat < 0 only"
    for kind in (LEGACY, CLASSIC):
        for bad in (np.nan, np.inf, -np.inf):
            one = np.asarray([bad], dtype=np.float64)
            docs = np.zeros((1, 10), dtype=np.uint32)
            scores = np.zeros((1, 10), dtype=np.float64)
            with arr._shared["lock"]:
                rc = _lib.lib().sa_score_batch_topk_sim(h, kind, _lib.p_u32(tids[:1]), _lib.p_u32(starts[:2]),
                                                       one.ctypes.data_as(dbl), 1, 0, None, avg, 1.2, 0.75, 10, None,
                                                       N, 0, _lib.p_u32(docs), scores.ctypes.data_as(dbl))
            assert rc != 0, (kind, bad)


# ------------------------------------------------------------------------------------------- overflow re-runs
def flood_case(n=10_000):
    """A view whose tile 0 holds the flood layout: the best scores in the 32 positions of each of 31 threads, the next
    in single positions of 32 other threads, so that more positions than candidate slots reach the tile bound.  z is
    the flood as a term (tf 5 / 1), za zb as a phrase (5 / 1 matches); s is a sparse term that never overflows."""
    from searcharray_b200 import SearchArray
    high = [4 * (t + 256 * j) + e for t in range(31) for j in range(8) for e in range(4)]
    low = [4 * t for t in range(31, 63)]
    special = high + low
    taken = set(special)
    rest = [p for p in range(TILE) if p not in taken]
    perm = np.empty(TILE, dtype=np.int64)
    perm[special] = np.arange(len(special))
    perm[rest] = np.arange(len(special), TILE)
    rng = np.random.default_rng(12)
    dl = rng.integers(1, 40, n).astype(np.float32)
    dl[:len(special)] = 10
    tf = {d: (5 if d < len(high) else 1) for d in range(len(special))}
    post = {}
    _add(post, "z", np.arange(len(special)), lambda d: list(range(tf[d])))
    _add(post, "za", np.arange(len(special)), lambda d: list(range(0, 2 * tf[d], 2)))
    _add(post, "zb", np.arange(len(special)), lambda d: list(range(1, 2 * tf[d], 2)))
    _add(post, "s", np.arange(len(special) + 5, n, 97), lambda d: [3 + d % 3])
    host = _host(post, dl)
    arr = SearchArray.from_host_index(host)
    rows = np.concatenate([perm, np.arange(TILE, n)])
    return host, arr, rows, np.sort(np.asarray(high))


def test_overflow_reruns():
    """A term and a phrase query whose tile overflows, on a view, under each kind, with and without a where mask:
    one exact re-run each (k >= 10, and classic at every k), next to a query that does not overflow."""
    host, arr, rows, high = flood_case()
    o = Oracle(host, arr.avg_doc_length)
    view = arr[rows]
    where = np.random.default_rng(6).random(len(rows)) < 0.7
    where[:TILE] |= np.isin(rows[:TILE], np.arange(1024))
    for kind in (IMPACT, LEGACY, CLASSIC, BM25):
        sim = sim_of(kind)
        for qs, first, again in ((["s", "z"], (1, 2), (1, 2)), (["s", ["za", "zb"]], (1, 3), (0, 2))):
            for w in (None, where):
                for k in KS:
                    st, d = check(view, qs, k, sim, kind, lambda i: o.dense("flood", rows, qs[i], kind, sim),
                                  f"overflow {KIND_NAMES[kind]} {qs[1]}", where=w)
                    # one tf scan, a tile pass per row and one select for the batch, then the re-run's tf scan (a term),
                    # tile pass and select.  At k = 1 and 2 the float32 keys' bound keeps the tied tile within its
                    # 128 slots; classic keeps every tie at the bound and re-runs at every k.
                    rerun = kind == CLASSIC or k >= 10
                    want = tuple(f + (a if rerun else 0) for f, a in zip(first, again))
                    assert (st.term_kernel_launches, st.topk_kernel_launches) == want, \
                        (KIND_NAMES[kind], qs, k, st.term_kernel_launches, st.topk_kernel_launches)
                    assert np.array_equal(d[1], high[:k].astype(np.uint32))


def test_chunked_batch_with_overflow_in_second_chunk():
    """4,000,000 docs: one chunk holds 268 doc-space rows (4 GiB over a padded row of 4,005,888 floats), so 300
    queries on a 10 % mask view run as two chunks.  The second chunk has its own terms (idfs no first-chunk row has),
    phrases, per-query masks and one overflowing query: the chunk offsets of the idfs, the row-query map and the
    overflow flags.  The first chunk has 4 term rows and the overflowing term is the second chunk's term row 11, so a
    flag stored without the chunk's row offset would re-run global row 11, a phrase, in its place: the launch counts
    pin that the right row was re-run.  No other query has as many positions with a count in one tile as it has
    candidate slots, so none other can overflow."""
    from searcharray_b200 import SearchArray
    n, nq, over, chunk = 4_000_000, 300, 290, 268
    rng = np.random.default_rng(44)
    mask = rng.random(n) < 0.1
    rows = np.flatnonzero(mask)
    _, _, perm_rows, high = flood_case()
    flood_docs = rows[:TILE][np.argsort(perm_rows[:TILE])][:1024]   # view position p holds doc rows[p]
    dl = rng.integers(1, 40, n).astype(np.float32)
    dl[flood_docs] = 10
    tf = {int(d): (5 if i < 992 else 1) for i, d in enumerate(flood_docs)}
    post = {}
    _add(post, "x", np.sort(rng.choice(n, 6_000, replace=False)), lambda d: [3])
    _add(post, "y", np.sort(rng.choice(n, 4_000, replace=False)), lambda d: [5, 6])
    _add(post, "w", np.sort(rng.choice(n, 30_000, replace=False)), lambda d: [7] if d % 3 else [7, 30])
    ph = np.sort(rng.choice(n, 20_000, replace=False))
    _add(post, "pa", ph, lambda d: [9])
    _add(post, "pb", ph[::2], lambda d: [10])
    _add(post, "pc", ph[::3], lambda d: [11])
    _add(post, "z", flood_docs, lambda d: list(range(tf[d])))
    host = _host(post, dl)
    arr = SearchArray.from_host_index(host)
    view = arr[mask]
    o = Oracle(host, arr.avg_doc_length)
    first_terms = {0: "x", 67: "y", 134: "x", 201: "y"}
    queries = [first_terms.get(i, [["pa", "pb"], ["pb", "pc"]][i % 2]) if i < chunk else
               (("w" if i % 4 == 0 else "y") if i % 2 == 0 else ["pa", "pb"]) for i in range(nq)]
    queries[over] = "z"
    terms = [sum(isinstance(q, str) for q in part) for part in (queries[:chunk], queries[chunk:])]
    assert terms == [4, 16] and sum(isinstance(q, str) for q in queries[chunk:over]) == 11
    pats = np.zeros((3, len(view)), dtype=bool)
    pats[0] = np.random.default_rng(8).random(len(view)) < 0.6
    pats[1, TILE:] = True
    pats[2] = True
    pat_of = [2 if i == over else i % 3 for i in range(nq)]
    where = pats[pat_of]
    for kind in (BM25, LEGACY):
        sim = sim_of(kind)
        for k in (10, 32):
            reset(view)
            docs, scores = view.search_topk(queries, k=k, similarity=sim, where=where)
            st = stats(view)
            RAN.update(i for i in range(8) if st.sim_instances >> i & 1)
            assert st.sim_instances == bit(kind, 1), hex(st.sim_instances)
            # per chunk one tf scan, one tile pass for its terms, one per phrase and one select; then the re-run of
            # the overflowing term: a tf scan, a tile pass and a select
            want = (2 + 1, (1 + (chunk - 4) + 1) + (1 + (nq - chunk - 16) + 1) + 2)
            assert (st.term_kernel_launches, st.topk_kernel_launches) == want, \
                (KIND_NAMES[kind], k, st.term_kernel_launches, st.topk_kernel_launches)
            want = {}
            for i, q in enumerate(queries):
                wk = (repr(q), pat_of[i])
                if wk not in want:
                    dense = o.dense("mask4m", mask, q, kind, sim)
                    want[wk] = topk(np.where(pats[pat_of[i]], dense, dense.dtype.type(0)).astype(dense.dtype), k)
                wd, ws = want[wk]
                tag = f"4M {KIND_NAMES[kind]} query {i} {q!r} k={k}"
                assert np.array_equal(docs[i], wd), f"{tag}: ids {docs[i]} want {wd}"
                assert np.array_equal(bits_of(scores[i]), bits_of(ws)), f"{tag}: score bits"
            assert np.array_equal(docs[over], high[:k].astype(np.uint32))


# ------------------------------------------------------------------------------- filter and min / max posn
POSN_TOKENS = ["r0", "qa", "f2047", "f2048", "f2049", "f5000", "pa", "zzz"]
POSN_PHRASES = [["qa", "qb"], ["pa", "pb"], ["f5000", "f2049"], ["qa", "zzz"]]


@pytest.mark.parametrize("vname", ["len16385", "mask", "stepped", "view_of_view", "len8193"])
def test_min_max_posn_on_views(ctx, vname):
    """view.termfreqs and view.score (BM25) with min_posn, max_posn and both, for terms and phrases (slop 0 and 2),
    against the oracle: the row mask and the payload test in one filter pass, over lists of 2,047, 2,048, 2,049 and
    5,000 words (the filter's 2,048-word chunks), and a phrase of two multi-chunk lists."""
    key = VIEWS[vname]
    view = make_view(ctx.arr, key)
    o = ctx.oracle
    ov, _, _ = o.view(vname, key)
    for lo, hi in ((18, None), (None, 35), (18, 35)):
        for q in POSN_TOKENS + POSN_PHRASES:
            for slop in ((0,) if isinstance(q, str) else (0, 2)):
                ids = o.tids(q)
                arg = ids[0] if isinstance(q, str) else ids
                tag = f"{vname} {q!r} slop={slop} min={lo} max={hi}"
                got = view.termfreqs(q, slop=slop, min_posn=lo, max_posn=hi)
                want = ov.termfreqs(arg, slop=slop, min_posn=lo, max_posn=hi)
                assert np.array_equal(got, want), f"{tag}: counts differ at {np.flatnonzero(got != want)[:10]}"
                got = view.score(q, slop=slop, min_posn=lo, max_posn=hi)
                want = ov.score(arg, slop=slop, min_posn=lo, max_posn=hi)
                assert np.array_equal(bits_of(got), bits_of(np.asarray(want, dtype=np.float32))), f"{tag}: BM25 bits"
    full = view.termfreqs("qa")
    assert np.any(view.termfreqs("qa", min_posn=18, max_posn=35) != full), "the payload test removed nothing"


# --------------------------------------------------------------------------------------- document frequencies
def check_docfreqs(ctx, what):
    """sa_docfreq_rows_batch of every term (and an unknown one) on every view, against the oracle's slice dfs."""
    from searcharray_b200 import _lib
    tids = np.asarray(list(range(ctx.host.n_terms)) + [_lib.NO_TERM], dtype=np.uint32)
    # the straddling doc's words sit at list indices 4095 and 4096; two views hold it by construction
    w = ctx.host.term_words(ctx.host.term_dict.term_to_ids["straddle"]) >> np.uint64(36)
    assert len(w) > 2 * 4096 and w[STRADDLE_AT] == w[STRADDLE_AT + 1] and w[STRADDLE_AT - 1] != w[STRADDLE_AT]
    doc = int(w[STRADDLE_AT])
    around = np.arange(N) % 3 == 0
    around[doc] = True
    views = dict(VIEWS, around_straddle=slice(max(doc - 40, 0), doc + 40), straddle_mask=around)
    for name in ("around_straddle", "straddle_mask"):
        assert doc in view_rows(N, views[name]), name
    for vname, key in views.items():
        if key is None:
            continue
        view = make_view(ctx.arr, key)
        dfs = np.zeros(len(tids), dtype=np.uint64)
        dev = view._device()
        with view._shared["lock"]:
            view._apply_rows(dev)
            _lib.check(_lib.lib().sa_docfreq_rows_batch(dev.handle, _lib.p_u32(tids), len(tids), _lib.p_u64(dfs)))
        ov, _, _ = ctx.oracle.view(vname, key)
        want = [ov.docfreq(int(t)) for t in tids[:-1]] + [0]
        bad = [(ctx.host.term_dict.get_term(int(t)), int(dfs[i]), want[i]) for i, t in enumerate(tids[:-1])
               if int(dfs[i]) != want[i]]
        assert not bad and dfs[-1] == 0, f"{what} {vname}: (term, df, want) {bad}"


def test_docfreqs(ctx):
    """The records branch (tf table): a full 8-tile job and a partial one; docs at 8191 / 8192, tile 7 and the last
    doc; the words branch for the short lists."""
    check_docfreqs(ctx, "records")


def test_words_branch_without_tf_table():
    """The document-frequency and term checks in a process with SA_NO_TF_TABLE=1, where every list takes the words
    branch: jobs of 4,096 words, one doc straddling a job boundary."""
    env = dict(os.environ, SA_NO_TF_TABLE="1")
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_view_paths_worker.py")
    r = subprocess.run([sys.executable, worker], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.strip().splitlines()[-1] == "OK", r.stdout[-3000:]


def test_every_instance_ran(ctx):
    """The union of sim_instances over this module is all 8 tile kernels (the kind checks run here for any this
    session's selection skipped)."""
    for kind in (IMPACT, LEGACY, CLASSIC, BM25):
        for masked in (0, 1):
            if 2 * kind + masked not in RAN:
                check_kind_view(ctx, kind, "mask", slops=(0,), ks=(10,))
    assert RAN == set(range(8)), sorted(set(range(8)) - RAN)
