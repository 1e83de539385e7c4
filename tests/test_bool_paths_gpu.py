"""GPU: every branch of the batched boolean tile kernel (bool_tile_kernel in sa_bool.cu, through search_topk and
fields_topk) against the CPU oracle.  Each clause's float32 vector comes from oracle.search on that column's own index
under that column's k1, b and avgdl (a shard's through oracle.search.bm25 with its corpus size and global dfs), feature
values from the functions stated below, and the composition from tests/_nested_compose.py; `where=` is
np.where(mask, s, 0), the counts are (s > 0).sum() and np.bincount of the ranked docs' codes.  Ids, float32 score
bits, the NO_DOC / 0 padding, totals and facet counts must be equal.  sa_stats.bool_instances names the instances each
call launched (bit variant * 10 + form * 2 + masked), and every check asserts the exact set.

The frame has three columns over 5 full tiles and a partial one: `a` (doc lengths 1..59, some 0; k1 1.2, b 0.75) with
`w0` / `w1` / `w2` (tile directory and tf records), `s1` / `s2` (binary search over the words), `t0` / `t3` / `t5`
(tile 0 / 3 / the partial tile only), `pa` / `pb` (phrases at slop 0 and 2, a same-term phrase), `big` (tf 2^18 at
tile offsets 0 and 8191), `hot` / `cold` (a tile whose candidates overflow) and feature and facet columns; `b` (doc
lengths 20..299, some 0; k1 0.9, b 0.4) with its own postings; `z`, b's postings under avgdl 0.  The records-term and
tf = 2^18 checks run again in a child process with SA_NO_TF_TABLE=1 (tests/_bool_paths_worker.py), where the records
terms take the words path over their tile directory."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest

from _bool_compose import topk
from _nested_compose import compose_nested

pytestmark = pytest.mark.gpu

TILE = 8192
N = 5 * TILE + 300
KS = (1, 10, 16, 17, 32)
BIG_TF = 1 << 18
BIG_DOCS = (0, 2 * TILE + TILE - 1)          # tile offsets 0 and 8191
OR_AND, OCCUR, FIELDS, DISMAX, NESTED = range(5)
PLAIN, FEATURE, COUNT = range(3)
INSTANCES = [(f, m, v) for v in (PLAIN, FEATURE, COUNT) for f in range(5) for m in (0, 1) if v == PLAIN or f > OR_AND]
SIMS = {"a": (1.2, 0.75), "b": (0.9, 0.4), "z": (1.2, 0.75)}
RAN = set()                                   # bool_instances bits seen by this module's calls


def bit(form, masked, variant):
    return 1 << (variant * 10 + form * 2 + masked)


# ------------------------------------------------------------------------------------------------------------ corpus
def _postings(n, rng):
    postings = {}

    def add(name, docs, posns_of):
        d, p = [], []
        for doc in np.unique(np.asarray(docs, dtype=np.int64)):
            ps = sorted(set(posns_of(doc)))
            d += [doc] * len(ps)
            p += ps
        postings[name] = (np.asarray(d, dtype=np.int64), np.asarray(p, dtype=np.int64))
    return postings, add


def _host(postings, doc_lens, doc_base):
    from searcharray_b200.indexing import index_from_term_postings
    from searcharray_b200.roaringish import encode_postings
    names = list(postings)
    words = [encode_postings(d + doc_base, p) for d, p in (postings[t] for t in names)]
    return index_from_term_postings(names, words, doc_lens)


def column_a(n=N, doc_base=0, seed=31):
    rng = np.random.default_rng(seed)
    doc_lens = rng.integers(1, 60, n).astype(np.float32)
    doc_lens[rng.random(n) < 0.03] = 0
    doc_lens[list(BIG_DOCS)] = BIG_TF
    postings, add = _postings(n, rng)

    def rand_posns(doc):
        return rng.integers(30, 200, rng.integers(1, 4)).tolist()
    add("w0", np.flatnonzero(rng.random(n) < 0.45), rand_posns)             # tf records
    add("w1", np.flatnonzero(rng.random(n) < 0.2), rand_posns)
    add("w2", rng.choice(n, 1200, replace=False), rand_posns)
    add("s1", rng.choice(3 * TILE, 400, replace=False), rand_posns)         # binary search over the words
    add("s2", np.concatenate([rng.choice(np.arange(TILE, 3 * TILE), 200, replace=False),
                              rng.choice(np.arange(4 * TILE, n), 100, replace=False)]), rand_posns)
    add("t0", rng.choice(TILE, 300, replace=False), rand_posns)             # one tile each
    add("t3", 3 * TILE + rng.choice(TILE, 300, replace=False), rand_posns)
    add("t5", 5 * TILE + rng.choice(n - 5 * TILE, 120, replace=False), rand_posns)
    ph = rng.choice(n, 3000, replace=False)
    add("pa", ph, lambda doc: [10, 11] if doc % 5 == 0 else [10])
    add("pb", ph[:2000], lambda doc: [11] if doc % 2 else [13])
    # four threads of tile 1 own its best docs, many others hold lower scores: its candidates overflow
    hot = TILE + np.asarray([4 * t + e + 1024 * j for t in range(4) for e in range(4) for j in range(8)])
    add("hot", hot, lambda doc: list(range(40, 40 + 2 + doc % 5)))
    add("cold", np.setdiff1d(TILE + rng.choice(TILE, 1500, replace=False), hot), lambda doc: [40])
    # tf 2^18 at tile offsets 0 and 8191 next to 2,000 ordinary docs (a records term)
    small = np.sort(rng.choice(np.setdiff1d(np.arange(n), BIG_DOCS), 2000, replace=False))
    runs = dict(zip(small.tolist(), rng.integers(1, 4, len(small)).tolist()))
    add("big", np.concatenate([small, BIG_DOCS]),
        lambda doc: list(range(BIG_TF)) if doc in BIG_DOCS else (18 * np.arange(runs[doc])).tolist())
    return _host(postings, doc_lens, doc_base)


def column_b(n=N, doc_base=0, seed=23):
    rng = np.random.default_rng(seed)
    doc_lens = rng.integers(20, 300, n).astype(np.float32)
    doc_lens[rng.random(n) < 0.03] = 0
    postings, add = _postings(n, rng)

    def rand_posns(doc):
        return rng.integers(5, 250, rng.integers(1, 5)).tolist()
    add("w0", np.flatnonzero(rng.random(n) < 0.3), rand_posns)
    add("b1", np.flatnonzero(rng.random(n) < 0.5), rand_posns)
    add("bs", rng.choice(np.arange(TILE, n), 700, replace=False), rand_posns)
    add("b2", 2 * TILE + rng.choice(TILE, 1500, replace=False), rand_posns)
    qd = rng.choice(n, 2500, replace=False)
    add("qa", qd, lambda doc: [7])
    add("qb", qd[:1800], lambda doc: [8] if doc % 4 else [9])
    return _host(postings, doc_lens, doc_base)


def feature_columns(n=N, seed=7):
    """`fx`: 0, -0, denormals, ordinary values and 3e38 (x + pivot overflows float32 under a pivot of 1e38); tile 4
    holds only values <= 0 (0 and -0), so its tile flag is unset; the partial tile holds values.  `pop`: integers."""
    rng = np.random.default_rng(seed)
    kind = rng.integers(0, 6, n)
    fx = np.select([kind == 0, kind == 1, kind == 2, kind == 3, kind == 4],
                   [np.float32(0), np.float32(-0.0), np.float32(1e-45), np.float32(1e-40),
                    (rng.random(n) * 100).astype(np.float32)], np.float32(0)).astype(np.float32)
    fx[kind == 5] = (rng.random(int((kind == 5).sum())) * 7).astype(np.float32)
    fx[rng.choice(n, 5, replace=False)] = np.float32(3e38)
    fx[4 * TILE:5 * TILE] = np.where(rng.random(TILE) < 0.5, np.float32(-0.0), np.float32(0))
    fx[5 * TILE + 17] = np.float32(42.5)
    pop = np.where(rng.random(n) < 0.8, rng.integers(1, 1000, n), 0).astype(np.float32)
    return {"fx": fx, "pop": pop}


def facet_columns(n=N, seed=9):
    """Four facets of 1,024 buckets (together the 16 KB histogram) and a small one, each with -1 codes."""
    rng = np.random.default_rng(seed)
    out = {}
    for i in range(4):
        c = rng.integers(0, 1024, n).astype(np.int32)
        c[rng.random(n) < 0.2] = -1
        out[f"g{i}"] = (c, 1024)
    c = rng.integers(-1, 3, n).astype(np.int32)
    out["small"] = (c, 3)
    return out


def feature_value(f, x):
    """Lucene's FeatureField functions, stated here: +0 where x is not > 0; x; x / (x + pivot) rounded in float32
    after each step; float32(log(float64(s) + float64(x)))."""
    x = np.asarray(x, dtype=np.float32)
    p = np.float32(f.param)
    with np.errstate(over="ignore", under="ignore"):
        if f.function == "linear":
            v = x.copy()
        elif f.function == "saturation":
            v = np.divide(x, np.add(x, p, dtype=np.float32), dtype=np.float32)
        else:
            v = np.log(np.float64(p) + x.astype(np.float64)).astype(np.float32)
    return np.where(x > 0, v, np.float32(0)).astype(np.float32)


class Oracle:
    """Per-clause float32 vectors of oracle.search, per column under that column's parameters.  shard: (corpus size,
    avgdl, {column: global dfs}) of a shard whose local postings the hosts hold."""

    def __init__(self, hosts, avgdl, features=None, shard=None):
        from oracle import search as osearch
        self.hosts, self.features, self.shard = hosts, features or {}, shard
        self.oidx = {c: osearch.OracleIndex({t: h.term_words(t) for t in range(h.n_terms)}, h.doc_lens,
                                            avg_doc_length=avgdl[c]) for c, h in hosts.items()}
        self.cache = {}

    def vec(self, col, clause, slop=0, k1=None, b=None):
        from oracle import search as osearch
        k1 = SIMS[col][0] if k1 is None else k1
        b = SIMS[col][1] if b is None else b
        key = (col, repr(clause), slop, k1, b)
        if key not in self.cache:
            toks = [clause] if isinstance(clause, str) else list(clause)
            ids = [self.hosts[col].term_dict.term_to_ids.get(t) for t in toks]
            o = self.oidx[col]
            if self.shard is None:
                v = o.score(ids[0] if isinstance(clause, str) else ids, k1=k1, b=b, slop=slop)
            elif any(i is None for i in ids):
                v = np.zeros(len(o), dtype=np.float32)
            else:
                size, avg, gdf = self.shard
                tfs = o.termfreqs(ids[0] if isinstance(clause, str) else ids, slop=slop)
                v = osearch.bm25(tfs, [gdf[col][i] for i in ids], o.doc_lens, avg, size, k1, b)
            self.cache[key] = np.asarray(v, dtype=np.float32)
        return self.cache[key]

    def scorer(self, slop=0):
        """score(clause) for compose_nested: a term / phrase / Feature on column a, or a Field of one."""
        from searcharray_b200 import Feature, Field

        def score(c):
            col = "a"
            if isinstance(c, Field):
                col, c = c.field, c.clause
            if isinstance(c, Feature):
                return feature_value(c, self.features[col][c.name])
            return self.vec(col, c, slop)
        return score


class Ctx:
    def __init__(self):
        from searcharray_b200 import SearchArray
        ha, hb = column_a(), column_b()
        self.hosts = {"a": ha, "b": hb, "z": hb}
        self.frame = pd.DataFrame({"a": SearchArray.from_host_index(ha), "b": SearchArray.from_host_index(hb)})
        self.frame["z"] = SearchArray.from_host_index(hb, avg_doc_length=0.0)
        self.arr = self.frame["a"].array
        self.features = feature_columns()
        for name, v in self.features.items():
            self.arr.set_feature(name, v)
        self.facets = facet_columns()
        for name, (c, nb) in self.facets.items():
            self.arr.set_facet(name, c, n_buckets=nb)
        bf = np.random.default_rng(4).integers(-1, 7, N).astype(np.int32)
        self.frame["b"].array.set_facet("bf", bf, n_buckets=7)
        self.codes = {("a", k): c for k, (c, _) in self.facets.items()}
        self.codes[("b", "bf")] = bf
        self.oracle = Oracle(self.hosts, {c: self.frame[c].array.avg_doc_length for c in self.frame.columns},
                             {"a": self.features})


@pytest.fixture(scope="module")
def ctx():
    return Ctx()


# ------------------------------------------------------------------------------------------------------------ checks
def _handles(frame):
    hs = []
    for c in frame.columns:
        h = frame[c].array._device().handle
        if h not in hs:
            hs.append(h)
    return hs


def sims_of(cols=SIMS, override=None):
    from searcharray_b200 import bm25_similarity
    out = {c: bm25_similarity(k1=k1, b=b) for c, (k1, b) in cols.items()}
    out.update(override or {})
    return out


def run(frame, queries, k, fields, where=None, facets=None, slop=0, sims=None):
    """(docs, scores, n_redone, hits or None, bool_instances over the frame's indexes) of one call."""
    from searcharray_b200 import _lib, solr
    from searcharray_b200.postings import pack_where
    sims = sims or sims_of()
    hs = _handles(frame)
    for h in hs:
        _lib.check(_lib.lib().sa_stats_reset(h))
    if fields:
        out = solr._fields_topk(frame, queries, k, {c: sims[c] for c in frame.columns}, slop, where, facets)
    else:
        arr = frame["a"].array
        bits = None if where is None else pack_where(where, len(arr), len(queries))
        out = arr._search_topk_bool(queries, k, sims["a"], slop, bits, facets)
    inst = 0
    for h in hs:
        st = _lib.SaStats()
        _lib.check(_lib.lib().sa_stats_get(h, ctypes.byref(st)))
        inst |= st.bool_instances
    for i in range(64):
        if inst >> i & 1:
            RAN.add(i)
    return out[0], out[1], out[2], (out[3] if facets is not None else None), inst


def assert_topk(docs, scores, dense, k, what, doc_base=0):
    wd, ws = topk(dense, k, doc_base)
    assert np.array_equal(np.asarray(docs, dtype=np.uint32), wd), f"{what}: ids {docs} want {wd}"
    assert np.array_equal(np.asarray(scores, dtype=np.float32).view(np.uint32), ws.view(np.uint32)), \
        f"{what}: score bits {scores} want {ws}"


def check(frame, queries, k, what, fields, score, want_bits, where=None, facets=None, codes=None, slop=0, sims=None,
          doc_base=0, redone=None):
    """One call against the composition of score(clause): ids, bits, padding, counts and the instances launched.
    want_bits: the bits of the first pass and the store passes; an overflow re-run adds re_bit (see expect)."""
    docs, scores, n_redone, hits, inst = run(frame, queries, k, fields, where, facets, slop, sims)
    assert docs.shape == (len(queries), k) and docs.dtype == np.uint32 and scores.dtype == np.float32
    first, re_bit = want_bits
    want = first | (re_bit if n_redone else 0)
    assert inst == want, f"{what} k={k}: bool_instances {inst:#x} want {want:#x} (n_redone {n_redone})"
    if redone is not None:
        assert n_redone == redone, f"{what} k={k}: {n_redone} queries re-run, want {redone}"
    cache = {}
    for i, q in enumerate(queries):
        dense = compose_nested(score, q, cache)
        if where is not None:
            dense = np.where(where[i], dense, np.float32(0)).astype(np.float32)
        tag = f"{what} #{i} {q!r} k={k}"
        assert_topk(docs[i], scores[i], dense, k, tag, doc_base)
        if hits is not None:
            ranked = dense > 0
            assert hits.total[i] == int(ranked.sum()), f"{tag}: total {hits.total[i]} want {int(ranked.sum())}"
            for key in facets:
                c = codes[key]
                want_c = np.bincount(c[ranked & (c >= 0)], minlength=hits.facets[key].shape[1])
                assert np.array_equal(hits.facets[key][i], want_c), \
                    f"{tag}: facet {key} counts differ at buckets {np.flatnonzero(hits.facets[key][i] != want_c)}"
    return n_redone


def expect(form, masked, variant, nested=False, features=None):
    """(bits of the first pass and the store passes, bit of an overflow re-run) of a call of `form`; the store
    passes and the re-run run FEATURE when the batch has a feature clause (by default: the FEATURE and COUNT batches
    of `batch`), PLAIN otherwise."""
    rest = FEATURE if (variant != PLAIN if features is None else features) else PLAIN
    first = bit(form, masked, variant) | (bit(NESTED, 0, rest) if nested else 0)
    return first, bit(form, masked, rest)


def masks(n_queries, n=N, seed=3):
    """Per-query masks: random docs; tiles 0-1 left out entirely; only tile 3 and the partial tile."""
    rng = np.random.default_rng(seed)
    out = np.zeros((n_queries, n), dtype=bool)
    for i in range(n_queries):
        kind = i % 3
        if kind == 0:
            out[i] = rng.random(n) < 0.7
        elif kind == 1:
            out[i, 2 * TILE:] = rng.random(n - 2 * TILE) < 0.5
        else:
            out[i, 3 * TILE:4 * TILE] = True
            out[i, 5 * TILE:] = True
    return out


# ------------------------------------------------------------------------------------------------- the batches
def _F(fields, col):
    from searcharray_b200 import Field
    return (lambda c: Field(col, c)) if fields else (lambda c: c)


def feature_clauses(fields):
    from searcharray_b200 import Boost, Feature
    fa = _F(fields, "a")
    return [fa(Feature("fx")), fa(Feature("fx", "saturation", pivot=1e38)), fa(Feature("fx", "saturation", pivot=0.5)),
            fa(Feature("fx", "log", scaling_factor=1)), Boost(fa(Feature("pop", "log", scaling_factor=3.5)), 0.5),
            fa(Feature("pop", "saturation", pivot=50))]


def batch(form, variant):
    """(queries, fields) of an instance: every role, zero weights, each list path, one-tile terms, an unknown token,
    tf 2^18, phrases, the avgdl-0 column; feature clauses in every role for the FEATURE and COUNT variants."""
    from searcharray_b200 import And, Bool, Boost, DisMax, Or
    fields = form >= FIELDS
    A, B, Z = _F(fields, "a"), _F(fields, "b"), _F(fields, "z")
    feats = feature_clauses(fields) if variant != PLAIN else []
    if form == OR_AND:
        return [Or(["w0", "w1", "s1"], mm=2), And(["t3", "w2"]), Or([["pa", "pb"], "s2", "big"]),
                Or(["zzz", "t5"]), Or(["w1", "w1", "s2"], mm=3), And([["pa", "pa"], "w0"]), Or(["t0", "t3"], mm=2),
                Or(["big", "t0", ["pb", "zzz"]])], False
    if form == OCCUR:
        qs = [Bool(must=["w0"], should=[Boost("w1", 2), "s1", Boost("big", 0)], must_not=["t0"], mm=1),
              Bool(filter=["t3"], should=["w0", ["pa", "pb"]]), Bool(must=[Boost("s2", 0)], should=["w2", "zzz"], mm=0),
              Bool(should=["w0", "w1"], must_not=[["pa", "pb"]], filter=["w2"]), Bool(must=["t5"], should=["w1"]),
              Bool(should=["big", "s1", "zzz"], mm=2), Or([Boost("w0", 3), "t0"])]
    elif form == FIELDS:
        qs = [Bool(must=[A("w0")], should=[B("w0"), B("bs"), Z("b1")], mm=1),
              Bool(filter=[B("b2")], should=[A("w0"), A("s1"), Boost(B("b1"), 0.5)]),
              Or([A(["pa", "pb"]), B(["qa", "qb"]), A("big"), B("zzz")]),
              Bool(should=[A("t5"), B("b1")], must_not=[B("bs")], mm=1),
              Bool(must=[Boost(A("t3"), 0)], should=[B("w0"), Z("w0")]), And([A("w1"), B("b1"), A("s2")])]
    elif form == DISMAX:
        qs = [Bool(must=[DisMax([A("w0"), B("w0")], tie=0.3)],
                   should=[DisMax([A("s1"), Boost(B("bs"), 2), A("t0")], tie=0.0), B("b1")]),
              Or([DisMax([A("w1"), B("b2")], tie=1.0), DisMax([A(["pa", "pb"]), B(["qa", "qb"])], tie=0.5), A("t3")],
                 mm=2),
              Bool(should=[DisMax([Boost(A("w2"), 0), B("bs"), A("t0")], tie=0.2)],
                   must_not=[DisMax([A("t3"), B("b2")])], filter=[A("w0")]),
              Bool(filter=[DisMax([A("t5"), Z("b1")])], should=[A("big"), DisMax([B("zzz"), A("s2")], tie=0.7)])]
    else:
        qs = [Bool(must=[Or([A("w0"), And([B("b1"), A("w1")])])],
                   should=[Boost(Bool(should=[A("s1"), DisMax([A("s2"), B("bs")], tie=0.1)]), 2), B("w0")],
                   filter=[Or([A("w2"), B("b2")])], must_not=[And([A("t3"), B("b1")])], mm=1),
              Or([And([A(["pa", "pb"]), Or([B("qa"), Bool(must=[A("w1")], should=[B("b1")])])]), A("t5")]),
              Bool(should=[Boost(Or([A("big"), Z("w0")]), 0), A("t0")], must=[Or([A("w0"), A("t3")])])]
    if feats:
        f = feats
        qs += [Bool(should=[A("w1"), f[1]]), Bool(must=[f[0]], should=[A("s2")]),
               Bool(should=[A("w0")], filter=[f[3]], must_not=[f[5]]), Bool(should=[Boost(f[0], 0), A("t5")], mm=1),
               Bool(should=[f[2], f[4]], mm=2), Bool(should=[f[0], A("w2")])]
        if form == NESTED:
            qs += [Bool(should=[Or([A("w1"), f[2]], mm=2), Bool(must=[f[3]], should=[A("t3")])], must_not=[And([f[0]])])]
        if form == DISMAX:
            qs += [Bool(should=[DisMax([A("w0"), A("s1")], tie=0.5), f[4]])]
    return qs, fields


FACETS = {False: ["g0", "g1", "g2", "g3"], True: [("a", "g0"), ("b", "bf"), ("a", "small"), ("a", "g3")]}


@pytest.mark.parametrize("form, masked, variant", INSTANCES)
def test_instance(ctx, form, masked, variant):
    """Each of the 26 instances of the table: a batch that runs it, the exact instance bits, and the oracle."""
    qs, fields = batch(form, variant)
    where = masks(len(qs)) if masked else None
    facets = FACETS[fields] if variant == COUNT else None
    codes = {k: ctx.codes[("a", k) if isinstance(k, str) else k] for k in (facets or [])}
    nested = form == NESTED
    for slop in ((0, 2) if variant == PLAIN and not masked else (0,)):
        for k in KS:
            check(ctx.frame, qs, k, f"instance {form},{masked},{variant} slop={slop}", fields, ctx.oracle.scorer(slop),
                  expect(form, masked, variant, nested), where, facets, codes, slop)


@pytest.mark.parametrize("form", [OR_AND, OCCUR, DISMAX, NESTED])
def test_64_clauses(ctx, form):
    """64-clause queries at mm 0, 1, n and 64 (a SHOULD count of 64 in the per-doc hit bytes and in s_present's low
    16 bits), a group first at clause 63 and a DisMax whose last member (clause 63) is absent from most tiles."""
    from searcharray_b200 import And, Bool, DisMax, Or
    base = ["w0"] * 31 + ["w1"] * 31 + ["w2"]
    if form == OR_AND:
        qs = [Or(base + ["t3"], mm=m) for m in (0, 1, 64)] + [And(["w0", "w1"] * 32)]
    elif form == OCCUR:
        qs = [Bool(should=base + ["t3"], mm=m) for m in (0, 1, 64)]
        qs += [Bool(must=["w0"], should=base[:62] + ["t3"], mm=m) for m in (1, 63)]
        qs += [Bool(should=base, must=["t3"]), Bool(should=base, must_not=["t0"], mm=63)]
    elif form == DISMAX:
        qs = [Bool(should=[DisMax(["w0", "w1"], tie=0.5)] + base[:61] + ["t3"], mm=m) for m in (0, 1, 63)]
        qs += [Bool(should=base[:62] + [DisMax(["w1", "t3"], tie=0.5)], mm=m) for m in (1, 63)]
        qs += [Bool(should=base[:62] + [DisMax(["w0", "t0"], tie=1.0)], mm=63),
               Bool(should=base[:63] + [DisMax(["t3"])], mm=64)]
    else:
        qs = [Bool(should=[Or(base[:62], mm=m), "w2", "t3"], mm=3) for m in (1, 62)]
        qs += [Bool(should=["w2", Or(["w0", And(["w1"] * 30 + ["t3"])] + ["w1"] * 30)], mm=2)]
    for k in KS:
        check(ctx.frame, qs, k, f"64 clauses form {form}", False, ctx.oracle.scorer(), expect(form, 0, PLAIN,
                                                                                            form == NESTED))


def test_dismax_ties_roles_and_absent_members(ctx):
    """DisMax at tie 0 and 1 in every role, zero-weight members, a last member absent from most tiles and an absent
    first member, on one column (the one-entry field table)."""
    from searcharray_b200 import Bool, Boost, DisMax, Or
    qs = []
    for tie in (0.0, 1.0):
        qs += [Bool(must=[DisMax(["w0", "s1", "t0"], tie=tie)], should=["w1"]),
               Bool(should=[DisMax(["t3", "w1"], tie=tie), DisMax([Boost("w2", 0), "t5"], tie=tie)], mm=1),
               Bool(filter=[DisMax(["s2", "t0"], tie=tie)], should=["w0"]),
               Bool(should=["w0"], must_not=[DisMax(["t3", "zzz"], tie=tie)]),
               Or([DisMax([Boost("w0", 0), Boost("w1", 0)], tie=tie), "s1"], mm=2),
               Bool(should=[DisMax([["pa", "pb"], "big", "t0"], tie=tie)])]
    for k in KS:
        check(ctx.frame, qs, k, "dismax", False, ctx.oracle.scorer(), expect(DISMAX, 0, PLAIN))


def test_nested_three_levels_every_role(ctx):
    from searcharray_b200 import And, Bool, Boost, DisMax, Or
    qs = [Bool(must=[Or([And(["w0", Or(["s1", Bool(must=["w1"], must_not=["t0"])])]), "t3"])],
               should=[Boost(Or(["w2", And(["w0", "w1"])]), 0.5)], filter=[Or(["w0", Or(["w1", And(["s2"])])])],
               must_not=[And(["w1", Or(["s1", "t5"], mm=2)])]),
          Or([Or([Or([Or(["t3", "w2"], mm=2)])]), Boost(And(["w0", DisMax(["w1", "s2"], tie=0.4)]), 0)], mm=1),
          Bool(should=[Bool(should=[Bool(should=["big", ["pa", "pb"]], mm=1)], must=["w0"]), "t0"], mm=2)]
    for k in KS:
        check(ctx.frame, qs, k, "nested", False, ctx.oracle.scorer(), expect(NESTED, 0, PLAIN, True))


def test_stale_nested_rows(ctx):
    """A nested node's row keeps a previous call's values where, in this call, the child ranks nothing: a tile pruned
    before the fold (only its flag is written) and a tile whose fold ranks nothing.  The parent must read neither."""
    from searcharray_b200 import And, Bool, Or
    score = ctx.oracle.scorer()
    fill = [Bool(should=["w2", Or(["w0", "w1"])]), Bool(should=["s1", Or(["w1"])])]
    for second in ([Bool(should=["w2", And(["t3", "w1"])]), Bool(should=["s1", Or(["t0"])])],
                   [Bool(should=["w2", Bool(should=["w1"], must_not=["w1"])]),
                    Bool(should=["s1", Bool(must=["w0"], filter=["t5"])])]):
        for k in (10, 32):
            check(ctx.frame, fill, k, "fill", False, score, expect(NESTED, 0, PLAIN, True))
            check(ctx.frame, second, k, "stale", False, score, expect(NESTED, 0, PLAIN, True))
            where = masks(len(second))
            check(ctx.frame, fill, k, "fill", False, score, expect(NESTED, 0, PLAIN, True))
            check(ctx.frame, second, k, "stale masked", False, score, expect(NESTED, 1, PLAIN, True), where)


def assert_contract(got, want, what):
    assert np.array_equal(np.isnan(got), np.isnan(want)), f"{what}: NaN masks differ"
    ok = ~np.isnan(want)
    np.testing.assert_allclose(got[ok], want[ok], rtol=1e-5, atol=0, err_msg=what)


@pytest.mark.parametrize("k1, b", [(0.0, 0.75), (1.2, 1.0), (1.2, 1.5)])
def test_exotic_parameters(ctx, k1, b):
    """Parameters that are not sparse-safe on the OCCUR, WHERE, COUNT and FIELDS instances: .score of each term
    against the oracle under the 1e-5 contract with the same NaN mask, then the top k bit for bit against the
    composition of .score.  Phrases and DisMax members stay refused."""
    from searcharray_b200 import Bool, Boost, DisMax, Field, Or, _lib, bm25_similarity
    sim = bm25_similarity(k1=k1, b=b)
    arr = ctx.arr
    terms = ("w0", "w1", "s1", "s2", "t3", "big", "zzz")
    for t in terms:
        assert_contract(arr.score(t, similarity=sim), ctx.oracle.vec("a", t, k1=k1, b=b), f"a {t!r}")
    feats = ctx.oracle.scorer()

    def score(c):
        if isinstance(c, Field):
            return arr.score(c.clause, similarity=sim) if c.field == "a" else feats(c)
        return arr.score(c, similarity=sim)
    qs = [Bool(must=["w0"], should=["s1", Boost("w1", 2)], must_not=["t3"]), Bool(filter=["w1"], should=["w0", "big"]),
          Bool(should=[Boost("w0", 0), "s1", "zzz"], mm=1), Or(["s2", "t3"])]
    sims = sims_of(override={"a": sim})
    frame_a = ctx.frame
    for k in (1, 10, 17, 32):
        check(frame_a, qs, k, f"exotic {k1},{b}", False, score, expect(OCCUR, 0, PLAIN), sims=sims)
        check(frame_a, qs, k, f"exotic where {k1},{b}", False, score, expect(OCCUR, 1, PLAIN), masks(len(qs)),
              sims=sims)
        check(frame_a, qs, k, f"exotic count {k1},{b}", False, score, expect(OCCUR, 0, COUNT, features=False), None, ["g0", "small"],
              {"g0": ctx.codes[("a", "g0")], "small": ctx.codes[("a", "small")]}, sims=sims)
        fq = [Bool(must=[Field("a", "w0")], should=[Field("b", "b1"), Field("a", "s1")]),
              Or([Field("b", "w0"), Field("a", "big"), Field("b", "bs")], mm=2)]
        check(frame_a, fq, k, f"exotic fields {k1},{b}", True, score, expect(FIELDS, 0, PLAIN), sims=sims)
    with pytest.raises(_lib.SearchArrayB200Error, match="ordinary BM25 parameters"):
        arr.search_topk([Bool(should=[["pa", "pb"], "w0"])], k=10, similarity=sim)
    with pytest.raises((ValueError, _lib.SearchArrayB200Error)):
        arr.search_topk([Bool(should=[DisMax(["w0", "w1"])])], k=10, similarity=sim)


@pytest.mark.parametrize("count", [False, True])
def test_overflow_rerun_every_form(ctx, count):
    """A query whose tile overflows its candidate slots is re-run exactly, on every form, once; a counting call's
    re-run runs the instance without COUNT and its counts stay those of the first pass."""
    from searcharray_b200 import Bool, DisMax, Or
    A, B = _F(True, "a"), _F(True, "b")
    per_form = {OR_AND: ([Or(["hot", "cold"]), Or(["w2", "s1"])], False),
                OCCUR: ([Bool(should=["hot", "cold"], must_not=["t0"]), Bool(should=["w0"], filter=["t0"])], False),
                FIELDS: ([Or([A("hot"), A("cold"), B("zzz")]), Bool(should=[B("bs")])], True),
                DISMAX: ([Bool(should=[DisMax([A("hot"), A("cold")], tie=1.0)]), Bool(should=[A("w1")])], True),
                NESTED: ([Bool(should=[Or([A("hot"), A("cold")])]), Bool(should=[Or([A("s1")])])], True)}
    for form, (qs, fields) in per_form.items():
        facets = ([] if not fields else [("a", "g1")]) if count else None
        codes = {("a", "g1"): ctx.codes[("a", "g1")]}
        shown = COUNT if count else PLAIN
        if count and form == OR_AND:
            form_run = OCCUR                            # an Or / And that counts runs as roles and weights
        else:
            form_run = form
        for k in (10, 16):
            check(ctx.frame, qs, k, f"overflow form {form}", fields, ctx.oracle.scorer(),
                  expect(form_run, 0, shown, form == NESTED, features=False), None, facets, codes, redone=1)


def test_shard_doc_base_global_df():
    """A shard (doc_base 1,000,003, corpus size 3,000,000, avgdl 31.5, global dfs) on the fields, DisMax and nested
    forms: global ids, every clause scored with the shard's corpus size and global dfs."""
    from searcharray_b200 import And, Bool, Boost, DisMax, Field, Or, SearchArray
    base, size, avg = 1_000_003, 3_000_000, 31.5
    local = {"a": column_a(), "b": column_b()}
    hosts = {"a": column_a(doc_base=base), "b": column_b(doc_base=base)}
    gdf = {c: np.asarray([int(h.term_lengths[i]) + 1000 * (i + 1) for i in range(h.n_terms)], dtype=np.uint64)
           for c, h in local.items()}
    frame = pd.DataFrame({c: SearchArray.from_host_index(h, doc_base=base, corpus_size=size, avg_doc_length=avg,
                                                         global_df=gdf[c]) for c, h in hosts.items()})
    oracle = Oracle(local, {"a": avg, "b": avg}, shard=(size, avg, gdf))
    A, B = (lambda c: Field("a", c)), (lambda c: Field("b", c))
    qs = {FIELDS: [Bool(must=[A("w0")], should=[B("b1"), A("s1")]), Or([A(["pa", "pb"]), B("bs"), A("big")], mm=1),
                   Bool(filter=[A("t3")], should=[Boost(B("w0"), 2)], must_not=[B("b2")])],
          DISMAX: [Bool(should=[DisMax([A("w0"), B("w0")], tie=0.2), DisMax([A("s2"), B("bs"), A("t0")])], mm=1),
                   Or([DisMax([A(["pa", "pb"]), B(["qa", "qb"])], tie=1.0), A("t5")])],
          NESTED: [Bool(must=[Or([A("w1"), And([B("b1"), A("s1")])])], should=[Boost(Or([A("t3"), B("bs")]), 3)]),
                   Or([And([A("w0"), Or([B("b2"), A("zzz")])]), DisMax([A("s2"), B("qa")], tie=0.5)])]}
    for form, q in qs.items():
        for k in (1, 10, 32):
            check(frame, q, k, f"shard form {form}", True, oracle.scorer(), expect(form, 0, PLAIN, form == NESTED),
                  sims=sims_of({"a": SIMS["a"], "b": SIMS["b"]}), doc_base=base)


def test_feature_values_refused_before_the_kernel(ctx):
    """NaN, inf and negative feature values never reach the fold: the index refuses them."""
    from searcharray_b200 import _lib
    for bad in (np.nan, np.inf, -1.0, -1e-45):
        v = ctx.features["pop"].copy()
        v[123] = bad
        with pytest.raises(ValueError):
            ctx.arr.set_feature("bad", v)
        h = ctx.arr._device().handle
        assert _lib.lib().sa_index_set_feature(h, 15, _lib.p_f32(v), len(v)) != 0


# --------------------------------------------------------------------------------------------- launch groups
def _big_case(n, seed):
    """n docs: `x` (records), `y` (binary search), phrase terms `pa` / `pb`, and `hot` / `cold`: tile 1's best 1,024
    docs all owned by warp 0, so that the tile bound comes from the other warps' lower maxima and its candidates
    overflow 256 slots (k = 32)."""
    from searcharray_b200 import SearchArray
    rng = np.random.default_rng(seed)
    doc_lens = rng.integers(1, 40, n).astype(np.float32)
    postings, add = _postings(n, rng)
    add("x", np.sort(rng.choice(n, n // 20, replace=False)), lambda doc: [3])
    add("y", np.sort(rng.choice(n, 400, replace=False)), lambda doc: [5])
    ph = np.sort(rng.choice(n, 20000, replace=False))
    add("pa", ph, lambda doc: [7])
    add("pb", ph[::2], lambda doc: [8])
    hot = TILE + np.asarray([4 * t + e + 1024 * j for t in range(32) for e in range(4) for j in range(8)])
    add("hot", hot, lambda doc: list(range(40, 42 + doc % 5)))
    add("cold", np.setdiff1d(TILE + rng.choice(TILE, 1500, replace=False), hot), lambda doc: [40])
    host = _host(postings, doc_lens, 0)
    return host, SearchArray.from_host_index(host)


def test_group_split_by_candidate_slots():
    """~4M docs at k = 32: 1,067 queries per launch group, so a batch of 1,100 is two launches.  Per-query mask
    rows, counts and an overflowing query in the second group check the per-group offsets of the mask rows, the
    totals and facet rows and the overflow flags."""
    from searcharray_b200 import Bool, Or
    from searcharray_b200.postings import pack_where
    n, nq, k = 4_000_000, 1100, 32
    host, arr = _big_case(n, 41)
    fac = np.random.default_rng(2).integers(-1, 1024, n).astype(np.int32)
    arr.set_facet("f", fac, n_buckets=1024)
    oracle = Oracle({"a": host}, {"a": arr.avg_doc_length})
    pats = np.zeros((3, n), dtype=bool)
    pats[0] = np.random.default_rng(8).random(n) < 0.6
    pats[1, 2 * TILE:n // 2] = True
    pats[2] = True
    templates = [Bool(should=["x", "y"], mm=1), Or(["x", "y"], mm=2), Bool(must=["x"], must_not=["y"])]
    over = 1090                                              # in the second group
    queries = [templates[i % 3] for i in range(nq)]
    queries[over] = Bool(should=["hot", "cold"])
    packed = pack_where(pats, n, 3)[[i % 3 if i != over else 2 for i in range(nq)]]
    from searcharray_b200 import _lib
    h = arr._device().handle
    _lib.check(_lib.lib().sa_stats_reset(h))
    docs, scores, n_redone, hits = arr._search_topk_bool(queries, k, sims_of()["a"], 0, packed, ["f"])
    st = _lib.SaStats()
    _lib.check(_lib.lib().sa_stats_get(h, ctypes.byref(st)))
    RAN.update(i for i in range(64) if st.bool_instances >> i & 1)
    assert st.bool_instances == bit(OCCUR, 1, COUNT) | bit(OCCUR, 1, PLAIN), hex(st.bool_instances)
    assert n_redone == 1
    score = oracle.scorer()
    want = {}
    for i, q in enumerate(queries):
        key = (repr(q), i % 3 if i != over else 2)
        if key not in want:
            dense = np.where(pats[key[1]], compose_nested(score, q), np.float32(0)).astype(np.float32)
            r = dense > 0
            want[key] = topk(dense, k) + (int(r.sum()), np.bincount(fac[r & (fac >= 0)], minlength=1024))
        wd, ws, total, counts = want[key]
        tag = f"query {i} {q!r} mask {key[1]}"
        assert np.array_equal(docs[i], wd), f"{tag}: ids {docs[i]} want {wd}"
        assert np.array_equal(scores[i].view(np.uint32), ws.view(np.uint32)), f"{tag}: score bits"
        assert hits.total[i] == total, f"{tag}: total {hits.total[i]} want {total}"
        assert np.array_equal(hits.facets["f"][i], counts), f"{tag}: facet counts"


def test_nested_group_split_by_phrase_rows():
    """~2M docs: nested queries with 63 phrase rows and a nested node each, more than the 512 rows of one ~4 GB group:
    node rows are numbered within each launch group."""
    from searcharray_b200 import Bool, Or
    n = 2_000_000
    host, arr = _big_case(n, 43)
    oracle = Oracle({"a": host}, {"a": arr.avg_doc_length})
    queries = [Bool(should=[Or([["pa", "pb"]] * 62 + ["x" if i % 2 else "y"], mm=1), ["pa", "pb"]], mm=1 + i % 2)
               for i in range(9)]                                                  # 9 x 64 rows
    first, _ = expect(NESTED, 0, PLAIN, True)
    docs, scores, n_redone, _, inst = run(pd.DataFrame({"a": arr}), queries, 10, False)
    assert inst == first, hex(inst)
    score = oracle.scorer()
    cache = {}
    for i, q in enumerate(queries):
        assert_topk(docs[i], scores[i], compose_nested(score, q, cache), 10, f"2M nested #{i}")


# ------------------------------------------------------------------------------------------ SA_NO_TF_TABLE
def check_records_paths(ctx, what):
    """The records-term and tf = 2^18 checks (in the worker: the words path over a tile directory)."""
    from searcharray_b200 import And, Bool, Boost, DisMax, Field, Or
    score = ctx.oracle.scorer()
    qs = [Or(["big", "w0"], mm=2), Bool(must=["big"], should=[Boost("w1", 2)]), Bool(should=["big"], must_not=["w2"]),
          And(["w0", "w1"]), Or(["big"])]
    for k in KS:
        check(ctx.frame, qs[:3] + qs[4:], k, what, False, score, expect(OCCUR, 0, PLAIN))
        check(ctx.frame, qs[3:4], k, what, False, score, expect(OR_AND, 0, PLAIN))
        fq = [Bool(should=[DisMax([Field("a", "big"), Field("b", "b1")], tie=0.5), Field("a", "w2")]),
              Or([Field("a", "big"), Field("b", "w0")])]
        check(ctx.frame, fq, k, what + " dismax", True, score, expect(DISMAX, 0, PLAIN))
        check(ctx.frame, qs, k, what + " masked", False, score, expect(OCCUR, 1, PLAIN), masks(len(qs)))
    docs, _ = ctx.arr.search_topk([Bool(should=["big"])], k=2)
    assert sorted(docs[0].tolist()) == list(BIG_DOCS), f"{what}: tf 2^18 docs {docs[0]}"


def test_records_and_tf_2_18(ctx):
    check_records_paths(ctx, "records")


def test_words_path_with_directory():
    """The records-term and tf = 2^18 checks in a process with SA_NO_TF_TABLE=1."""
    env = dict(os.environ, SA_NO_TF_TABLE="1")
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_bool_paths_worker.py")
    r = subprocess.run([sys.executable, worker], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.strip().splitlines()[-1] == "OK", r.stdout[-3000:]


def test_every_instance_ran(ctx):
    """The union of bool_instances over this module is all 26 instances (the instance checks run here for any this
    session's selection skipped)."""
    for form, masked, variant in INSTANCES:
        if variant * 10 + form * 2 + masked not in RAN:
            test_instance(ctx, form, masked, variant)
    want = {variant * 10 + form * 2 + masked for form, masked, variant in INSTANCES}
    assert len(want) == 26 and RAN >= want, sorted(want - RAN)
    assert RAN == want, sorted(RAN - want)
