"""GPU: boolean queries over several DataFrame fields (solr.fields_topk, sa_multi_score_batch_topk_bool, the FIELDS
instance of bool_tile_kernel in sa_bool.cu) against compose_occur with each clause scored by its own column's .score: ids
and float32 score bits must be equal.

The synthetic frame spans five 8192-doc tiles and has fields that differ in vocabulary, doc lengths and avgdl:
`fa` is test_bool_topk_gpu.py's corpus (doc lengths 1..59; `w0` / `w1` / `w2` with a tile directory and a tf table,
`s1` / `s2` on the binary-search path, `t0` / `t3` in one tile each, `pa` / `pb` phrases, `hot` / `cold` overflowing a
tile's candidate slots); `fb` (doc lengths 20..299) shares `w0` and the phrase terms `pa` / `pb` with other postings
and has its own `b1` (tf table), `bs` (binary search), `b2` (tile 2 only) and phrase `qa qb`.  The role checks run
again in a child process with SA_NO_TF_TABLE=1 (tests/_bool_fields_worker.py), where the long lists take the words
path with a tile directory."""
import ctypes
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pandas as pd
import pytest

from _bool_fields_compose import field_scorer, query_of, record_groups
from _bool_occur_compose import compose_occur
from _tmdb_index import load_field
from conftest import GOLDEN
from test_bool_topk_gpu import KS, TILE, assert_topk, synth_corpus

pytestmark = pytest.mark.gpu

A, B, Z = "fa", "fb", "fz"


def fb_corpus(n=5 * TILE + 300, doc_base=0, seed=23):
    from searcharray_b200.indexing import index_from_term_postings
    from searcharray_b200.roaringish import encode_postings
    rng = np.random.default_rng(seed)
    doc_lens = rng.integers(20, 300, n).astype(np.float32)
    postings = {}

    def add(name, docs, posns_of):
        d, p = [], []
        for doc in np.unique(np.asarray(docs, dtype=np.int64)):
            ps = sorted(set(posns_of(doc)))
            d += [doc] * len(ps)
            p += ps
        postings[name] = (np.asarray(d, dtype=np.int64), np.asarray(p, dtype=np.int64))

    def rand_posns(doc):
        return rng.integers(5, 250, rng.integers(1, 5)).tolist()

    add("w0", np.flatnonzero(rng.random(n) < 0.3), rand_posns)
    add("b1", np.flatnonzero(rng.random(n) < 0.5), rand_posns)
    add("bs", rng.choice(np.arange(TILE, n), 700, replace=False), rand_posns)
    add("b2", 2 * TILE + rng.choice(TILE, 1500, replace=False), rand_posns)
    ph = rng.choice(n, 4000, replace=False)
    add("pa", ph, lambda doc: [20, 21] if doc % 3 == 0 else [20])
    add("pb", ph[::2], lambda doc: [21] if doc % 2 else [23])
    qd = rng.choice(n, 2500, replace=False)
    add("qa", qd, lambda doc: [7])
    add("qb", qd[: 1800], lambda doc: [8] if doc % 4 else [9])
    names = list(postings)
    words = [encode_postings(d + doc_base, p) for d, p in (postings[t] for t in names)]
    return index_from_term_postings(names, words, doc_lens), names


class Frame:
    def __init__(self):
        from searcharray_b200 import SearchArray
        ha, _ = synth_corpus()
        hb, _ = fb_corpus()
        self.frame = pd.DataFrame({A: SearchArray.from_host_index(ha), B: SearchArray.from_host_index(hb)})
        # the same postings as fb under avgdl 0: .score is 0 everywhere
        self.frame[Z] = SearchArray.from_host_index(hb, avg_doc_length=0.0)

    def score(self, sims=None, slop=0):
        from searcharray_b200 import bm25_similarity
        sims = sims or {}
        return field_scorer({f: (lambda c, f=f: self.frame[f].array.score(c, similarity=sims.get(f, bm25_similarity()),
                                                                         slop=slop))
                             for f in self.frame.columns})


@pytest.fixture(scope="module")
def synth():
    return Frame()


def check_batch(frame, queries, k, score, what, doc_base=0, slop=0, similarity=None):
    """fields_topk(queries) against compose_occur(score, q) for every query of the batch."""
    from searcharray_b200 import bm25_similarity, fields_topk
    docs, scores = fields_topk(frame, queries, k=k, similarity=similarity or bm25_similarity(), slop=slop)
    assert docs.shape == (len(queries), k) and docs.dtype == np.uint32 and scores.dtype == np.float32
    for i, q in enumerate(queries):
        assert_topk(docs[i], scores[i], compose_occur(score, q), k, f"{what} {q!r} k={k}", doc_base)
    return docs, scores


def role_queries(F):
    """Cross-field term clauses in every role, boosts, duplicates and unknown tokens; F(field, clause) makes a
    clause."""
    from searcharray_b200 import And, Bool, Boost, Or
    return [
        Bool(must=[F(A, "w0")], should=[F(B, "w0"), F(B, "bs")], mm=0),
        Bool(must=[F(B, "b1")], should=[F(A, "w1"), F(A, "s1"), F(B, "w0")], mm=2),
        Bool(must=[F(A, "s2")], should=[F(B, "b1")]),                       # MUST on fa's binary-search path
        Bool(filter=[F(B, "b2")], should=[F(A, "w0"), F(A, "s1")]),         # FILTER on fb's tile 2 only
        Bool(should=[F(A, "w0"), F(B, "w0")], must_not=[F(B, "b1")]),
        Bool(should=[F(B, "bs"), F(A, "s2")], must_not=[F(A, "t0")]),
        Bool(must=[Boost(F(A, "w0"), 0.5)], should=[Boost(F(B, "w0"), 2), Boost(F(A, "s1"), 0)], filter=[F(B, "b1")],
             must_not=[F(A, "t3")], mm=1),
        Bool(must=[Boost(F(B, "b2"), 0)], should=[F(A, "w0")]),             # a zero weight still requires a match
        Bool(must=[F(A, "w0"), F(A, "w0")], should=[F(B, "bs"), F(B, "bs")], must_not=[F(B, "b2"), F(B, "b2")],
             filter=[F(B, "b1"), F(B, "b1")], mm=1),
        Bool(must=[F(B, "zzz")], should=[F(A, "w0")]),
        Bool(should=[F(A, "w0"), F(B, "s1")], must_not=[F(A, "zzz")]),       # s1 is unknown in fb
        Or([Boost(F(A, "w0"), 2), F(B, "w0")]),                              # most_fields
        Or([F(A, "w1"), F(B, "b1"), F(B, "bs")], mm=2),
        And([F(A, "w2"), Boost(F(B, "b1"), 3)]),
    ]


def fld(f, c):
    from searcharray_b200 import Field
    return Field(f, c)


def check_roles(frame, score, what):
    for k in KS:
        check_batch(frame, role_queries(fld), k, score, f"{what} k={k}")


def test_roles_terms(synth):
    check_roles(synth.frame, synth.score(), "fields")


def test_roles_words_path_with_directory():
    """The role checks in a process with SA_NO_TF_TABLE=1: every long list on the words path with a tile
    directory."""
    env = dict(os.environ, SA_NO_TF_TABLE="1")
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_bool_fields_worker.py")
    r = subprocess.run([sys.executable, worker], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.strip().splitlines()[-1] == "OK", r.stdout[-3000:]


def test_one_field_equals_search_topk(synth):
    """Every clause on one field: fields_topk gives that column's search_topk ids and score bits, for Bool, Or and
    And, phrases included."""
    from searcharray_b200 import And, Bool, Or
    arr = synth.frame[A].array
    plain = role_queries(lambda f, c: c) + [Or(["w0", "s1"]), And(["w1", "w2"]), Or([["pa", "pb"], "t3"], mm=1),
                                            Bool(must=[["pa", "pb"]], should=["w0"])]
    fielded = role_queries(lambda f, c: fld(A, c)) + [
        Or([fld(A, "w0"), fld(A, "s1")]), And([fld(A, "w1"), fld(A, "w2")]),
        Or([fld(A, ["pa", "pb"]), fld(A, "t3")], mm=1), Bool(must=[fld(A, ["pa", "pb"])], should=[fld(A, "w0")])]
    from searcharray_b200 import fields_topk
    for slop in (0, 2):
        for k in (1, 10, 32):
            wd, ws = arr.search_topk(plain, k=k, slop=slop)
            gd, gs = fields_topk(synth.frame, fielded, k=k, slop=slop)
            assert np.array_equal(gd, wd) and np.array_equal(gs.view(np.uint32), ws.view(np.uint32)), (slop, k)


@pytest.mark.parametrize("slop", [0, 2])
def test_phrases(synth, slop):
    from searcharray_b200 import Bool, Boost, Or
    F = fld
    queries = [Bool(must=[F(A, ["pa", "pb"])], should=[F(B, "w0"), F(A, "w1")]),
               Bool(should=[F(B, "w0"), F(A, "w2")], filter=[F(B, ["qa", "qb"])]),
               Bool(should=[F(A, "w0"), F(B, "b1")], must_not=[F(B, ["qa", "qb"])]),
               Or([Boost(F(A, ["pa", "pb"]), 2), Boost(F(B, ["qa", "qb"]), 0.5), F(B, ["pa", "pb"])]),
               Bool(must=[F(B, ["qa", "zzz"])], should=[F(A, "w0")]),
               Bool(must=[F(B, ["pa", "pb"])], should=[F(A, ["pa", "pb"]), F(A, "s1")], must_not=[F(A, "t3")], mm=1)]
    for k in KS:
        check_batch(synth.frame, queries, k, synth.score(slop=slop), f"slop={slop}", slop=slop)


def test_similarity_dict(synth):
    """Per-field parameters, including ones that are not sparse-safe on one field (NaN / -0.0 / negative scores
    there), with a phrase on the other field."""
    from searcharray_b200 import Bool, Boost, Or, bm25_similarity
    F = fld
    for sims in ({A: bm25_similarity(k1=0.9, b=0.4), B: bm25_similarity(k1=1.8, b=0.9)},
                 {A: bm25_similarity(k1=1.2, b=1.0)}, {A: bm25_similarity(k1=0.0)},
                 {B: bm25_similarity(k1=1.2, b=1.5)}):
        queries = role_queries(fld)
        if B not in sims or sims[B].b < 1:
            queries += [Bool(must=[F(B, ["qa", "qb"])], should=[F(A, "w0"), Boost(F(A, "s1"), 2)]),
                        Or([F(A, "zzz"), F(B, ["pa", "pb"])])]
        for k in (1, 10, 32):
            check_batch(synth.frame, queries, k, synth.score(sims), f"sims={sims}", similarity=sims)
    # one similarity for every field
    sim = bm25_similarity(k1=2.0, b=0.3)
    check_batch(synth.frame, role_queries(fld), 10, synth.score({A: sim, B: sim}), "one sim", similarity=sim)


def test_zero_avgdl_field(synth):
    """A field whose avgdl is 0 scores 0 everywhere: a MUST / FILTER clause on it ranks nothing, a MUST_NOT clause on
    it vetoes nothing, phrases on it are accepted."""
    from searcharray_b200 import Bool, Or, fields_topk
    F = fld
    queries = [Bool(must=[F(Z, "w0")], should=[F(A, "w0")]), Bool(filter=[F(Z, ["qa", "qb"])], should=[F(A, "w1")]),
               Bool(should=[F(A, "w0"), F(B, "b2")], must_not=[F(Z, "b1"), F(Z, ["pa", "pb"])]),
               Or([F(Z, "b1"), F(A, "w1"), F(Z, ["qa", "qb"])]), Or([F(Z, "w0"), F(A, "t3")], mm=2)]
    for k in (1, 10, 32):
        docs, _ = check_batch(synth.frame, queries, k, synth.score(), "zero avgdl")
        assert np.all(docs[[0, 1, 4]] == 0xFFFFFFFF) and np.all(docs[[2, 3], 0] != 0xFFFFFFFF)
    d, s = fields_topk(synth.frame, [Or([F(Z, "w0"), F(Z, ["pa", "pb"])])], k=10)
    assert np.all(d == 0xFFFFFFFF) and np.all(s == 0)


def test_overflow_rerun(synth):
    """Queries whose tile overflows its candidate slots are re-run exactly."""
    from searcharray_b200 import Bool, Boost, bm25_similarity
    from searcharray_b200.solr import _fields_topk
    F = fld
    queries = [Bool(should=[F(A, "hot"), F(A, "cold")], must_not=[F(B, "b2")]),
               Bool(must=[F(A, "hot")], should=[Boost(F(B, "zzz"), 2), F(A, "cold")]),
               Bool(filter=[F(B, "b1")], should=[F(A, "w0")])]
    for k in (10, 16):
        docs, scores, n_redone = _fields_topk(synth.frame, queries, k, bm25_similarity(), 0)
        assert n_redone > 0
        for i, q in enumerate(queries):
            assert_topk(docs[i], scores[i], compose_occur(synth.score(), q), k, f"overflow {q!r} k={k}")


def test_shard_doc_base_global_df():
    from searcharray_b200 import Bool, Boost, Or, SearchArray
    F = fld
    base = 1_000_003
    la, na = synth_corpus()
    lb, nb = fb_corpus()
    ha, _ = synth_corpus(doc_base=base)
    hb, _ = fb_corpus(doc_base=base)
    ga = np.asarray([int(la.term_lengths[i]) + 1000 * (i + 1) for i in range(len(na))], dtype=np.uint64)
    gb = np.asarray([int(lb.term_lengths[i]) + 700 * (i + 2) for i in range(len(nb))], dtype=np.uint64)
    frame = pd.DataFrame({A: SearchArray.from_host_index(ha, doc_base=base, corpus_size=3_000_000, avg_doc_length=31.5,
                                                         global_df=ga),
                          B: SearchArray.from_host_index(hb, doc_base=base, corpus_size=3_000_000,
                                                         avg_doc_length=150.25, global_df=gb)})
    score = field_scorer({f: (lambda c, f=f: frame[f].array.score(c)) for f in (A, B)})
    queries = [Bool(must=[F(A, "w0")], should=[F(B, "w0"), F(B, "bs")]), Bool(should=[F(A, "w0"), F(B, "b1")],
                                                                              must_not=[F(A, "s1")]),
               Bool(filter=[F(B, "b2")], should=[Boost(F(A, "w0"), 2)]), Or([Boost(F(A, ["pa", "pb"]), 3), F(B, "bs")]),
               Bool(must=[F(B, ["qa", "qb"])], should=[F(A, "w1")], must_not=[F(A, "w2")])]
    for k in (1, 10, 32):
        check_batch(frame, queries, k, score, "shard", doc_base=base)


def test_batch_spans_two_groups():
    """~2M docs, two fields: a batch with more phrase clauses than one ~4 GB group of rows holds (512 rows of 8 MB),
    rows built on both fields."""
    from searcharray_b200 import Or, SearchArray
    from searcharray_b200.indexing import index_from_term_postings
    from searcharray_b200.roaringish import encode_postings
    rng = np.random.default_rng(5)
    n = 2_000_000

    def field(seed_shift, lo, hi):
        docs = np.sort(rng.choice(n, 20000, replace=False))
        pa = encode_postings(docs, np.full(len(docs), 3 + seed_shift))
        pb = encode_postings(docs[::2], np.full(len(docs[::2]), 4 + seed_shift))
        x_docs = np.sort(rng.choice(n, 50000, replace=False))
        x = encode_postings(x_docs, np.full(len(x_docs), 7))
        return SearchArray.from_host_index(index_from_term_postings(["pa", "pb", "x"], [pa, pb, x],
                                                                    rng.integers(lo, hi, n).astype(np.float32)))
    frame = pd.DataFrame({A: field(0, 1, 30), B: field(5, 10, 90)})
    score = field_scorer({f: (lambda c, f=f: frame[f].array.score(c)) for f in (A, B)})
    queries = [Or([fld(A, ["pa", "pb"])] * 31 + [fld(B, ["pa", "pb"])] * 32 + [fld(B if i % 2 else A, "x")],
                  mm=1 + i % 2) for i in range(9)]                                   # 567 phrase rows
    check_batch(frame, queries, 10, score, "2M docs")


def test_golden():
    """The real reference's composed top 10 of every record, on the TMDB title and overview fields: ids and score
    bits, and the same against this library's per-field .score at every k."""
    from searcharray_b200 import SearchArray, bm25_similarity, fields_topk
    with open(os.path.join(GOLDEN, "bool_fields.json")) as f:
        fixture = json.load(f)
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    frame = pd.DataFrame({f: SearchArray.from_host_index(load_field(z, f)) for f in ("title_tokens", "overview_tokens")})
    for group in record_groups(fixture["queries"]).values():
        r0 = group[0]
        sims = {f: bm25_similarity(k1=kb[0], b=kb[1]) for f, kb in r0["sim"].items()}
        queries = [query_of(r) for r in group]
        docs, scores = fields_topk(frame, queries, k=10, similarity=sims, slop=r0["slop"])
        for i, r in enumerate(group):
            n = len(r["top_ids"])
            what = f"{queries[i]!r} slop={r['slop']} sim={r['sim']}"
            assert docs[i][:n].tolist() == r["top_ids"], what
            assert scores[i][:n].view(np.uint32).tolist() == r["top_bits"], what
            assert np.all(docs[i][n:] == 0xFFFFFFFF), what
        score = field_scorer({f: (lambda c, f=f: frame[f].array.score(
            c, similarity=sims.get(f, bm25_similarity()), slop=r0["slop"])) for f in frame.columns})
        for k in KS:
            check_batch(frame, queries, k, score, "tmdb", slop=r0["slop"], similarity=sims)


def test_threads_mix_fields_topk_and_score(synth):
    """Three threads on the same columns: two run fields_topk, one .score on both fields; every result equals the
    one computed alone."""
    from searcharray_b200 import fields_topk
    frame = synth.frame
    qa, qb = role_queries(fld)[:7], role_queries(fld)[7:]
    want_a = fields_topk(frame, qa, k=10)
    want_b = fields_topk(frame, qb, k=10, slop=2)
    want_s = [(f, t, frame[f].array.score(t).copy()) for f, t in ((A, "w0"), (B, "b1"), (A, ["pa", "pb"]),
                                                                   (B, ["qa", "qb"]))]
    errors = []

    def run(fn):
        try:
            for _ in range(8):
                fn()
        except Exception as e:                      # noqa: BLE001 -- reported below
            errors.append(repr(e))

    def same(got, want):
        return np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))

    def t_a():
        assert same(fields_topk(frame, qa, k=10), want_a)

    def t_b():
        assert same(fields_topk(frame, qb, k=10, slop=2), want_b)

    def t_s():
        for f, t, w in want_s:
            assert np.array_equal(frame[f].array.score(t).view(np.uint32), w.view(np.uint32))
    ts = [threading.Thread(target=run, args=(fn,)) for fn in (t_a, t_b, t_s)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors


def test_c_abi_validation(synth):
    """The entry point checks each clause's field slot and term ids against that field, and refuses one index under
    two parameter sets."""
    from searcharray_b200 import _lib
    from searcharray_b200.solr import _Multi
    a, b = synth.frame[A].array, synth.frame[B].array
    ta, tb = a.host.term_dict.term_to_ids, b.host.term_dict.term_to_ids
    docs = np.empty(10, dtype=np.uint32)
    scores = np.empty(10, dtype=np.float32)

    def call(multi, fields, terms, avgdl, k1=(1.2, 1.2)):
        q_starts = np.asarray([0, len(terms)], dtype=np.uint32)
        c_starts = np.arange(len(terms) + 1, dtype=np.uint32)
        f = np.asarray(fields, dtype=np.uint32)
        t = np.asarray(terms, dtype=np.uint32)
        ones = np.ones(len(terms), dtype=np.float32)
        occ = np.zeros(len(terms), dtype=np.uint8)
        mm = np.asarray([1], dtype=np.uint32)
        avgdl = np.asarray(avgdl, dtype=np.float32)
        kk, bb = np.asarray(k1, dtype=np.float32), np.full(len(k1), 0.75, dtype=np.float32)
        return _lib.lib().sa_multi_score_batch_topk_bool(
            multi.handle, 1, _lib.p_u32(q_starts), None, _lib.p_u32(f), _lib.p_u32(t), _lib.p_u32(c_starts),
            _lib.p_f32(ones), _lib.p_f32(ones), _lib.p_u8(occ), None, None, _lib.p_u32(mm), 1, 0, _lib.p_f32(avgdl),
            _lib.p_f32(kk), _lib.p_f32(bb), 10, None, 0, 0, _lib.p_u32(docs), _lib.p_f32(scores), None,
            0, None, None, None, None)
    m, ab = _Multi([a, b]), (a.avg_doc_length, b.avg_doc_length)
    assert call(m, [0, 1], [ta["w0"], tb["b1"]], ab) == 0
    assert call(m, [0, 2], [ta["w0"], tb["b1"]], ab) != 0                 # no field slot 2
    assert call(m, [0, 0], [ta["w0"], b.host.n_terms + a.host.n_terms], ab) != 0   # a term id out of fa's range
    same, aa = _Multi([a, a]), (a.avg_doc_length, a.avg_doc_length)
    assert call(same, [0, 1], [ta["w0"], ta["w1"]], aa) == 0             # one index, one parameter set: locked once
    assert call(same, [0, 1], [ta["w0"], ta["w1"]], aa, k1=(1.2, 2.0)) != 0
    assert call(same, [0, 1], [ta["w0"], ta["w1"]], ab) != 0
    assert b"share an index" in _lib.lib().sa_last_error()


def test_c_abi_pairings(synth):
    """The nullable arrays alone select the form, so a pairing no form takes is SA_ERR_ARG before any device work:
    weights without roles, groups without ties or without roles, clause_node without groups, n_nodes != n_queries
    without clause_node, and on the multi-field entry NULL weights or roles.  The same call with the pairing
    completed runs."""
    from searcharray_b200 import _lib
    from searcharray_b200.solr import _Multi
    a, b = synth.frame[A].array, synth.frame[B].array
    ta, tb = a.host.term_dict.term_to_ids, b.host.term_dict.term_to_ids
    docs = np.empty(10, dtype=np.uint32)
    scores = np.empty(10, dtype=np.float32)
    n_starts = np.asarray([0, 2], dtype=np.uint32)
    c_starts = np.arange(3, dtype=np.uint32)
    ones = np.ones(2, dtype=np.float32)
    occ = np.zeros(2, dtype=np.uint8)
    groups = np.arange(2, dtype=np.uint32)
    ties = np.zeros(2, dtype=np.float32)
    nodes = np.full(2, 0xFFFFFFFF, dtype=np.uint32)
    mm = np.asarray([1], dtype=np.uint32)
    opt = lambda x, p: None if x is None else p(x)      # noqa: E731

    def single(w, o, g, t, node, n_nodes=1):
        terms = np.asarray([ta["w0"], ta["w1"]], dtype=np.uint32)
        return _lib.lib().sa_score_batch_topk_bool(
            a._device().handle, n_nodes, _lib.p_u32(n_starts), opt(node, _lib.p_u32), _lib.p_u32(terms),
            _lib.p_u32(c_starts), _lib.p_f32(ones), opt(w, _lib.p_f32), opt(o, _lib.p_u8), opt(g, _lib.p_u32),
            opt(t, _lib.p_f32), _lib.p_u32(mm), 1, 0, a.avg_doc_length, 1.2, 0.75, 10, None, 0, 0, _lib.p_u32(docs),
            _lib.p_f32(scores), None, 0, None, None, None, None)
    assert single(None, None, None, None, None) == 0
    assert single(ones, occ, None, None, None) == 0
    assert single(ones, occ, groups, ties, None) == 0
    assert single(ones, occ, groups, ties, nodes) == 0
    assert single(ones, None, None, None, None) == 2                          # weights without roles
    assert b"clause_weight and clause_occur" in _lib.lib().sa_last_error()
    assert single(None, occ, None, None, None) == 2
    assert single(ones, occ, groups, None, None) == 2                         # groups without ties
    assert b"clause_group and clause_tie" in _lib.lib().sa_last_error()
    assert single(None, None, groups, ties, None) == 2                        # groups without roles
    assert b"clause_group and clause_tie" in _lib.lib().sa_last_error()
    assert single(ones, occ, None, None, nodes) == 2                          # clause_node without groups
    assert b"clause_node needs the DisMax arrays" in _lib.lib().sa_last_error()
    assert single(ones, occ, groups, ties, None, n_nodes=2) == 2              # n_nodes != n_queries without clause_node
    assert b"n_nodes == n_queries" in _lib.lib().sa_last_error()

    def multi(w, o, g=None, t=None):
        f = np.asarray([0, 1], dtype=np.uint32)
        terms = np.asarray([ta["w0"], tb["b1"]], dtype=np.uint32)
        avgdl = np.asarray([a.avg_doc_length, b.avg_doc_length], dtype=np.float32)
        kk, bb = np.full(2, 1.2, dtype=np.float32), np.full(2, 0.75, dtype=np.float32)
        return _lib.lib().sa_multi_score_batch_topk_bool(
            mh.handle, 1, _lib.p_u32(n_starts), None, _lib.p_u32(f), _lib.p_u32(terms), _lib.p_u32(c_starts),
            _lib.p_f32(ones), opt(w, _lib.p_f32), opt(o, _lib.p_u8), opt(g, _lib.p_u32), opt(t, _lib.p_f32),
            _lib.p_u32(mm), 1, 0, _lib.p_f32(avgdl), _lib.p_f32(kk), _lib.p_f32(bb), 10, None, 0, 0,
            _lib.p_u32(docs), _lib.p_f32(scores), None, 0, None, None, None, None)
    mh = _Multi([a, b])
    assert multi(ones, occ) == 0
    assert multi(ones, occ, groups, ties) == 0
    assert multi(None, occ) == 2                                              # NULL weights
    assert b"NULL argument" in _lib.lib().sa_last_error()
    assert multi(ones, None) == 2                                             # NULL roles
    assert multi(None, None) == 2
    assert multi(ones, occ, groups, None) == 2
    assert b"clause_group and clause_tie" in _lib.lib().sa_last_error()


def test_launches_one_tile_launch_per_group(synth):
    """A term-only multi-field batch is one tile launch and one select, whatever the number of queries."""
    from searcharray_b200 import Bool, Boost, _lib, fields_topk
    h = synth.frame[A].array._device().handle
    launches = []
    for nq in (1, 4, 64):
        queries = [Bool(must=[fld(A, "w0")], should=[Boost(fld(B, "b1"), 2), fld(A, "s1")], must_not=[fld(B, "b2")],
                        mm=i % 3) for i in range(nq)]
        fields_topk(synth.frame, queries, k=10)              # warm: both norm tables for these parameters
        _lib.check(_lib.lib().sa_stats_reset(h))
        fields_topk(synth.frame, queries, k=10)
        st = _lib.SaStats()
        _lib.check(_lib.lib().sa_stats_get(h, ctypes.byref(st)))
        launches.append(st.total_launches)
    assert launches == [2, 2, 2], launches
