"""GPU: disjunction-max clauses (query.DisMax; sa_score_batch_topk_bool and sa_multi_score_batch_topk_bool with
groups, the DISMAX instances of bool_tile_kernel in sa_bool.cu) against compose_dismax with each clause scored by this library's .score: ids
and float32 score bits must be equal.

The synthetic frame is tests/test_bool_fields_gpu.py's: five 8192-doc tiles, `fa` (`w0` / `w1` / `w2` with a tile
directory and a tf table, `s1` / `s2` on the binary-search path, `t0` / `t3` in one tile each, `pa` / `pb` phrases,
`hot` / `cold` overflowing a tile's candidate slots) and `fb` (`b1`, `bs`, `b2` in tile 2 only, phrase `qa qb`), plus
`fz`, fb's postings under avgdl 0.  The role checks run again in a child process with SA_NO_TF_TABLE=1
(tests/_dismax_worker.py), where the long lists take the words path with a tile directory."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest

from _bool_fields_compose import field_scorer
from _dismax_compose import compose_dismax, query_of, record_groups
from _tmdb_index import load_field
from conftest import GOLDEN
from test_bool_fields_gpu import A, B, Z, Frame, fb_corpus
from test_bool_topk_gpu import KS, assert_topk, synth_corpus

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def synth():
    return Frame()


def fld(f, c):
    from searcharray_b200 import Field
    return Field(f, c)


def check_batch(frame, queries, k, score, what, doc_base=0, slop=0, similarity=None):
    """fields_topk(queries) against compose_dismax(score, q) for every query of the batch."""
    from searcharray_b200 import bm25_similarity, fields_topk
    docs, scores = fields_topk(frame, queries, k=k, similarity=similarity or bm25_similarity(), slop=slop)
    assert docs.shape == (len(queries), k) and docs.dtype == np.uint32 and scores.dtype == np.float32
    for i, q in enumerate(queries):
        assert_topk(docs[i], scores[i], compose_dismax(score, q), k, f"{what} {q!r} k={k}", doc_base)
    return docs, scores


def check_single(arr, queries, k, what, slop=0, doc_base=0):
    """search_topk(queries) on one column against compose_dismax over its .score."""
    docs, scores = arr.search_topk(queries, k=k, slop=slop)
    for i, q in enumerate(queries):
        assert_topk(docs[i], scores[i], compose_dismax(lambda c: arr.score(c, slop=slop), q), k,
                    f"{what} {q!r} k={k}", doc_base)
    return docs, scores


def dismax_queries(F):
    """DisMax groups in every role over the synthetic tiles; F(field, clause) makes a leaf."""
    from searcharray_b200 import And, Bool, Boost, DisMax, Or
    return [
        DisMax([Boost(F(A, "w0"), 2), F(B, "w0")], tie=0.3),                          # best_fields, top level
        Or([DisMax([F(A, "w1"), F(B, "b1")], tie=0.1), DisMax([F(A, "s1"), F(B, "bs")], tie=0.1)], mm=2),
        # a MUST group whose members sit in disjoint tiles (t0: one tile, b2: tile 2, t3: another): tiles without
        # any of them are pruned, tiles with one are folded with the others absent
        Bool(must=[DisMax([F(A, "t0"), F(B, "b2"), F(A, "t3")], tie=0.5)], should=[F(A, "w0"), F(B, "b1")]),
        Bool(filter=[DisMax([F(A, "t0"), F(B, "b2")])], should=[DisMax([F(A, "w2"), F(B, "w0")], tie=1.0)]),
        Bool(should=[F(A, "w0"), F(B, "b1")], must_not=[DisMax([F(A, "t3"), F(B, "b2")], tie=0.2)]),
        Bool(must=[DisMax([F(A, "s2"), Boost(F(B, "bs"), 0.5)], tie=0.7)], should=[F(A, "w1")]),
        Bool(should=[DisMax([F(A, "w0"), F(B, "zzz"), F(A, "s1")], tie=0.4), F(B, "b1"), F(A, "t3")], mm=2),
        Bool(must=[DisMax([Boost(F(A, "w0"), 0), Boost(F(B, "b2"), 0)])], should=[F(B, "b1")]),   # zero weights
        Bool(must=[DisMax([F(A, "zzz"), F(B, "zzz")])], should=[F(A, "w0")]),          # nothing present: pruned
        Or([DisMax([F(A, "w0"), F(A, "w0"), Boost(F(B, "w0"), 3)], tie=0.25), F(B, "bs")]),
        And([DisMax([F(A, "w1"), F(B, "b1")], tie=0.05), DisMax([F(A, "w2"), F(B, "w0")], tie=0.05)]),
        Bool(must=[F(A, "w0")], should=[DisMax([F(B, "b2"), F(Z, "b1")], tie=0.3)], filter=[F(B, "b1")],
             must_not=[DisMax([F(Z, "w0"), F(A, "s2")])], mm=1),                        # fz: avgdl 0, empty
    ]


def check_roles(frame, score, what):
    for k in KS:
        check_batch(frame, dismax_queries(fld), k, score, f"{what} k={k}")


def test_roles_fields(synth):
    check_roles(synth.frame, synth.score(), "dismax")


def test_roles_words_path_with_directory():
    """The role checks in a process with SA_NO_TF_TABLE=1: every long list on the words path with a tile
    directory."""
    env = dict(os.environ, SA_NO_TF_TABLE="1")
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_dismax_worker.py")
    r = subprocess.run([sys.executable, worker], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.strip().splitlines()[-1] == "OK", r.stdout[-3000:]


def test_single_field_search_topk(synth):
    """The same groups on one column through search_topk (synonyms), and through fields_topk with every leaf on that
    column: the same ids and score bits."""
    from searcharray_b200 import fields_topk
    arr = synth.frame[A].array
    plain = dismax_queries(lambda f, c: c if f != Z else "zzz")
    fielded = dismax_queries(lambda f, c: fld(A, c if f != Z else "zzz"))
    for k in KS:
        wd, ws = check_single(arr, plain, k, "single")
        gd, gs = fields_topk(synth.frame, fielded, k=k)
        assert np.array_equal(gd, wd) and np.array_equal(gs.view(np.uint32), ws.view(np.uint32)), k


@pytest.mark.parametrize("slop", [0, 2])
def test_phrase_members(synth, slop):
    from searcharray_b200 import Bool, Boost, DisMax, Or
    F = fld
    queries = [DisMax([Boost(F(A, ["pa", "pb"]), 2), F(B, ["qa", "qb"]), F(B, ["pa", "pb"])], tie=0.3),
               Bool(must=[DisMax([F(A, ["pa", "pb"]), F(B, "b2")], tie=0.1)], should=[F(B, "w0"), F(A, "w1")]),
               Bool(should=[F(A, "w0"), F(B, "b1")], must_not=[DisMax([F(B, ["qa", "qb"]), F(A, "t3")])]),
               Or([DisMax([F(A, ["pa", "zzz"]), F(B, ["qa", "qb"])], tie=1.0), F(A, "s1")], mm=1),
               Bool(filter=[DisMax([F(B, ["pa", "pb"]), F(A, ["pa", "pb"])])], should=[F(A, "w2")])]
    for k in KS:
        check_batch(synth.frame, queries, k, synth.score(slop=slop), f"slop={slop}", slop=slop)
    arr = synth.frame[A].array
    single = [DisMax([["pa", "pb"], "t3", Boost("s1", 0.5)], tie=0.2),
              Bool(must=[DisMax([["pa", "pb"], "t0"])], should=["w0"])]
    for k in (1, 10):
        check_single(arr, single, k, f"single slop={slop}", slop=slop)


def test_overflow_rerun(synth):
    """Queries whose tile overflows its candidate slots are re-run exactly."""
    from searcharray_b200 import Bool, DisMax, bm25_similarity
    from searcharray_b200.solr import _fields_topk
    F = fld
    queries = [DisMax([F(A, "hot"), F(A, "cold")], tie=0.5),
               Bool(must=[DisMax([F(A, "hot"), F(B, "zzz")], tie=0.1)], should=[F(A, "cold")]),
               Bool(filter=[F(B, "b1")], should=[DisMax([F(A, "w0"), F(B, "w0")])])]
    for k in (10, 16):
        docs, scores, n_redone = _fields_topk(synth.frame, queries, k, bm25_similarity(), 0)
        assert n_redone > 0
        for i, q in enumerate(queries):
            assert_topk(docs[i], scores[i], compose_dismax(synth.score(), q), k, f"overflow {q!r} k={k}")
    arr = synth.frame[A].array
    docs, scores, n_redone = arr._search_topk_bool([DisMax(["hot", "cold"], tie=0.3)], 10, bm25_similarity(), 0)
    assert n_redone == 1
    assert_topk(docs[0], scores[0], compose_dismax(arr.score, DisMax(["hot", "cold"], tie=0.3)), 10, "single overflow")


def test_shard_doc_base_global_df():
    from searcharray_b200 import Bool, Boost, DisMax, Or, SearchArray
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
    queries = [DisMax([Boost(F(A, "w0"), 2), F(B, "w0")], tie=0.3),
               Bool(must=[DisMax([F(A, "t0"), F(B, "b2")], tie=0.1)], should=[F(B, "b1")]),
               Or([DisMax([Boost(F(A, ["pa", "pb"]), 3), F(B, ["qa", "qb"])], tie=0.5), F(B, "bs")]),
               Bool(should=[F(A, "w1")], must_not=[DisMax([F(A, "w2"), F(B, "b2")])])]
    for k in (1, 10, 32):
        check_batch(frame, queries, k, score, "shard", doc_base=base)
    arr = frame[A].array
    for k in (1, 10):
        check_single(arr, [DisMax(["w0", "s1", ["pa", "pb"]], tie=0.2), Bool(must=[DisMax(["t0", "t3"])],
                                                                               should=["w1"])], k, "shard single",
                     doc_base=base)


def test_batch_spans_two_groups():
    """~2M docs, two fields: a batch with more phrase members than one ~4 GB group of rows holds (512 rows of 8 MB),
    so it runs as two launch groups."""
    from searcharray_b200 import DisMax, Or, SearchArray
    from searcharray_b200.indexing import index_from_term_postings
    from searcharray_b200.roaringish import encode_postings
    rng = np.random.default_rng(7)
    n = 2_000_000

    def field(shift, lo, hi):
        docs = np.sort(rng.choice(n, 20000, replace=False))
        pa = encode_postings(docs, np.full(len(docs), 3 + shift))
        pb = encode_postings(docs[::2], np.full(len(docs[::2]), 4 + shift))
        x_docs = np.sort(rng.choice(n, 50000, replace=False))
        x = encode_postings(x_docs, np.full(len(x_docs), 7))
        return SearchArray.from_host_index(index_from_term_postings(["pa", "pb", "x"], [pa, pb, x],
                                                                    rng.integers(lo, hi, n).astype(np.float32)))
    frame = pd.DataFrame({A: field(0, 1, 30), B: field(5, 10, 90)})
    score = field_scorer({f: (lambda c, f=f: frame[f].array.score(c)) for f in (A, B)})
    queries = [Or([DisMax([fld(A, ["pa", "pb"]), fld(B, ["pa", "pb"])], tie=0.1 * (j % 4)) for j in range(31)] +
                  [DisMax([fld(B, "x"), fld(A, "x")], tie=0.5)], mm=1 + i % 2) for i in range(9)]   # 558 rows
    check_batch(frame, queries, 10, score, "2M docs")


def test_launches_one_tile_launch_per_group(synth):
    """A term-only DisMax batch is one tile launch and one select, whatever the number of queries, on both entry
    points."""
    from searcharray_b200 import Bool, Boost, DisMax, _lib, fields_topk
    h = synth.frame[A].array._device().handle
    arr = synth.frame[A].array

    def fields_batch(nq):
        return [Bool(must=[DisMax([fld(A, "w0"), Boost(fld(B, "b1"), 2)], tie=0.1)],
                     should=[fld(A, "s1"), DisMax([fld(B, "bs"), fld(A, "t3")])], must_not=[fld(B, "b2")], mm=i % 2)
                for i in range(nq)]

    def single_batch(nq):
        return [Bool(must=[DisMax(["w0", Boost("w1", 2)], tie=0.1)], should=["s1", DisMax(["s2", "t3"])],
                     must_not=["t0"], mm=i % 2) for i in range(nq)]
    for run, make in ((lambda qs: fields_topk(synth.frame, qs, k=10), fields_batch),
                      (lambda qs: arr.search_topk(qs, k=10), single_batch)):
        launches = []
        for nq in (1, 4, 64):
            queries = make(nq)
            run(queries)                                   # warm: the norm tables for these parameters
            _lib.check(_lib.lib().sa_stats_reset(h))
            run(queries)
            st = _lib.SaStats()
            _lib.check(_lib.lib().sa_stats_get(h, ctypes.byref(st)))
            launches.append(st.total_launches)
        assert launches == [2, 2, 2], launches


def test_mixed_batch_leaves_other_queries_alone(synth):
    """Plain, Or, Bool and DisMax queries in one search_topk batch: the DisMax queries match the composition, the
    others are bit-identical to the same queries run without them."""
    from searcharray_b200 import And, Bool, Boost, DisMax, Or
    arr = synth.frame[A].array
    others = ["w0", ["pa", "pb"], Or(["w1", "s1"]), And(["w0", "w2"]), Bool(must=["w0"], should=[Boost("s1", 2)]),
              Or([Boost("w1", 3), "t3"])]
    dms = [DisMax(["w0", "w1"], tie=0.2), Bool(must=[DisMax(["t0", "t3"])], should=["w2"]),
           Or([DisMax(["s1", "s2"], tie=1.0), "w0"], mm=2)]
    mixed = [others[0], dms[0], others[1], others[2], dms[1], others[3], others[4], dms[2], others[5]]
    for k in (1, 10, 32):
        md, ms = arr.search_topk(mixed, k=k)
        od, os_ = arr.search_topk(others, k=k)
        idx = [0, 2, 3, 5, 6, 8]
        assert np.array_equal(md[idx], od) and np.array_equal(ms[idx].view(np.uint32), os_.view(np.uint32))
        for i, q in zip((1, 4, 7), dms):
            assert_topk(md[i], ms[i], compose_dismax(arr.score, q), k, f"mixed {q!r}")


def test_single_member_is_its_clause(synth):
    """DisMax([c]) gives c's ids and score bits in every role, at every tie, through both entry points."""
    from searcharray_b200 import Bool, Boost, DisMax, Or, fields_topk
    arr = synth.frame[A].array
    for tie in (0.0, 0.3, 1.0):
        for leaf, c in ((lambda x: x, "w0"), (lambda x: x, ["pa", "pb"]), (lambda x: fld(A, x), "s1"),
                        (lambda x: fld(B, x), "b2")):
            roles = [lambda x: Bool(must=[x], should=[leaf("w1")]), lambda x: Bool(should=[x, leaf("s2")], mm=1),
                     lambda x: Bool(filter=[x], should=[leaf("w2")]), lambda x: Bool(should=[leaf("w0")], must_not=[x])]
            plain = [r(leaf(c)) for r in roles]
            one = [r(DisMax([leaf(c)], tie=tie)) for r in roles]
            if isinstance(leaf("x"), str):
                pd_, ps = arr.search_topk(plain, k=10)
                od, os_ = arr.search_topk(one, k=10)
            else:
                pd_, ps = fields_topk(synth.frame, plain, k=10)
                od, os_ = fields_topk(synth.frame, one, k=10)
            assert np.array_equal(pd_, od) and np.array_equal(ps.view(np.uint32), os_.view(np.uint32)), (c, tie)
            # a boosted member scores as the boosted clause
            plain = [Bool(must=[Boost(leaf(c), 2.5)], should=[leaf("w1")]), Or([Boost(leaf(c), 0.5), leaf("w0")])]
            one = [Bool(must=[DisMax([Boost(leaf(c), 2.5)], tie=tie)], should=[leaf("w1")]),
                   Or([DisMax([Boost(leaf(c), 0.5)], tie=tie), leaf("w0")])]
            if isinstance(leaf("x"), str):
                pd_, ps = arr.search_topk(plain, k=10)
                od, os_ = arr.search_topk(one, k=10)
            else:
                pd_, ps = fields_topk(synth.frame, plain, k=10)
                od, os_ = fields_topk(synth.frame, one, k=10)
            assert np.array_equal(pd_, od) and np.array_equal(ps.view(np.uint32), os_.view(np.uint32)), (c, tie)


def test_golden():
    """The real reference's composed top 10 of every record on the TMDB title and overview fields, through fields_topk
    (Field records) and search_topk (single-field records): ids and score bits, and the same against this library's
    .score at every k."""
    from searcharray_b200 import SearchArray, bm25_similarity, fields_topk
    with open(os.path.join(GOLDEN, "dismax.json")) as f:
        fixture = json.load(f)
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    frame = pd.DataFrame({f: SearchArray.from_host_index(load_field(z, f)) for f in ("title_tokens", "overview_tokens")})
    for group in record_groups(fixture["queries"]).values():
        r0 = group[0]
        sims = {f: bm25_similarity(k1=kb[0], b=kb[1]) for f, kb in r0["sim"].items()}
        queries = [query_of(r) for r in group]
        if r0["field"] is None:
            docs, scores = fields_topk(frame, queries, k=10, similarity=sims, slop=r0["slop"])
        else:
            docs, scores = frame[r0["field"]].array.search_topk(
                queries, k=10, similarity=sims.get(r0["field"], bm25_similarity()), slop=r0["slop"])
        for i, r in enumerate(group):
            n = len(r["top_ids"])
            what = f"{queries[i]!r} slop={r['slop']} sim={r['sim']}"
            assert docs[i][:n].tolist() == r["top_ids"], what
            assert scores[i][:n].view(np.uint32).tolist() == r["top_bits"], what
            assert np.all(docs[i][n:] == 0xFFFFFFFF), what
        if r0["field"] is None:
            score = field_scorer({f: (lambda c, f=f: frame[f].array.score(
                c, similarity=sims.get(f, bm25_similarity()), slop=r0["slop"])) for f in frame.columns})
            for k in KS:
                check_batch(frame, queries, k, score, "tmdb", slop=r0["slop"], similarity=sims)


def test_c_abi_rejections(synth):
    """Split groups, groups across queries, mixed occur, a bad tie, mm over groups and non-sparse members are errors;
    the same arrays with the fault removed run."""
    from searcharray_b200 import _lib
    from searcharray_b200.solr import _Multi
    a, b = synth.frame[A].array, synth.frame[B].array
    ta, tb = a.host.term_dict.term_to_ids, b.host.term_dict.term_to_ids
    docs = np.empty(20, dtype=np.uint32)
    scores = np.empty(20, dtype=np.float32)
    terms = np.asarray([ta["w0"], ta["w1"], ta["s1"], ta["w2"]], dtype=np.uint32)

    def single(q_starts, groups, ties, occurs=(0, 0, 0, 0), mm=(1, 1), k1=1.2, bb=0.75):
        q_starts = np.asarray(q_starts, dtype=np.uint32)
        c_starts = np.arange(5, dtype=np.uint32)
        idf = np.ones(4, dtype=np.float32)
        g = np.asarray(groups, dtype=np.uint32)
        t = np.asarray(ties, dtype=np.float32)
        o = np.asarray(occurs, dtype=np.uint8)
        m = np.asarray(mm, dtype=np.uint32)
        return _lib.lib().sa_score_batch_topk_bool(
            a._device().handle, len(q_starts) - 1, _lib.p_u32(q_starts), None, _lib.p_u32(terms), _lib.p_u32(c_starts),
            _lib.p_f32(idf), _lib.p_f32(idf), _lib.p_u8(o), _lib.p_u32(g), _lib.p_f32(t), _lib.p_u32(m),
            len(q_starts) - 1, 0, a.avg_doc_length, k1, bb, 10, None, 0, 0, _lib.p_u32(docs), _lib.p_f32(scores), None,
            0, None, None, None, None)
    assert single([0, 2, 4], [0, 0, 2, 2], [0.1, 0, 0.3, 0]) == 0
    assert single([0, 2, 4], [0, 1, 2, 2], [0, 0, 0, 0]) == 0               # plain clauses
    assert single([0, 4], [0, 0, 2, 2], [0.1, 0, 0.3, 0], mm=(2,)) == 0
    assert single([0, 4], [0, 0, 2, 2], [0.1, 0, 0.3, 0], mm=(3,)) != 0    # mm over groups
    assert b"SHOULD groups" in _lib.lib().sa_last_error()
    assert single([0, 4], [0, 1, 0, 3], [0, 0, 0, 0], mm=(1,)) != 0        # a split group
    assert single([0, 2, 4], [0, 0, 0, 2], [0, 0, 0, 0]) != 0               # a group crossing queries
    assert single([0, 2, 4], [0, 0, 3, 3], [0, 0, 0, 0]) != 0               # a group that starts after its clause
    assert single([0, 2, 4], [0, 0, 2, 2], [0, 0, 0, 0], occurs=(0, 1, 0, 0)) != 0   # mixed occur
    assert b"differ in occur" in _lib.lib().sa_last_error()
    for bad in (-0.5, 1.5, float("nan"), float("inf")):
        assert single([0, 2, 4], [0, 0, 2, 2], [bad, 0, 0, 0]) != 0
    assert single([0, 2, 4], [0, 0, 2, 2], [0, 0, 0, 0], k1=0.0) != 0       # non-sparse members
    assert b"DisMax members" in _lib.lib().sa_last_error()
    assert single([0, 2, 4], [0, 0, 2, 2], [0, 0, 0, 0], bb=1.0) != 0
    assert single([0, 2, 4], [0, 1, 2, 3], [0, 0, 0, 0], k1=0.0) == 0       # plain clauses need no sparse parameters

    # the multi entry point: the same checks, members on two fields
    def multi(groups, ties, k1=(1.2, 1.2)):
        q_starts = np.asarray([0, 2], dtype=np.uint32)
        f = np.asarray([0, 1], dtype=np.uint32)
        t = np.asarray([ta["w0"], tb["b1"]], dtype=np.uint32)
        c_starts = np.arange(3, dtype=np.uint32)
        ones = np.ones(2, dtype=np.float32)
        occ = np.zeros(2, dtype=np.uint8)
        m = np.asarray([1], dtype=np.uint32)
        avgdl = np.asarray([a.avg_doc_length, b.avg_doc_length], dtype=np.float32)
        kk, bb = np.asarray(k1, dtype=np.float32), np.full(2, 0.75, dtype=np.float32)
        return _lib.lib().sa_multi_score_batch_topk_bool(
            mh.handle, 1, _lib.p_u32(q_starts), None, _lib.p_u32(f), _lib.p_u32(t), _lib.p_u32(c_starts),
            _lib.p_f32(ones), _lib.p_f32(ones), _lib.p_u8(occ), _lib.p_u32(np.asarray(groups, dtype=np.uint32)),
            _lib.p_f32(np.asarray(ties, dtype=np.float32)), _lib.p_u32(m), 1, 0, _lib.p_f32(avgdl), _lib.p_f32(kk),
            _lib.p_f32(bb), 10, None, 0, 0, _lib.p_u32(docs), _lib.p_f32(scores), None, 0, None, None, None, None)
    mh = _Multi([a, b])
    assert multi([0, 0], [0.3, 0]) == 0
    assert multi([0, 1], [0, 0]) == 0
    assert multi([1, 1], [0, 0]) != 0
    assert multi([0, 0], [2.0, 0]) != 0
    assert multi([0, 0], [0.3, 0], k1=(1.2, 0.0)) != 0
