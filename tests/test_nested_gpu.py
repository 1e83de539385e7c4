"""GPU: nested boolean queries (an Or / And / Bool as a clause of another; sa_score_batch_topk_bool and
sa_multi_score_batch_topk_bool with clause_node, the NESTED instances of bool_tile_kernel in sa_bool.cu) against compose_nested with each clause
scored by this library's .score: ids and float32 score bits must be equal.

The synthetic frame is tests/test_bool_fields_gpu.py's: five 8192-doc tiles, `fa` (`w0` / `w1` / `w2` with a tile
directory and a tf table, `s1` / `s2` on the binary-search path, `t0` / `t3` in one tile each, `pa` / `pb` phrases,
`hot` / `cold` overflowing a tile's candidate slots) and `fb` (`b1`, `bs`, `b2` in tile 2 only, phrase `qa qb`), plus
`fz`, fb's postings under avgdl 0.  The role checks run again in a child process with SA_NO_TF_TABLE=1
(tests/_nested_worker.py), where the long lists take the words path with a tile directory."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pandas as pd
import pytest

from _bool_fields_compose import field_scorer
from _nested_compose import compose_nested, query_of
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
    """fields_topk(queries) against compose_nested(score, q) for every query of the batch."""
    from searcharray_b200 import bm25_similarity, fields_topk
    docs, scores = fields_topk(frame, queries, k=k, similarity=similarity or bm25_similarity(), slop=slop)
    assert docs.shape == (len(queries), k) and docs.dtype == np.uint32 and scores.dtype == np.float32
    for i, q in enumerate(queries):
        assert_topk(docs[i], scores[i], compose_nested(score, q), k, f"{what} {q!r} k={k}", doc_base)
    return docs, scores


def check_single(arr, queries, k, what, slop=0, doc_base=0):
    """search_topk(queries) on one column against compose_nested over its .score."""
    docs, scores = arr.search_topk(queries, k=k, slop=slop)
    for i, q in enumerate(queries):
        assert_topk(docs[i], scores[i], compose_nested(lambda c: arr.score(c, slop=slop), q), k,
                    f"{what} {q!r} k={k}", doc_base)
    return docs, scores


def nested_queries(F):
    """Nested queries in every role over the synthetic tiles; F(field, clause) makes a leaf."""
    from searcharray_b200 import And, Bool, Boost, DisMax, Or
    shared = And([F(A, "w0"), F(B, "b1")])
    return [
        Or([And([F(A, "w0"), F(A, "w1")]), And([F(A, "w0"), F(B, "b1")])]),                  # or of ands
        Bool(must=[F(A, "w2"), Or([F(A, "s1"), F(B, "bs"), F(A, "w1")], mm=2)]),              # required sub-query
        Bool(should=[F(A, "w0")], must_not=[And([F(A, "w1"), F(B, "b1")])]),                 # excluded conjunction
        Bool(filter=[Or([F(A, "t0"), F(B, "b2")])], should=[F(A, "w1"), F(B, "w0")]),        # filter: a few tiles
        # a MUST nested clause whose leaves sit in a few tiles only: the other tiles are pruned through its flags
        Bool(must=[Or([F(A, "t0"), F(A, "t3")])], should=[F(A, "w0"), F(B, "b1")]),
        Bool(must=[And([F(A, "t0"), F(B, "b2")])], should=[F(A, "w0")]),                      # maybe empty everywhere
        Bool(must=[Or([F(A, "zzz"), F(B, "zzz")])], should=[F(A, "w0")]),                     # empty everywhere
        Bool(should=[F(A, "w0"), Or([F(A, "zzz")])], mm=1),                                     # empty SHOULD child
        Or([Boost(And([F(A, "w0"), F(B, "w0")]), 2.5), F(B, "bs")]),                             # boosted
        Bool(must=[Boost(Or([F(A, "w1"), F(B, "b1")]), 0)], should=[F(A, "s2")]),               # weight 0
        Or([Or([F(A, "w0"), F(A, "w1"), F(B, "b1"), F(B, "bs")], mm="75%"), F(A, "s1"),
            Or([F(A, "w2"), F(B, "w0")], mm="-1")], mm="2<-25%"),                               # Solr mm specs
        Or([Bool(must=[And([F(A, "w0"), Or([F(A, "w1"), F(B, "b2")])])], should=[F(B, "bs")]), F(A, "t3")]),  # depth 3
        Bool(must=[Or([DisMax([Boost(F(A, "w0"), 2), F(B, "w0")], tie=0.3),
                       DisMax([F(A, "w1"), F(B, "b1")], tie=0.1)], mm=2)], should=[F(A, "s1")]),  # DisMax inside
        Bool(should=[shared, Boost(shared, 2)], must_not=[Bool(must=[shared], filter=[F(A, "t3")])]),  # shared object
        Bool(should=[F(A, "w0"), Bool(must=[F(B, "b1")], must_not=[F(A, "w1")])], mm=2),
        Or([Or([Or([Or([F(A, "w0")])])]), F(Z, "b1")]),                                        # a chain, fz: avgdl 0
    ]


def check_roles(frame, score, what):
    for k in KS:
        check_batch(frame, nested_queries(fld), k, score, f"{what} k={k}")


def test_roles_fields(synth):
    check_roles(synth.frame, synth.score(), "nested")


def test_roles_words_path_with_directory():
    """The role checks in a process with SA_NO_TF_TABLE=1: every long list on the words path with a tile
    directory."""
    env = dict(os.environ, SA_NO_TF_TABLE="1")
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_nested_worker.py")
    r = subprocess.run([sys.executable, worker], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.strip().splitlines()[-1] == "OK", r.stdout[-3000:]


def test_single_field_search_topk(synth):
    """The same trees on one column through search_topk, and through fields_topk with every leaf on that column: the
    same ids and score bits."""
    from searcharray_b200 import fields_topk
    arr = synth.frame[A].array
    plain = nested_queries(lambda f, c: c if f != Z else "zzz")
    fielded = nested_queries(lambda f, c: fld(A, c if f != Z else "zzz"))
    for k in KS:
        wd, ws = check_single(arr, plain, k, "single")
        gd, gs = fields_topk(synth.frame, fielded, k=k)
        assert np.array_equal(gd, wd) and np.array_equal(gs.view(np.uint32), ws.view(np.uint32)), k


@pytest.mark.parametrize("slop", [0, 2])
def test_phrase_leaves(synth, slop):
    from searcharray_b200 import And, Bool, Boost, Or
    F = fld
    queries = [Or([And([F(A, ["pa", "pb"]), F(A, "w0")]), And([F(B, ["qa", "qb"]), F(B, "b1")])]),
               Bool(must=[Or([Boost(F(A, ["pa", "pb"]), 2), F(B, ["pa", "pb"])])], should=[F(A, "w1")]),
               Bool(should=[F(A, "w0")], must_not=[Or([F(B, ["qa", "qb"]), F(A, ["pa", "zzz"])])])]
    for k in KS:
        check_batch(synth.frame, queries, k, synth.score(slop=slop), f"slop={slop}", slop=slop)
    arr = synth.frame[A].array
    single = [Or([And([["pa", "pb"], "w0"]), "t3"]), Bool(must=[Or([["pa", "pb"], "t0"])], should=["w1"])]
    for k in (1, 10):
        check_single(arr, single, k, f"single slop={slop}", slop=slop)


def test_one_leaf_or_is_its_leaf(synth):
    """Or([a, Or([b])]) gives Or([a, b])'s ids and score bits, on both entry points, and so does a nested Bool of one
    should clause in every role of a Bool."""
    from searcharray_b200 import Bool, Or, fields_topk
    arr = synth.frame[A].array
    for a, b in (("w0", "w1"), ("s1", ["pa", "pb"]), ("t0", "zzz"), ("w2", "t3")):
        flat = [Or([a, b]), Or([a, b], mm=2), Bool(must=[a], should=[b]), Bool(should=[a], must_not=[b]),
                Bool(should=[a], filter=[b])]
        nest = [Or([a, Or([b])]), Or([a, Or([b])], mm=2), Bool(must=[a], should=[Or([b])]),
                Bool(should=[a], must_not=[Or([b])]), Bool(should=[a], filter=[Bool(should=[b])])]
        fd, fs = arr.search_topk(flat, k=10)
        nd, ns = arr.search_topk(nest, k=10)
        assert np.array_equal(fd, nd) and np.array_equal(fs.view(np.uint32), ns.view(np.uint32)), (a, b)
        F = fld
        fd, fs = fields_topk(synth.frame, [Or([F(A, a), F(B, "b1")])], k=10)
        nd, ns = fields_topk(synth.frame, [Or([F(A, a), Or([F(B, "b1")])])], k=10)
        assert np.array_equal(fd, nd) and np.array_equal(fs.view(np.uint32), ns.view(np.uint32)), a


def test_overflow_rerun(synth):
    """Queries whose tile overflows its candidate slots are re-run exactly, their nested rows rebuilt."""
    from searcharray_b200 import And, Bool, Or, bm25_similarity
    from searcharray_b200.solr import _fields_topk
    F = fld
    queries = [Or([Or([F(A, "hot"), F(A, "cold")])]),
               Bool(must=[Or([F(A, "hot"), F(B, "zzz")])], should=[F(A, "cold")]),
               Bool(filter=[F(B, "b1")], should=[And([F(A, "w0"), F(B, "w0")])])]
    for k in (10, 16):
        docs, scores, n_redone = _fields_topk(synth.frame, queries, k, bm25_similarity(), 0)
        assert n_redone >= 1
        for i, q in enumerate(queries):
            assert_topk(docs[i], scores[i], compose_nested(synth.score(), q), k, f"overflow {q!r} k={k}")
    arr = synth.frame[A].array
    q = Or([Or(["hot", "cold"])])
    docs, scores, n_redone = arr._search_topk_bool([q, Or(["w1", And(["s1", "w2"])])], 10, bm25_similarity(), 0)
    assert n_redone >= 1
    assert_topk(docs[0], scores[0], compose_nested(arr.score, q), 10, "single overflow")


def test_shard_doc_base_global_df():
    from searcharray_b200 import And, Bool, Boost, Or, SearchArray
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
    queries = [Or([And([F(A, "w0"), F(B, "b1")]), And([F(A, "w1"), F(B, "w0")])]),
               Bool(must=[Or([F(A, "t0"), F(B, "b2")])], should=[F(B, "b1")]),
               Or([Boost(And([F(A, ["pa", "pb"]), F(B, "bs")]), 3), F(B, "bs")]),
               Bool(should=[F(A, "w1")], must_not=[And([F(A, "w2"), F(B, "b1")])])]
    for k in (1, 10, 32):
        check_batch(frame, queries, k, score, "shard", doc_base=base)
    arr = frame[A].array
    for k in (1, 10):
        check_single(arr, [Or([And(["w0", "s1"]), ["pa", "pb"]]), Bool(must=[Or(["t0", "t3"])], should=["w1"])], k,
                     "shard single", doc_base=base)


def test_batch_spans_two_groups():
    """~2M docs, two fields: a batch whose phrase and nested rows do not fit one ~4 GB group of rows (512 rows of
    8 MB), so it runs as two launch groups."""
    from searcharray_b200 import And, Or, SearchArray
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
    # per query 30 nested nodes and 30 phrase leaves: 60 rows, 9 queries = 540 rows
    queries = [Or([And([fld(A if j % 2 else B, ["pa", "pb"]), fld(B, "x")]) for j in range(30)] + [fld(A, "x")],
                  mm=1 + i % 2) for i in range(9)]
    check_batch(frame, queries, 10, score, "2M docs")


def test_mixed_batch_leaves_other_queries_alone(synth):
    """Plain, Or, Bool, DisMax and nested queries in one search_topk batch: the nested ones match the composition,
    the others are bit-identical to the same queries run without them."""
    from searcharray_b200 import And, Bool, Boost, DisMax, Or
    arr = synth.frame[A].array
    others = ["w0", ["pa", "pb"], Or(["w1", "s1"]), And(["w0", "w2"]), Bool(must=["w0"], should=[Boost("s1", 2)]),
              DisMax(["w0", "w1"], tie=0.2), Or([DisMax(["s1", "s2"], tie=1.0), "w0"], mm=2)]
    nest = [Or([And(["w0", "w1"]), And(["s1", "w2"])]), Bool(must=[Or(["t0", "t3"])], should=["w2"]),
            Bool(should=["w0"], must_not=[And(["w1", DisMax(["s1", "s2"])])])]
    mixed = [others[0], nest[0], others[1], others[2], nest[1], others[3], others[4], nest[2], others[5], others[6]]
    for k in (1, 10, 32):
        md, ms = arr.search_topk(mixed, k=k)
        od, os_ = arr.search_topk(others, k=k)
        idx = [0, 2, 3, 5, 6, 8, 9]
        assert np.array_equal(md[idx], od) and np.array_equal(ms[idx].view(np.uint32), os_.view(np.uint32))
        for i, q in zip((1, 4, 7), nest):
            assert_topk(md[i], ms[i], compose_nested(arr.score, q), k, f"mixed {q!r}")


def test_fields_sharing_one_index(synth):
    """Two column names of one array (one device index, one norm table) in one nested query."""
    from searcharray_b200 import And, Bool, Or
    frame = pd.DataFrame({A: synth.frame[A].array, "fa2": synth.frame[A].array, B: synth.frame[B].array})
    score = field_scorer({f: (lambda c, f=f: frame[f].array.score(c)) for f in frame.columns})
    queries = [Or([And([fld(A, "w0"), fld("fa2", "w1")]), And([fld("fa2", "s1"), fld(B, "b1")])]),
               Bool(must=[Or([fld("fa2", "t0"), fld(A, "t3")])], should=[fld(B, "w0")])]
    for k in (1, 10):
        check_batch(frame, queries, k, score, "shared index")


def test_golden():
    """The real reference's composed top 10 of every record on the TMDB title and overview fields, through fields_topk
    (Field records) and search_topk (single-field records): ids and score bits, and the same against this library's
    .score at every k."""
    from searcharray_b200 import SearchArray, bm25_similarity, fields_topk
    with open(os.path.join(GOLDEN, "nested.json")) as f:
        fixture = json.load(f)
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    frame = pd.DataFrame({f: SearchArray.from_host_index(load_field(z, f)) for f in ("title_tokens", "overview_tokens")})
    for r in fixture["queries"]:
        sims = {f: bm25_similarity(k1=kb[0], b=kb[1]) for f, kb in r["sim"].items()}
        q = query_of(r)
        what = f"{q!r} slop={r['slop']} sim={r['sim']}"
        if r["field"] is None:
            docs, scores = fields_topk(frame, [q], k=10, similarity=sims, slop=r["slop"])
        else:
            docs, scores = frame[r["field"]].array.search_topk(
                [q], k=10, similarity=sims.get(r["field"], bm25_similarity()), slop=r["slop"])
        n = len(r["top_ids"])
        assert docs[0][:n].tolist() == r["top_ids"], what
        assert scores[0][:n].view(np.uint32).tolist() == r["top_bits"], what
        assert np.all(docs[0][n:] == 0xFFFFFFFF), what
        if r["field"] is None:
            score = field_scorer({f: (lambda c, f=f: frame[f].array.score(
                c, similarity=sims.get(f, bm25_similarity()), slop=r["slop"])) for f in frame.columns})
            for k in KS:
                check_batch(frame, [q], k, score, "tmdb", slop=r["slop"], similarity=sims)


def test_c_abi_rejections(synth):
    """Malformed node layouts are SA_ERR_ARG; the well-formed layout runs."""
    from searcharray_b200 import _lib
    from searcharray_b200.query import SA_NO_NODE
    a = synth.frame[A].array
    ta = a.host.term_dict.term_to_ids
    X = SA_NO_NODE
    docs = np.empty(20, dtype=np.uint32)
    scores = np.empty(20, dtype=np.float32)

    def call(n_starts, c_node, c_terms, groups=None, mm=None, nq=1):
        """Clause c is a leaf with the terms c_terms[c] (a list of names) or nested node c_node[c]."""
        n_starts = np.asarray(n_starts, dtype=np.uint32)
        nc = int(n_starts[-1])
        terms = np.asarray([ta[t] for ts in c_terms for t in ts], dtype=np.uint32)
        c_starts = np.asarray(np.cumsum([0] + [len(ts) for ts in c_terms]), dtype=np.uint32)
        ones = np.ones(nc, dtype=np.float32)
        occ = np.zeros(nc, dtype=np.uint8)
        g = np.asarray(range(nc) if groups is None else groups, dtype=np.uint32)
        t = np.zeros(nc, dtype=np.float32)
        m = np.asarray(mm or [1] * (len(n_starts) - 1), dtype=np.uint32)
        return _lib.lib().sa_score_batch_topk_bool(
            a._device().handle, len(n_starts) - 1, _lib.p_u32(n_starts), _lib.p_u32(np.asarray(c_node, dtype=np.uint32)),
            _lib.p_u32(terms), _lib.p_u32(c_starts), _lib.p_f32(ones), _lib.p_f32(ones), _lib.p_u8(occ), _lib.p_u32(g),
            _lib.p_f32(t), _lib.p_u32(m), nq, 0, a.avg_doc_length, 1.2, 0.75, 10, None, 0, 0, _lib.p_u32(docs),
            _lib.p_f32(scores), None, 0, None, None, None, None)
    # query 0 = Or(w0, node 1); node 1 = Or(w1, s1)
    assert call([0, 2, 4], [X, 1, X, X], [["w0"], [], ["w1"], ["s1"]]) == 0
    assert call([0, 2, 4], [X, 2, X, X], [["w0"], [], ["w1"], ["s1"]]) != 0          # out of range
    assert call([0, 2, 4], [1, 1, X, X], [[], [], ["w1"], ["s1"]]) != 0              # shared
    assert b"more than one clause" in _lib.lib().sa_last_error()
    assert call([0, 2, 4, 5], [X, 1, X, X, X], [["w0"], [], ["w1"], ["s1"], ["w2"]]) != 0     # unreferenced node 2
    assert b"referenced by no clause" in _lib.lib().sa_last_error()
    assert call([0, 2, 4, 6], [X, 2, X, 1, X, X], [["w0"], [], ["w1"], [], ["s1"], ["w2"]]) != 0   # a self reference
    assert call([0, 2, 4], [X, 0, X, X], [["w0"], [], ["w1"], ["s1"]]) != 0          # a top-level node referenced
    assert call([0, 2, 4], [X, 1, X, X], [["w0"], ["w2"], ["w1"], ["s1"]]) != 0      # a nested clause with terms
    assert b"has no terms" in _lib.lib().sa_last_error()
    assert call([0, 2, 4], [X, 1, X, X], [["w0"], [], ["w1"], ["s1"]], groups=[0, 0, 2, 3]) != 0   # a DisMax member
    assert b"DisMax member" in _lib.lib().sa_last_error()
    assert call([0, 2, 4], [X, 1, X, X], [["w0"], [], ["w1"], ["s1"]], mm=[1, 3]) != 0   # a node's mm
    assert call([0, 2, 4], [X, 1, X, X], [["w0"], [], ["w1"], ["s1"]], nq=2) != 0     # node 1 is top-level too
    assert call([0, 2, 4], [X, 1, X, X], [["w0"], [], ["w1"], ["s1"]]) == 0
