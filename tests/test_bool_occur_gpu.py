"""GPU: Bool (must / should / filter / must_not) and Boost in search_topk (sa_score_batch_topk_bool with weights and
roles, the OCCUR instances of bool_tile_kernel in sa_bool.cu) against the composition of tests/_bool_occur_compose.py: ids and float32 score
bits must be equal.

The corpus is test_bool_topk_gpu.py's synthetic five-tile corpus: `w0` / `w1` / `w2` have a tile directory and a tf
table (records), `s1` / `s2` are found by binary search over their words, `t0` / `t3` live in one tile each (a MUST
on them prunes the other tiles), `pa` / `pb` make phrases, `hot` / `cold` overflow a tile's candidate slots.  The
same role checks run again in a child process with SA_NO_TF_TABLE=1 (tests/_bool_occur_worker.py), where the long
lists take the words path with a tile directory."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from _bool_compose import expand
from _bool_occur_compose import compose_occur, query_of
from _tmdb_index import load_field
from conftest import GOLDEN
from test_bool_topk_gpu import KS, TILE, Synth, assert_topk, synth_corpus

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def synth():
    return Synth()


def check_batch(arr, queries, k, score, what, doc_base=0, slop=0, similarity=None):
    """search_topk(queries) against compose_occur(score, q) for every Bool / Or query of the batch."""
    from searcharray_b200 import bm25_similarity
    from searcharray_b200.query import is_boolean
    sim = similarity or bm25_similarity()
    docs, scores = arr.search_topk(queries, k=k, similarity=sim, slop=slop)
    assert docs.shape == (len(queries), k) and scores.dtype == np.float32
    for i, q in enumerate(queries):
        if is_boolean(q):
            assert_topk(docs[i], scores[i], compose_occur(score, q), k, f"{what} {q!r} k={k}", doc_base)
    return docs, scores


def role_queries():
    """Term clauses in every role on the tf-table and binary-search paths (the words path with a directory under
    SA_NO_TF_TABLE=1), boosts, duplicates, unknown tokens."""
    from searcharray_b200 import And, Bool, Boost, Or
    return [
        Bool(must=["w0"], should=["w1", "s1"], mm=0), Bool(must=["w0"], should=["w1", "s1", "w2"], mm=1),
        Bool(must=["w0"], should=["w1", "s1", "w2"], mm=2),
        Bool(must=["w1", "s2"], should=["w0"]),                          # MUST on the binary-search path
        Bool(filter=["w0"], should=["w1", "s1"]), Bool(filter=["s1", "w1"], should=["w0", "w2"], mm=1),
        Bool(should=["w0", "w1"], must_not=["w2"]), Bool(should=["w1", "s2"], must_not=["w0"]),
        Bool(should=["w0"], must_not=["s1", "t0"]),                       # MUST_NOT absent from most tiles
        Bool(must=[Boost("w0", 0.5)], should=[Boost("w1", 2), Boost("s1", 0)], filter=["w2"], must_not=["t0"],
             mm=1),
        Bool(must=[Boost("t0", 0)], should=["w0"]),                       # a zero weight still requires a match
        Bool(must=["w0", "w0"], should=["s1", "s1"], must_not=["t3", "t3"], filter=["w1", "w1"], mm=1),
        Bool(must=["zzz"], should=["w0"]), Bool(should=["w0", "zzz"], must_not=["zzz"], filter=["w1"]),
        Bool(should=["w0"], filter=["zzz"]), Bool(must=["w2"], should=[Boost("zzz", 3)]),
        Or([Boost("w0", 3), "w1", Boost("s2", 0.5)]), Or([Boost("w1", 0), "s1"], mm=2),
        And([Boost("w1", 2), "w0", Boost("s2", 0.25)]),
    ]


def check_roles(arr, score, what):
    for k in KS:
        check_batch(arr, role_queries(), k, score, f"{what} k={k}")


def test_roles_terms(synth):
    check_roles(synth.arr, synth.oracle(), "synth")


def test_roles_words_path_with_directory():
    """The role checks in a process with SA_NO_TF_TABLE=1: every long list on the words path with a tile
    directory."""
    env = dict(os.environ, SA_NO_TF_TABLE="1")
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_bool_occur_worker.py")
    r = subprocess.run([sys.executable, worker], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.strip().splitlines()[-1] == "OK", r.stdout[-3000:]


def test_must_confined_to_one_tile(synth):
    """A MUST clause that lives in tile 3 only: every other tile is published empty, the results are tile 3's."""
    from searcharray_b200 import Bool, Boost
    queries = [Bool(must=["t3"], should=["w0", "w1"]), Bool(must=["t3"], should=["w0", "w1"], mm=2),
               Bool(filter=["t3"], should=[Boost("w0", 2), "s2"], must_not=["w1"]),
               Bool(must=["t3", "t0"], should=["w0"])]                     # no tile holds both: nothing ranks
    for k in KS:
        docs, _ = check_batch(synth.arr, queries, k, synth.oracle(), "tile 3")
        got = docs[:3][docs[:3] != 0xFFFFFFFF].astype(np.int64)
        assert len(got) and np.all((got >= 3 * TILE) & (got < 4 * TILE))
        assert np.all(docs[3] == 0xFFFFFFFF)


@pytest.mark.parametrize("slop", [0, 2])
def test_phrases_in_every_role(synth, slop):
    from searcharray_b200 import Bool, Boost, Or
    queries = [Bool(must=[["pa", "pb"]], should=["w0", "w1"]), Bool(should=["w0", "w2"], filter=[["pa", "pb"]]),
               Bool(should=["w0", "w1"], must_not=[["pa", "pb"]]),
               Bool(should=[Boost(["pa", "pb"], 2), "w2"], must_not=[["pa", "pa"]]),
               Or([Boost(["pa", "pb"], 0.5), Boost("w1", 3)]), Bool(must=[["pa", "zzz"]], should=["w0"]),
               Bool(should=["w0"], must_not=[["pb", "zzz"]]),
               Bool(must=[Boost(["pb", "pa"], 0)], should=[["pa", "pb"], "s1"], filter=["w0"], mm=1)]
    for k in KS:
        check_batch(synth.arr, queries, k, synth.oracle(slop=slop), f"slop={slop}", slop=slop)


def test_overflow_rerun(synth):
    """Bool queries whose tile overflows its candidate slots are re-run exactly."""
    from searcharray_b200 import Bool, Boost, bm25_similarity
    queries = [Bool(should=["hot", "cold"], must_not=["t0"]), Bool(must=["hot"], should=[Boost("cold", 2)]),
               Bool(filter=["w2"], should=["w0"])]
    for k in (10, 16):
        docs, scores, n_redone = synth.arr._search_topk_bool(queries, k, bm25_similarity(), 0)
        assert n_redone > 0
        for i, q in enumerate(queries):
            assert_topk(docs[i], scores[i], compose_occur(synth.oracle(), q), k, f"overflow {q!r} k={k}")


@pytest.mark.parametrize("k1, b", [(0.0, 0.75), (1.2, 1.0), (1.2, 1.5)])
def test_exotic_parameters(synth, k1, b):
    """Term clauses in every role under parameters that are not sparse-safe (NaN / -0.0 / negative scores): each
    clause's exact score is tested, as .score gives it."""
    from searcharray_b200 import Bool, Boost, Or, bm25_similarity
    sim = bm25_similarity(k1=k1, b=b)
    arr = synth.arr
    queries = [Bool(must=["w0"], should=["s1", "w1"]), Bool(filter=["w1"], should=["w0"], must_not=["s2"]),
               Bool(should=[Boost("w0", 2), "s1"], must_not=["w2"], mm=1), Or([Boost("w0", 0.5), "zzz"]),
               Bool(must=["t3"], should=["w0"], must_not=["zzz"])]
    for k in (1, 10, 32):
        check_batch(arr, queries, k, lambda c: arr.score(c, similarity=sim), f"k1={k1} b={b}", similarity=sim)


def test_shard_doc_base_global_df():
    from searcharray_b200 import Bool, Boost, Or, SearchArray
    base = 1_000_003
    local, names = synth_corpus()
    host, _ = synth_corpus(doc_base=base)
    gdf = np.asarray([int(local.term_lengths[i]) + 1000 * (i + 1) for i in range(len(names))], dtype=np.uint64)
    arr = SearchArray.from_host_index(host, doc_base=base, corpus_size=3_000_000, avg_doc_length=31.5, global_df=gdf)
    queries = [Bool(must=["w0"], should=["w2", "s1"]), Bool(should=["w0", "w2"], must_not=["s1"]),
               Bool(filter=["t0"], should=[Boost("w0", 2)]), Or([Boost(["pa", "pb"], 3), "s2"]),
               Bool(must=[["pa", "pb"]], should=["w1"], must_not=["w2"])]
    for k in (1, 10, 32):
        check_batch(arr, queries, k, lambda c: arr.score(c), "shard", doc_base=base)


def test_mixed_batch(synth):
    """Plain, Or, boosted Or and Bool queries in one batch: each equals its own answer, in query order."""
    from searcharray_b200 import And, Bool, Boost, Or
    arr = synth.arr
    mixed = ["w1", Or(["w0", "t0"], mm=2), Or([Boost("w0", 2), "s1"]), ["pa", "pb"],
             Bool(must=["w2"], should=["w0"], must_not=["s2"]), And(["s1", "w2"]), "t3",
             Bool(filter=[["pa", "pb"]], should=["w1"])]
    for k in (1, 10, 32):
        d, s = check_batch(arr, mixed, k, synth.oracle(), "mixed")
        for idx, sub in (([0, 3, 6], ["w1", ["pa", "pb"], "t3"]), ([1, 5], [mixed[1], mixed[5]]),
                         ([2, 4, 7], [mixed[2], mixed[4], mixed[7]])):
            wd, ws = arr.search_topk(sub, k=k)
            assert np.array_equal(d[idx], wd) and np.array_equal(s[idx].view(np.uint32), ws.view(np.uint32))


def test_unit_weights_take_the_or_path(synth, monkeypatch):
    """An Or / And whose weights are all 1.0 gives the unboosted query's bits, through the Or / And instance (NULL
    weights and roles); a Bool with only SHOULD clauses of weight 1 gives the same bits through the occur instance."""
    from searcharray_b200 import And, Bool, Boost, Or
    from searcharray_b200.query import OR_AND, bool_form
    arr = synth.arr
    plain = [Or(["w0", ["pa", "pb"], "s1"], mm=2), And(["w1", "w2"]), Or(["t0", "w0", "t3"])]
    unit = [Or([Boost("w0", 1), ["pa", "pb"], Boost("s1", 1.0)], mm=2), And([Boost("w1", 1), Boost("w2", 1)]),
            Or([Boost("t0", 1), "w0", "t3"])]
    as_bool = [Bool(should=q.clauses, mm=q.mm) for q in plain]
    for k in (1, 10, 32):
        wd, ws = arr.search_topk(plain, k=k)
        bd, bs = arr.search_topk(as_bool, k=k)
        assert [bool_form(q) for q in unit] == [OR_AND] * len(unit)
        from searcharray_b200.postings import _PreparedBool
        seen, real = [], _PreparedBool.run

        def spy(self, *a):
            seen.append((self.batch.weights, self.batch.occurs))
            return real(self, *a)
        with monkeypatch.context() as m:
            m.setattr(_PreparedBool, "run", spy)
            gd, gs = arr.search_topk(unit, k=k)
        assert seen == [(None, None)], "unit weights took the occur instance"
        assert np.array_equal(gd, wd) and np.array_equal(gs.view(np.uint32), ws.view(np.uint32))
        assert np.array_equal(bd, wd) and np.array_equal(bs.view(np.uint32), ws.view(np.uint32))


def test_launches_one_tile_launch_per_group(synth):
    """A term-only Bool batch is one tile launch and one select, whatever the number of queries."""
    from searcharray_b200 import Bool, Boost, _lib
    arr = synth.arr
    h = arr._device().handle
    launches = []
    for nq in (1, 4, 64):
        queries = [Bool(must=["w0"], should=[Boost("w1", 2), "s1"], must_not=["t0"], mm=i % 3) for i in range(nq)]
        arr.search_topk(queries, k=10)                      # warm: the norm table for these parameters
        _lib.check(_lib.lib().sa_stats_reset(h))
        arr.search_topk(queries, k=10)
        st = _lib.SaStats()
        _lib.check(_lib.lib().sa_stats_get(h, ctypes.byref(st)))
        launches.append(st.total_launches)
    assert launches == [2, 2, 2], launches


def test_c_abi_validation(synth):
    """The entry point checks occur values, weights and mm against the SHOULD clauses."""
    from searcharray_b200 import _lib
    arr = synth.arr
    h = arr._device().handle
    tid = arr.host.term_dict.term_to_ids
    terms = np.asarray([tid["w0"], tid["w1"]], dtype=np.uint32)
    q_starts = np.asarray([0, 2], dtype=np.uint32)
    c_starts = np.asarray([0, 1, 2], dtype=np.uint32)
    idf = np.ones(2, dtype=np.float32)
    docs = np.empty(10, dtype=np.uint32)
    scores = np.empty(10, dtype=np.float32)

    def call(weights, occurs, mm):
        w = np.asarray(weights, dtype=np.float32)
        o = np.asarray(occurs, dtype=np.uint8)
        m = np.asarray([mm], dtype=np.uint32)
        return _lib.lib().sa_score_batch_topk_bool(
            h, 1, _lib.p_u32(q_starts), None, _lib.p_u32(terms), _lib.p_u32(c_starts), _lib.p_f32(idf), _lib.p_f32(w),
            _lib.p_u8(o), None, None, _lib.p_u32(m), 1, 0, arr.avg_doc_length, 1.2, 0.75, 10, None, 0, 0,
            _lib.p_u32(docs), _lib.p_f32(scores), None, 0, None, None, None, None)
    assert call([1, 1], [1, 0], 1) == 0
    assert call([1, 1], [1, 0], 2) != 0                       # one SHOULD clause
    assert call([1, 1], [1, 4], 0) != 0
    assert call([1, -1], [1, 0], 0) != 0
    assert call([1, float("nan")], [1, 0], 0) != 0


def test_golden(synth):
    """The real reference's composed top 10 of every Bool / boosted Or record: ids and score bits."""
    from searcharray_b200 import SearchArray
    with open(os.path.join(GOLDEN, "bool_occur.json")) as f:
        fixture = json.load(f)
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    arrs = {f: SearchArray.from_host_index(load_field(z, f)) for f in ("title_tokens", "overview_tokens")}
    arrs["scenario"] = SearchArray.index(expand(fixture["scenario_docs"]))
    for corpus, arr in arrs.items():
        recs = [r for r in fixture["queries"] if r["corpus"] == corpus]
        assert recs
        docs, scores = arr.search_topk([query_of(r) for r in recs], k=10)
        for i, r in enumerate(recs):
            n = len(r["top_ids"])
            what = f"{corpus} {query_of(r)!r}"
            assert docs[i][:n].tolist() == r["top_ids"], what
            assert scores[i][:n].view(np.uint32).tolist() == r["top_bits"], what
            assert np.all(docs[i][n:] == 0xFFFFFFFF), what
        for k in KS:
            check_batch(arr, [query_of(r) for r in recs], k, lambda c: arr.score(c), corpus)

