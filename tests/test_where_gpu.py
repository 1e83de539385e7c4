"""GPU: the `where=` document mask of search_topk and fields_topk (where_bits of sa_score_batch_topk_bool,
sa_multi_score_batch_topk_bool and sa_score_batch_topk_sim; the WHERE instances of bool_tile_kernel in sa_bool.cu,
sim_where_tile_kernel in sa_view.cu).  For every query the result must be the top k of np.where(mask_q, S_q, 0),
S_q being what the call without a mask ranks -- .score for a plain query, compose_nested over .score for a boolean
one, the per-field composition for fields_topk -- ids exact and score bits exact, so a mask never changes a score.

The masks cover the kernel's branches: all true (equal to the unmasked call), all false, random, a contiguous range
off the 8,192-doc tile grid, every other tile empty (the early exit), a single doc, the last partial tile only, a
mask that removes each tile's best docs of a dense term (a tile bound taken before the mask would lose the allowed
docs below it) and a different mask per query."""
import os

import numpy as np
import pandas as pd
import pytest

from _bool_fields_compose import field_scorer
from _nested_compose import compose_nested
from _tmdb_index import load_field
from conftest import GOLDEN
from test_view_topk_gpu import N_DOCS, random_host

pytestmark = pytest.mark.gpu

NO_DOC = 0xFFFFFFFF
TILE = 8192
KS = (1, 10, 32)


def want(dense, k):
    """The top k of dense (score > 0, score desc, id asc) in dense's dtype; empty slots NO_DOC / 0."""
    nz = np.flatnonzero(dense > 0)
    order = nz[np.lexsort((nz, -dense[nz].astype(np.float64)))][:k]
    docs = np.full(k, NO_DOC, dtype=np.uint32)
    scores = np.zeros(k, dtype=dense.dtype)
    docs[:len(order)] = order
    scores[:len(order)] = dense[order]
    return docs, scores


def check(docs, scores, dense, mask, what):
    wd, ws = want(np.where(mask, dense, dense.dtype.type(0)), docs.shape[-1])
    assert scores.dtype == dense.dtype, what
    assert np.array_equal(docs, wd), f"{what}: ids {docs} want {wd}"
    assert np.array_equal(scores.view(np.uint8), ws.view(np.uint8)), f"{what}: scores {scores} want {ws}"


@pytest.fixture(scope="module")
def corpus():
    from searcharray_b200 import SearchArray
    host = random_host(np.random.default_rng(11), N_DOCS, 12, 0.6)
    arr = SearchArray.from_host_index(host)
    dfs = np.asarray([arr.docfreq(f"t{i}") for i in range(12)])
    return arr, [f"t{i}" for i in np.argsort(dfs)]          # terms by df, rarest first


def queries_of(terms, slop):
    """Every query kind over the corpus' terms (a phrase with the call's slop), rarest term first."""
    from searcharray_b200 import And, Bool, Boost, DisMax, Or
    r0, r1, r2, mid, d1, d0 = terms[0], terms[1], terms[3], terms[6], terms[-2], terms[-1]
    return [r0, mid, d0, "missing", [d0, d1], [mid, d0, d1],
            Or([r2, mid]), And([d1, d0]), Or([r1, mid, d1], mm=2), Or([[d0, d1], r2]),
            Bool(must=[d1], should=[Boost(mid, 2.0), Boost(r2, 0.0)], filter=[d0], must_not=[r1]),
            Bool(should=[Boost(d0, 0.5), mid], must_not=["missing"], mm=1),
            DisMax([mid, Boost(d1, 1.5)], tie=0.3),
            Or([And([d0, d1]), And([mid, r2])]),
            Bool(must=[Or([d0, mid], mm=1)], must_not=[And([d1, r1])])]


def dense_of(arr, q, slop):
    from searcharray_b200.query import is_boolean
    if is_boolean(q):
        return compose_nested(lambda c: arr.score(c, slop=slop), q)
    return np.asarray(arr.score(q, slop=slop), dtype=np.float32)


def masks(arr, dense_term):
    """name -> bool[N] over the corpus, as the module docstring lists them."""
    n = len(arr)
    rng = np.random.default_rng(3)
    tile = np.arange(n) // TILE
    s = np.asarray(arr.score(dense_term))
    best = np.zeros(n, dtype=bool)                     # each tile's 64 best docs of the dense term
    for t in range(tile[-1] + 1):
        idx = np.flatnonzero(tile == t)
        best[idx[np.argsort(-s[idx], kind="stable")[:64]]] = True
    one = np.zeros(n, dtype=bool)
    one[int(np.argmax(s))] = True
    return {
        "all": np.ones(n, dtype=bool),
        "none": np.zeros(n, dtype=bool),
        "random30": rng.random(n) < 0.3,
        "random1": rng.random(n) < 0.01,
        "range": (np.arange(n) >= 10_001) & (np.arange(n) < 123_457),
        "odd_tiles_empty": (tile % 2 == 0) & (rng.random(n) < 0.5),
        "one_doc": one,
        "last_partial_tile": tile == tile[-1],
        "minus_tile_best": ~best,
    }


@pytest.mark.parametrize("slop", [0, 2])
def test_masks_every_query_kind(corpus, slop):
    """One mixed batch of every query kind under each mask: search_topk(where=m) against np.where(m, S_q, 0)."""
    arr, terms = corpus
    queries = queries_of(terms, slop)
    dense = [dense_of(arr, q, slop) for q in queries]
    for name, m in masks(arr, terms[-1]).items():
        for k in KS:
            docs, scores = arr.search_topk(queries, k=k, slop=slop, where=m)
            assert docs.shape == (len(queries), k) and docs.dtype == np.uint32
            for i, q in enumerate(queries):
                check(docs[i], scores[i], dense[i], m, f"{name} {q!r} k={k} slop={slop}")
            if name == "all":                          # bit for bit the unmasked call
                d0, s0 = arr.search_topk(queries, k=k, slop=slop)
                assert np.array_equal(docs, d0) and np.array_equal(scores.view(np.uint32), s0.view(np.uint32))
            if name == "none":
                assert np.all(docs == NO_DOC) and np.all(scores == 0)


def test_mask_per_query(corpus):
    """A (Q, N) mask: each query ranks under its own row, in a batch split by kind; a boolean pd.Series is a mask."""
    arr, terms = corpus
    queries = queries_of(terms, 0)
    rng = np.random.default_rng(9)
    m = rng.random((len(queries), len(arr))) < rng.uniform(0.005, 0.9, (len(queries), 1))
    for k in KS:
        docs, scores = arr.search_topk(queries, k=k, where=m)
        for i, q in enumerate(queries):
            check(docs[i], scores[i], dense_of(arr, q, 0), m[i], f"row {i} {q!r} k={k}")
    series = pd.Series(m[0])
    docs, scores = arr.search_topk(queries[:3], k=10, where=series)
    for i, q in enumerate(queries[:3]):
        check(docs[i], scores[i], dense_of(arr, q, 0), m[0], f"series {q!r}")


@pytest.mark.parametrize("view", ["array", "mask_view", "stepped_view"])
def test_similarities_and_views(corpus, view):
    """bm25_impact, bm25_legacy_similarity and classic_similarity (and BM25 on a view) through the sim tile pass,
    with the mask over the view's positions, in the similarity's dtype."""
    from searcharray_b200 import bm25_impact, bm25_legacy_similarity, bm25_similarity, classic_similarity
    arr, terms = corpus
    rng = np.random.default_rng(4)
    a = {"array": arr, "mask_view": arr[rng.random(len(arr)) < 0.4], "stepped_view": arr[1::3]}[view]
    sims = [bm25_impact(), bm25_legacy_similarity(), classic_similarity()]
    if view != "array":
        sims.append(bm25_similarity())
    queries = [terms[0], terms[6], terms[-1], "missing", [terms[-1], terms[-2]]]
    per_query = rng.random((len(queries), len(a))) < 0.2
    for sim in sims:
        dense = [np.asarray(a.score(q, similarity=sim)) for q in queries]
        for name, m in (("random", rng.random(len(a)) < 0.3), ("range", np.arange(len(a)) >= len(a) // 3),
                        ("per_query", per_query)):
            for k in KS:
                docs, scores = a.search_topk(queries, k=k, similarity=sim, where=m)
                for i, q in enumerate(queries):
                    mq = m[i] if m.ndim == 2 else m
                    check(docs[i], scores[i], dense[i], mq, f"{view} {sim!r} {name} {q!r} k={k}")


def test_fields_topk_tmdb():
    """fields_topk on the TMDB title + overview frame under both mask shapes."""
    from searcharray_b200 import And, Bool, Boost, DisMax, Field, Or, SearchArray, fields_topk
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    T, O = "title_tokens", "overview_tokens"
    frame = pd.DataFrame({f: SearchArray.from_host_index(load_field(z, f)) for f in (T, O)})
    score = field_scorer({f: frame[f].array.score for f in (T, O)})
    queries = [Or([Field(T, "star"), Field(O, "war")]),
               Bool(must=[Field(O, "the")], should=[Boost(Field(T, "love"), 2.0)], must_not=[Field(O, "murder")]),
               Or([DisMax([Boost(Field(T, "alien"), 2.0), Field(O, "alien")], tie=0.1), Field(O, "space")]),
               Or([And([Field(T, "star"), Field(T, "wars")]), And([Field(O, "star"), Field(O, "trek")])]),
               Or([Field(O, ["the", "world"]), Field(T, "man")])]
    dense = [compose_nested(score, q) for q in queries]
    rng = np.random.default_rng(2)
    n = len(frame)
    for m in (rng.random(n) < 0.25, np.arange(n) < n // 2, rng.random((len(queries), n)) < 0.5):
        for k in KS:
            docs, scores = fields_topk(frame, queries, k=k, where=m)
            for i, q in enumerate(queries):
                check(docs[i], scores[i], dense[i], m[i] if m.ndim == 2 else m, f"tmdb {q!r} k={k}")


def test_fields_topk_synthetic_frame():
    """fields_topk on the two-column multi-tile synthetic frame of the boolean field tests, both mask shapes."""
    from test_bool_fields_gpu import A, B, Frame
    from searcharray_b200 import And, Bool, Field, Or, fields_topk
    fr = Frame()
    frame = fr.frame
    score = fr.score()
    queries = [Or([Field(A, "w0"), Field(B, "b1")]), Bool(must=[Field(B, "b1")], should=[Field(A, "w1")]),
               Or([And([Field(A, "w0"), Field(B, "w0")]), Field(B, "b2")])]
    dense = [compose_nested(score, q) for q in queries]
    rng = np.random.default_rng(8)
    n = len(frame)
    tile = np.arange(n) // TILE
    for m in (tile % 2 == 1, rng.random(n) < 0.05, rng.random((len(queries), n)) < 0.3):
        for k in KS:
            docs, scores = fields_topk(frame, queries, k=k, where=m)
            for i, q in enumerate(queries):
                check(docs[i], scores[i], dense[i], m[i] if m.ndim == 2 else m, f"synthetic {q!r} k={k}")


def test_fields_topk_without_nested_queries():
    """Batches with no nested query take the masked fields instance (Or / Bool of Field clauses) and the masked DisMax
    instance over a field table: both mask shapes, on TMDB and on the two-column synthetic frame."""
    from test_bool_fields_gpu import A, B, Frame
    from searcharray_b200 import Bool, Boost, DisMax, Field, Or, SearchArray, fields_topk
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    T, O = "title_tokens", "overview_tokens"
    tmdb = pd.DataFrame({f: SearchArray.from_host_index(load_field(z, f)) for f in (T, O)})
    fr = Frame()
    cases = [
        (tmdb, field_scorer({f: tmdb[f].array.score for f in (T, O)}),
         [Or([Field(T, "star"), Field(O, "war")]), Or([Field(T, "love"), Field(O, "love"), Field(O, "war")], mm=2),
          Bool(must=[Field(O, "the")], should=[Boost(Field(T, "love"), 2.0)], must_not=[Field(O, "murder")]),
          Or([Field(O, ["the", "world"]), Field(T, "man")])],
         [Or([DisMax([Boost(Field(T, "alien"), 2.0), Field(O, "alien")], tie=0.1), Field(O, "space")]),
          Bool(must=[DisMax([Field(T, "love"), Field(O, "love")], tie=0.3)], must_not=[Field(O, "war")])]),
        (fr.frame, fr.score(),
         [Or([Field(A, "w0"), Field(B, "b1")]), Bool(must=[Field(B, "b1")], should=[Field(A, "w1")]),
          Bool(filter=[Field(B, "b2")], should=[Boost(Field(A, "w0"), 0.5), Field(B, "w0")])],
         [Or([DisMax([Field(A, "w0"), Boost(Field(B, "w0"), 2.0)], tie=0.2), Field(B, "b2")])]),
    ]
    rng = np.random.default_rng(6)
    for frame, score, flat, dismax in cases:
        n = len(frame)
        for queries in (flat, dismax):
            dense = [compose_nested(score, q) for q in queries]
            for m in (rng.random(n) < 0.2, (np.arange(n) // TILE) % 2 == 1, rng.random((len(queries), n)) < 0.4):
                for k in KS:
                    docs, scores = fields_topk(frame, queries, k=k, where=m)
                    for i, q in enumerate(queries):
                        check(docs[i], scores[i], dense[i], m[i] if m.ndim == 2 else m, f"flat {q!r} k={k}")


def test_plain_queries_as_any_iterable(corpus):
    """A phrase given as a numpy array ranks with a mask as without one; an empty phrase is refused by the same
    exception type."""
    arr, terms = corpus
    phrase = np.array([terms[-1], terms[-2]])
    m = np.ones(len(arr), dtype=bool)
    d0, s0 = arr.search_topk([phrase, terms[-1]], k=10)
    d1, s1 = arr.search_topk([phrase, terms[-1]], k=10, where=m)
    assert np.array_equal(d0, d1) and np.array_equal(s0.view(np.uint32), s1.view(np.uint32))
    with pytest.raises(Exception) as unmasked:
        arr.search_topk([[]], k=10)
    with pytest.raises(type(unmasked.value)):
        arr.search_topk([[]], k=10, where=m)


def test_overflow_rerun():
    """Every doc of tile 0 holds a term once at one length, so all tie.  Query 0's mask allows the 320 docs that
    threads 10-19 own (docs 4 t + 1024 j + e), query 1's those of threads 20-29: neither set starts at doc 0, so a
    re-run without its mask, or with another query's row, returns other ids.  With fewer threads holding a tie than
    k = 32 the tile keeps every allowed tie, more than its 256 slots: each query is re-run exactly (n_redone), the
    second through the per-query row offset of the re-run."""
    from searcharray_b200 import Or, SearchArray, bm25_similarity
    from searcharray_b200.postings import pack_where
    arr = SearchArray.index(["tie pad pad pad" if d < TILE else "pad pad pad pad" for d in range(2 * TILE + 5)])
    m = np.zeros((2, len(arr)), dtype=bool)
    for row, t0 in enumerate((10, 20)):
        m[row, [4 * t + 1024 * j + e for t in range(t0, t0 + 10) for j in range(8) for e in range(4)]] = True
    dense = np.asarray(arr.score("tie"))
    for k in (10, 32):
        for where, rows in ((m[0], [0]), (m, [0, 1])):
            queries = ["tie"] * len(rows)
            docs, scores = arr.search_topk(queries, k=k, where=where)
            for i, r in enumerate(rows):
                check(docs[i], scores[i], dense, m[r], f"tie k={k} row {r}")
            d, s, n_redone = arr._search_topk_bool([Or(["tie"])] * len(rows), k, bm25_similarity(), 0,
                                                   pack_where(where, len(arr), len(rows)))
            assert k == 10 or n_redone == len(rows)
            assert np.array_equal(d, docs) and np.array_equal(s.view(np.uint32), scores.view(np.uint32))


def test_shard_rows():
    """On a doc-range shard the mask indexes the shard's own rows; ids are global."""
    from searcharray_b200 import Or, SearchArray
    from searcharray_b200.indexing import index_from_term_postings
    host = random_host(np.random.default_rng(12), 3 * TILE + 77, 6, 0.5)
    base = 1_000_003
    words = [host.term_words(t) + (np.uint64(base) << np.uint64(36)) for t in range(host.n_terms)]
    shard = SearchArray.from_host_index(
        index_from_term_postings([f"t{i}" for i in range(host.n_terms)], words, host.doc_lens), doc_base=base)
    m = np.random.default_rng(1).random(len(shard)) < 0.3
    queries = ["t0", "t3", Or(["t1", "t2"])]
    docs, scores = shard.search_topk(queries, k=10, where=m)
    for i, q in enumerate(queries):
        dense = dense_of(shard, q, 0)
        wd, ws = want(np.where(m, dense, np.float32(0)), 10)
        wd = np.where(wd == NO_DOC, wd, wd + np.uint32(base))
        assert np.array_equal(docs[i], wd) and np.array_equal(scores[i].view(np.uint32), ws.view(np.uint32)), q
