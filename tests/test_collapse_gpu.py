"""GPU: collapsed batched top-k (search_topk / fields_topk with `collapse=`; the COLLAPSE instances of bool_tile and
collapse_tile_collect, topk_collapse_kernel in sa_topk.cu, sa_index_set_group in sa_feature.cu) against collapse_ref
over the dense ranked vector S_q that compose_nested builds from .score (and Feature.apply, Range / In matches): ids and
score bits exact.

The corpus is tests/test_bool_topk_gpu.py's five-tile synthetic one.  Its group columns: `distinct` (arange) and
`none` (every doc -1), which return the call without `collapse` bit for bit; `pairs` ((doc + 1) // 2, groups across
the tile edges); `sparse` (half the docs -1, the others in ~N/6 groups); `tiny` (3 groups: fewer groups than k);
`tail` (groups only in the partial last tile); and `dominant`, one group holding each tile's 2,500 best docs of "w0",
so that a tile walks its ranked docs in several windows."""
import os

import numpy as np
import pandas as pd
import pytest

from _nested_compose import compose_nested
from _tmdb_index import load_field
from conftest import GOLDEN
from test_bool_fields_gpu import A, B, fb_corpus
from test_bool_topk_gpu import TILE, synth_corpus
from test_collapse_cpu import collapse_ref

pytestmark = pytest.mark.gpu

N = 5 * TILE + 300
K_VALUES = (1, 10, 32, 33, 100, 1024)


def group_columns(arr, n=N, seed=9):
    rng = np.random.default_rng(seed)
    sparse = np.where(rng.random(n) < 0.5, -1, rng.integers(0, n // 6, n))
    tail = np.full(n, -1)
    tail[5 * TILE:] = rng.integers(0, 5, n - 5 * TILE)
    dominant = np.arange(n) + 1
    s = arr.score("w0")
    for t in range(0, n, TILE):                       # each tile's 2,500 best docs of w0: group 0
        ids = np.arange(t, min(n, t + TILE))
        ranked = ids[s[ids] > 0]
        dominant[ranked[np.lexsort((ranked, -s[ranked].astype(np.float64)))][:2500]] = 0
    return {"distinct": np.arange(n), "none": np.full(n, -1), "pairs": (np.arange(n) + 1) // 2, "sparse": sparse,
            "tiny": rng.integers(0, 3, n), "tail": tail, "dominant": dominant}


@pytest.fixture(scope="module")
def arr():
    from searcharray_b200 import SearchArray
    host, _ = synth_corpus()
    a = SearchArray.from_host_index(host)
    rng = np.random.default_rng(3)
    a.set_feature("pop", np.where(rng.random(N) < 0.8, rng.integers(1, 6, N), 0).astype(np.float32))
    a.set_feature("year", rng.integers(1950, 2020, N).astype(np.float32))
    a.set_facet("lang", np.where(rng.random(N) < 0.1, -1, rng.integers(0, 20, N)), 20)
    a.groups_ = group_columns(a)
    return a


def forms():
    from searcharray_b200 import And, Bool, Boost, DisMax, Feature, In, Or, Range
    return {
        "plain": ["w0", "w1", ["pa", "pb"], "s1", "zzz"],
        "or_and": [Or(["w0", "w1", "s1"]), And(["w0", "w1"]), Or(["w2", "s1", "s2", "t0", "t3"], mm=2)],
        "occur": [Bool(must=["w0"], should=[Boost("w1", 2.0)], filter=["w2"]),
                  Bool(should=["w0", "w1"], must_not=["s1", "t3"], mm=1), Or([["pa", "pb"], "t0"])],
        "dismax": [Bool(must=[DisMax(["w0", "w1"], tie=0.3)], should=["s2"]), DisMax(["w1", "t3"], tie=0.0)],
        "nested": [Or([And(["w0", "w1"]), And(["s1", "t0"])]), Bool(should=["w1", Bool(must=["w0"], must_not=["w2"])])],
        "columns": [Bool(must=["w0"], should=[Feature("pop", "saturation", pivot=2)]),
                    Bool(must=[Or(["w0", "w1"])], filter=[Range("year", gte=1970, lt=1995), In("lang", [1, 4, 7])]),
                    Bool(should=["w1", Feature("pop")], must_not=[In("lang", [2])])],
    }


def dense_of(arr, q):
    """S_q before the mask: .score of a plain query, compose_nested of a boolean one."""
    from searcharray_b200 import Feature, In, Range
    from searcharray_b200.query import is_boolean
    if not is_boolean(q):
        return arr.score(q)

    def score(c):
        if isinstance(c, Feature):
            return c.apply(arr.host.features[c.name])
        if isinstance(c, Range):
            return c.match(arr.host.features[c.name]).astype(np.float32)
        if isinstance(c, In):
            return c.match(arr.host.facets[c.name][0]).astype(np.float32)
        return arr.score(c)
    return compose_nested(score, q)


def masked(dense, where, i):
    if where is None:
        return dense
    m = np.asarray(where)
    return np.where(m if m.ndim == 1 else m[i], dense, np.float32(0))


def check(arr, queries, dense, codes, k, what, where=None, facets=None, doc_base=0):
    """search_topk with collapse="g" (codes set on the array) against collapse_ref; with facets the hits must equal
    the call without collapse's.  Returns (docs, scores)."""
    out = arr.search_topk(queries, k=k, where=where, facets=facets, collapse="g")
    d, s = out[:2]
    assert d.shape == (len(queries), k) and s.dtype == np.float32
    for i in range(len(queries)):
        wd, ws = collapse_ref(masked(dense[i], where, i), codes, k)
        wd = np.where(wd == 0xFFFFFFFF, wd, wd + np.uint32(doc_base))
        assert np.array_equal(d[i], wd), f"{what} q{i} k={k}: ids {d[i][:12]} want {wd[:12]}"
        assert np.array_equal(s[i].view(np.uint32), ws.view(np.uint32)), f"{what} q{i} k={k}: score bits"
    if facets is not None:
        h0 = arr.search_topk(queries, k=k, where=where, facets=facets)[2]
        assert np.array_equal(out[2].total, h0.total), what
        for f in facets:
            assert np.array_equal(out[2].facets[f], h0.facets[f]), (what, f)
    return d, s


@pytest.fixture(scope="module")
def batch(arr):
    qs = [q for v in forms().values() for q in v]
    return qs, [dense_of(arr, q) for q in qs]


@pytest.mark.parametrize("column", ["distinct", "none", "pairs", "sparse", "tiny", "tail", "dominant"])
def test_forms_and_k(arr, batch, column):
    """Every form in one mixed batch, at every k, and the prefix property across k."""
    qs, dense = batch
    codes = arr.groups_[column]
    arr.set_group("g", codes)
    deepest = check(arr, qs, dense, codes, 1024, column)
    for k in K_VALUES[:-1]:
        d, s = check(arr, qs, dense, codes, k, column)
        assert np.array_equal(d, deepest[0][:, :k]) and np.array_equal(s.view(np.uint32),
                                                                      deepest[1][:, :k].view(np.uint32))


@pytest.mark.parametrize("column", ["distinct", "none"])
def test_identity_columns(arr, batch, column):
    """All codes distinct, or all -1: the call without collapse, bit for bit."""
    qs, _ = batch
    arr.set_group("g", arr.groups_[column])
    for k in K_VALUES:
        d0, s0 = arr.search_topk(qs, k=k)
        d, s = arr.search_topk(qs, k=k, collapse="g")
        assert np.array_equal(d, d0) and np.array_equal(s.view(np.uint32), s0.view(np.uint32)), (column, k)


@pytest.mark.parametrize("column", ["pairs", "sparse", "dominant"])
def test_where_and_facets(arr, batch, column):
    qs, dense = batch
    codes = arr.groups_[column]
    arr.set_group("g", codes)
    rng = np.random.default_rng(4)
    one = rng.random(N) < 0.3
    per = rng.random((len(qs), N)) < 0.5
    per[0, :3 * TILE] = False                         # whole tiles emptied by the mask
    per[1] = False
    for k in (10, 100):
        check(arr, qs, dense, codes, k, f"{column} where one", where=one)
        check(arr, qs, dense, codes, k, f"{column} where per query", where=per)
        check(arr, qs, dense, codes, k, f"{column} facets", facets=["lang"])
        check(arr, qs, dense, codes, k, f"{column} facets + where", where=per, facets=["lang"])


def test_score_docs_at_collapsed_docs(arr, batch):
    qs, _ = batch
    arr.set_group("g", arr.groups_["sparse"])
    for k in (10, 1024):
        d, s = arr.search_topk(qs, k=k, collapse="g")
        assert np.array_equal(arr.score_docs(qs, d).view(np.uint32), s.view(np.uint32)), k


def test_instances_and_windows(arr, batch):
    """Each form runs its COLLAPSE instance, masked and unmasked (bits 30 + 2 form + masked of bool_instances),
    nothing is re-run, and the dominant group makes tiles walk past their first window."""
    from searcharray_b200 import _lib, bm25_similarity
    from searcharray_b200.query import DISMAX, NESTED, OCCUR, OR_AND, bool_form, is_boolean
    qs, _ = batch
    arr.set_group("g", arr.groups_["dominant"])
    dev = arr._device()
    st = _lib.SaStats()
    mask = np.random.default_rng(5).random(N) < 0.9
    from searcharray_b200.postings import pack_where
    for form in (OR_AND, OCCUR, DISMAX, NESTED):
        part = [q for q in qs if is_boolean(q) and bool_form(q) == form]
        for m in (False, True):
            _lib.check(_lib.lib().sa_stats_reset(dev.handle))
            where = pack_where(mask, N, len(part)) if m else None
            out = arr._search_topk_bool(part, 10, bm25_similarity(), 0, where, None, "g")
            assert out[2] == 0
            _lib.check(_lib.lib().sa_stats_get(dev.handle, st))
            c_form = {OR_AND: 0, OCCUR: 1, DISMAX: 3, NESTED: 4}[form]     # the C table's forms (2: fields)
            assert st.bool_instances >> 30 == 1 << (2 * c_form + m), (form, m, hex(st.bool_instances))
            assert st.collapse_tiles > 0 and st.deep_tiles == 0
    _lib.check(_lib.lib().sa_stats_reset(dev.handle))
    arr.search_topk(["w0"], k=10, collapse="g")
    _lib.check(_lib.lib().sa_stats_get(dev.handle, st))
    assert st.collapse_windows > 0 and st.collapse_tiles == 6


def test_c_abi_refusals(arr):
    from searcharray_b200 import _lib
    u32 = lambda x: np.asarray(x, dtype=np.uint32)      # noqa: E731
    w0 = arr.host.term_dict.get_term_id("w0")
    dev = arr._device()
    docs = np.full((1, 10), 7, dtype=np.uint32)
    scores = np.zeros((1, 10), dtype=np.float32)
    idf = np.ones(1, dtype=np.float32)
    rc = _lib.lib().sa_score_batch_topk_bool_collapse(
        dev.handle, 3, 1, _lib.p_u32(u32([0, 1])), None, _lib.p_u32(u32([w0])), _lib.p_u32(u32([0, 1])),
        _lib.p_f32(idf), None, None, None, None, _lib.p_u32(u32([1])), 1, 0, arr.avg_doc_length, 1.2, 0.75, 10,
        None, 0, 0, _lib.p_u32(docs), _lib.p_f32(scores), None, 0, None, None, None, None)
    assert rc == 2 and b"group slot 3 is not set" in _lib.lib().sa_last_error() and (docs == 7).all()
    codes = np.zeros(N - 1, dtype=np.int32)
    assert _lib.lib().sa_index_set_group(dev.handle, 0, _lib.p_i32(codes), len(codes)) == 2
    assert _lib.lib().sa_index_set_group(dev.handle, 4, _lib.p_i32(codes), N) == 2


def test_shard_doc_base():
    from searcharray_b200 import And, Or, SearchArray
    base = 1_000_003
    host, _ = synth_corpus(doc_base=base)
    arr = SearchArray.from_host_index(host, doc_base=base, corpus_size=3_000_000, avg_doc_length=31.5,
                                      global_df=np.full(host.n_terms, 5000, dtype=np.uint64))
    codes = (np.arange(N) + 1) // 3
    arr.set_group("g", codes)
    qs = [Or(["w0", "w2", "s1"], mm=2), And(["t0", "w0"]), "w1"]
    for k in (10, 100):
        check(arr, qs, [dense_of(arr, q) for q in qs], codes, k, "shard", doc_base=base)


def test_fields_topk():
    """collapse=(column, name) on a column no clause reads, and on one a clause reads, with where and facets."""
    from searcharray_b200 import Bool, DisMax, Field, Or, SearchArray, fields_topk
    ha, _ = synth_corpus()
    hb, _ = fb_corpus()
    frame = pd.DataFrame({A: SearchArray.from_host_index(ha), B: SearchArray.from_host_index(hb)})
    codes = {A: (np.arange(N) + 1) // 2, B: np.random.default_rng(6).integers(0, 50, N)}
    frame[A].array.set_group("g", codes[A])
    frame[B].array.set_group("g", codes[B])
    frame[B].array.set_facet("f", np.arange(N) % 7, 7)

    def score(c):
        return frame[c.field].array.score(c.clause)
    qs = [Or([Field(A, "w0"), Field(A, "s1")]), Bool(must=[Field(A, "w1")], must_not=[Field(A, "t3")]),
          Bool(should=[DisMax([Field(A, "w0"), Field(B, "b1")], tie=0.3), Field(A, "w2")])]
    dense = [compose_nested(score, q) for q in qs]
    where = np.random.default_rng(7).random(N) < 0.6
    # the fields form's COLLAPSE instances (bits 30 + 2 * 2 + masked; the third query is a DisMax one)
    from searcharray_b200 import _lib
    dev = frame[A].array._device()
    st = _lib.SaStats()
    for w, bit in ((None, 34), (where, 35)):
        _lib.check(_lib.lib().sa_stats_reset(dev.handle))
        fields_topk(frame, qs[:2], k=10, where=w, collapse=(B, "g"))
        _lib.check(_lib.lib().sa_stats_get(dev.handle, st))
        assert st.bool_instances == 1 << bit, hex(st.bool_instances)
    for col in (A, B):
        for k in (10, 100):
            d, s = fields_topk(frame, qs, k=k, collapse=(col, "g"))
            d2, s2, hits = fields_topk(frame, qs, k=k, where=where, facets=[(B, "f")], collapse=(col, "g"))
            h0 = fields_topk(frame, qs, k=k, where=where, facets=[(B, "f")])[2]
            assert np.array_equal(hits.total, h0.total) and np.array_equal(hits.facets[(B, "f")], h0.facets[(B, "f")])
            for i in range(len(qs)):
                for got_d, got_s, S in ((d, s, dense[i]), (d2, s2, np.where(where, dense[i], np.float32(0)))):
                    wd, ws = collapse_ref(S, codes[col], k)
                    assert np.array_equal(got_d[i], wd) and np.array_equal(got_s[i].view(np.uint32),
                                                                           ws.view(np.uint32)), (col, k, i)


def test_select_walks_several_windows():
    """A column of 800 groups spread over every tile, with a term in every doc, at k = 1,024: each tile keeps at most 800
    leaders, so a query's 10 runs hold 8,000 keys, and the select's first window of 4,096 holds fewer than k groups.
    The select then walks a second window, below a 64-bit radix bound, with the run prefixes cut at it.  Each full tile
    walks all 8 of its windows (it never reaches k leaders), so a query counts 10 * 7 tile windows and 1 select window
    past the first."""
    from searcharray_b200 import Or, SearchArray, _lib
    from searcharray_b200.indexing import index_from_term_postings
    from searcharray_b200.roaringish import encode_postings
    n = 10 * TILE
    rng = np.random.default_rng(12)
    docs = np.arange(n)
    host = index_from_term_postings(["a"], [encode_postings(docs, np.zeros(n, dtype=np.int64))],
                                    rng.integers(1, 60, n).astype(np.float32))
    arr = SearchArray.from_host_index(host)
    codes = docs % 800
    arr.set_group("g", codes)
    qs = ["a", Or(["a"])]
    dense = [arr.score("a")] * 2
    dev = arr._device()
    st = _lib.SaStats()
    _lib.check(_lib.lib().sa_stats_reset(dev.handle))
    d, _ = check(arr, qs, dense, codes, 1024, "800 groups")
    _lib.check(_lib.lib().sa_stats_get(dev.handle, st))
    assert (d != 0xFFFFFFFF).sum(axis=1).tolist() == [800, 800]
    assert st.collapse_tiles == 2 * 10 and st.collapse_windows == 2 * (10 * 7 + 1), st.collapse_windows
    for k in (700, 801):                              # a select that stops inside its first or second window
        check(arr, qs, dense, codes, k, f"800 groups k={k}")


def test_tmdb():
    """Title queries on the TMDB corpus, one result per original language."""
    from searcharray_b200 import And, Or, SearchArray
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    fz = np.load(os.path.join(GOLDEN, "tmdb_facets.npz"))
    arr = SearchArray.from_host_index(load_field(z, "title_tokens"))
    codes = fz["original_language"].astype(np.int64)
    arr.set_group("g", codes)
    qs = [Or(["Star", "Wars"]), "the", And(["of", "the"]), ["Star", "Wars"], Or(["love", "war", "man"])]
    dense = [dense_of(arr, q) for q in qs]
    for k in (5, 50):
        d, _ = check(arr, qs, dense, codes, k, "tmdb")
        assert (d[1] != 0xFFFFFFFF).sum() > 3
