"""GPU: hit and facet counts of the batched top-k (search_topk / fields_topk with `facets=`; the COUNT instances of
bool_tile in sa_bool.cu and sa_index_set_facet in sa_feature.cu) against numpy over the dense ranked vector S_q that
compose_nested builds from .score (and Feature.apply): total == np.count_nonzero(S_q) and every facet row ==
np.bincount(codes[(S_q > 0) & (codes >= 0)]), exactly; docs and score bits equal to the call without `facets`.

The corpus is tests/test_bool_topk_gpu.py's five-tile synthetic one.  Its facet columns: `lang` (20 buckets, ~10 %
of docs without a value), `none` (every doc without a value), `tail` (codes in the last, partial tile only), `one`
(n_buckets = 1) and `wide` (1,024 buckets, code = doc % 1024, so a query that ranks every doc hits every bucket)."""
import os

import numpy as np
import pandas as pd
import pytest

from _nested_compose import compose_nested
from _tmdb_index import load_field
from conftest import GOLDEN
from test_bool_fields_gpu import A, B, fb_corpus
from test_bool_topk_gpu import TILE, synth_corpus

pytestmark = pytest.mark.gpu

N = 5 * TILE + 300


def facet_columns(n=N, seed=8):
    rng = np.random.default_rng(seed)
    lang = np.where(rng.random(n) < 0.1, -1, rng.integers(0, 20, n))
    tail = np.full(n, -1)
    tail[5 * TILE:] = rng.integers(0, 7, n - 5 * TILE)
    one = np.where(rng.random(n) < 0.7, 0, -1)
    return {"lang": (lang, 20), "none": (np.full(n, -1), 3), "tail": (tail, 7), "one": (one, 1),
            "wide": (np.arange(n) % 1024, 1024)}


def setup(arr, n=N):
    for name, (codes, nb) in facet_columns(n).items():
        arr.set_facet(name, codes, nb)
    arr.set_feature("all", np.ones(n, dtype=np.float32))
    arr.set_feature("pop", np.where(np.random.default_rng(2).random(n) < 0.8, 3.0, 0.0).astype(np.float32))


@pytest.fixture(scope="module")
def arr():
    from searcharray_b200 import SearchArray
    host, _ = synth_corpus()
    a = SearchArray.from_host_index(host)
    setup(a)
    return a


def dense_of(arr, q, slop=0):
    """S_q before the mask: .score of a plain query, compose_nested of a boolean one."""
    from searcharray_b200 import Feature
    from searcharray_b200.query import is_boolean
    if not is_boolean(q):
        return arr.score(q, slop=slop)

    def score(c):
        if isinstance(c, Feature):
            return c.apply(arr.host.features[c.name])
        return arr.score(c, slop=slop)
    return compose_nested(score, q)


def assert_counts(hits, i, dense, codes_of, facets, what):
    assert hits.total.dtype == np.int64 and hits.total[i] == np.count_nonzero(dense), \
        f"{what}: total {hits.total[i]} want {np.count_nonzero(dense)}"
    for f in facets:
        codes, nb = codes_of(f)
        want = np.bincount(codes[(dense > 0) & (codes >= 0)], minlength=nb)
        got = hits.facets[f][i]
        assert got.dtype == np.int64 and got.shape == (nb,), (what, f, got.shape)
        assert np.array_equal(got, want), f"{what} {f}: {np.flatnonzero(got != want)[:10]} differ"


def check(arr, queries, facets, what, k=10, where=None, slop=0):
    d0, s0 = arr.search_topk(queries, k=k, where=where, slop=slop)
    d, s, hits = arr.search_topk(queries, k=k, where=where, slop=slop, facets=facets)
    assert np.array_equal(d, d0) and np.array_equal(s.view(np.uint32), s0.view(np.uint32)), what
    assert hits.total.shape == (len(queries),) and set(hits.facets) == set(facets)
    m = None if where is None else np.asarray(where)
    for i, q in enumerate(queries):
        dense = dense_of(arr, q, slop)
        if m is not None:
            dense = np.where(m if m.ndim == 1 else m[i], dense, np.float32(0))
        assert_counts(hits, i, dense, lambda f: arr.host.facets[f], facets, f"{what} {q!r}")
    return hits


def test_plain_terms_and_phrases(arr):
    check(arr, ["w0", "s1", "t3", "zzz", "hot"], ["lang", "tail"], "terms")
    for slop in (0, 2):
        check(arr, [["pa", "pb"], ["pa", "pa"], "w2", ["pa", "zzz"]], ["lang", "one"], f"phrases slop={slop}",
              slop=slop)


def test_forms(arr):
    """Or / And / mm, Bool with filter and must_not, DisMax, nested and Feature queries in one mixed batch with plain
    ones: the counts scatter back into query order."""
    from searcharray_b200 import And, Bool, Boost, DisMax, Feature, Or
    qs = [Or(["w0", "w1", "s1"]), "w1", And(["w0", "w1"]), Or(["w2", "s1", "s2", "t0", "t3"], mm=2),
          Bool(must=["w0"], should=[Boost("w1", 2.0)], filter=["w2"]), ["pa", "pb"],
          Bool(should=["w0", "w1"], must_not=["s1", "t3"], mm=1),
          Bool(must=[DisMax(["w0", "w1"], tie=0.3)], should=["s2"]),
          Or([And(["w0", "w1"]), And(["s1", "t0"])]), Bool(should=["w1", Bool(must=["w0"], must_not=["w2"])]),
          Bool(must=["w0"], should=[Feature("pop", "saturation", pivot=2)]), Or(["t3", Feature("pop")], mm=2)]
    check(arr, qs, ["lang", "tail", "one", "none"], "forms")
    check(arr, qs, [], "totals only", k=1)


def test_where(arr):
    from searcharray_b200 import Bool, Or
    qs = [Or(["w0", "w1"]), "w2", Bool(must=["w1"], should=["s1"]), Or([["pa", "pb"], "t0"])]
    rng = np.random.default_rng(4)
    check(arr, qs, ["lang", "wide"], "where one", where=rng.random(N) < 0.3)
    per = rng.random((len(qs), N)) < 0.5
    per[0, :3 * TILE] = False                     # whole tiles emptied by the mask
    per[1, TILE:] = False
    per[3] = False
    check(arr, qs, ["lang", "tail"], "where per query", where=per)


def test_nothing_and_everything(arr):
    """A query that ranks nothing counts 0; one that ranks every doc counts N and hits every bucket of `wide`."""
    from searcharray_b200 import Bool, Feature, Or
    hits = check(arr, [Or(["zzz"]), Bool(should=[Feature("all")]), "zzz"], ["wide", "lang", "one", "none"], "extremes")
    assert hits.total.tolist() == [0, N, 0]
    assert (hits.facets["wide"][1] > 0).all() and hits.facets["wide"][1].sum() == N
    assert (hits.facets["none"] == 0).all()
    assert hits.facets["one"][1, 0] == np.count_nonzero(facet_columns()["one"][0] == 0)


def test_overflow_rerun_counts_once(arr):
    """test_overflow_rerun's batch: a re-run query is counted by the first pass only."""
    from searcharray_b200 import Or, bm25_similarity
    qs = [Or(["hot", "cold"]), Or(["hot", "cold", "w0"], mm=1), Or(["w2"])]
    for k in (10, 16):
        d0, s0, _ = arr._search_topk_bool(qs, k, bm25_similarity(), 0)
        docs, scores, n_redone, hits = arr._search_topk_bool(qs, k, bm25_similarity(), 0, facets=["lang", "wide"])
        assert n_redone > 0
        assert np.array_equal(docs, d0) and np.array_equal(scores.view(np.uint32), s0.view(np.uint32))
        for i, q in enumerate(qs):
            assert_counts(hits, i, dense_of(arr, q), lambda f: arr.host.facets[f], ["lang", "wide"], f"overflow {q!r}")


def test_four_facets_and_reset(arr):
    """Four facets in one call; a name set again is counted with its new codes."""
    from searcharray_b200 import Or, SearchArray
    check(arr, [Or(["w0", "s2"]), "w1"], ["wide", "lang", "tail", "one"], "four")
    host, _ = synth_corpus()
    b = SearchArray.from_host_index(host)
    b.search_topk(["w0"], k=5)                    # the device index exists before the facet is set
    cols = facet_columns()
    b.set_facet("x", *cols["lang"])
    check(b, [Or(["w0", "s2"])], ["x"], "set after device")
    b.set_facet("x", *cols["tail"])
    check(b, [Or(["w0", "s2"])], ["x"], "set again")


def test_c_abi_count_refusals(arr):
    """The count arguments of sa_score_batch_topk_bool, which search_topk checks before it calls: each bad one is
    SA_ERR_ARG with its message before any device work (out_docs and out_total untouched), and the same call with
    valid ones counts."""
    from searcharray_b200 import _lib
    from searcharray_b200.similarity import compute_idf
    u32 = lambda x: np.asarray(x, dtype=np.uint32)      # noqa: E731
    w0 = arr.host.term_dict.get_term_id("w0")
    idf = np.asarray([compute_idf(arr.corpus_size, np.asarray([arr.docfreq("w0")]))], dtype=np.float32)
    lang, nb = arr._facet_slot("lang")
    dev = arr._device()

    def call(fields, slots, null_counts=False):
        docs = np.full((1, 10), 7, dtype=np.uint32)
        scores = np.zeros((1, 10), dtype=np.float32)
        total = np.full(1, 7, dtype=np.uint32)
        counts = np.zeros((1, nb), dtype=np.uint32)
        with arr._shared["lock"]:
            dev.sync_facets(arr.host)
            rc = _lib.lib().sa_score_batch_topk_bool(
                dev.handle, 1, _lib.p_u32(u32([0, 1])), None, _lib.p_u32(u32([w0])), _lib.p_u32(u32([0, 1])),
                _lib.p_f32(idf), None, None, None, None, _lib.p_u32(u32([1])), 1, 0, arr.avg_doc_length, 1.2, 0.75, 10,
                None, 0, 0, _lib.p_u32(docs), _lib.p_f32(scores), None, len(slots), _lib.p_u32(u32(fields)),
                _lib.p_u32(u32(slots)), _lib.p_u32(total), None if null_counts else _lib.p_u32(counts))
        return rc, docs, total, counts

    for what, kw, msg in (("5 facets", dict(fields=[0] * 5, slots=range(5)), b"at most 4 facets in one call, not 5"),
                          ("unset slot", dict(fields=[0], slots=[7]), b"facet 0: facet slot 7 is not set"),
                          ("field 1", dict(fields=[1], slots=[lang]), b"facet 0: field 1 out of range (1 fields)"),
                          ("NULL out_facet_counts", dict(fields=[0], slots=[lang], null_counts=True),
                           b"NULL argument")):
        rc, docs, total, _ = call(**kw)
        assert rc == 2 and msg in _lib.lib().sa_last_error(), (what, rc, _lib.lib().sa_last_error())
        assert (docs == 7).all() and total[0] == 7, what
    rc, docs, total, counts = call([0], [lang])
    assert rc == 0, _lib.lib().sa_last_error()
    dense = arr.score("w0")
    codes = arr.host.facets["lang"][0]
    assert total[0] == np.count_nonzero(dense) > 0
    assert np.array_equal(counts[0], np.bincount(codes[(dense > 0) & (codes >= 0)], minlength=nb))


def test_shard_doc_base():
    from searcharray_b200 import And, Or, SearchArray
    base = 1_000_003
    host, _ = synth_corpus(doc_base=base)
    arr = SearchArray.from_host_index(host, doc_base=base, corpus_size=3_000_000, avg_doc_length=31.5,
                                      global_df=np.full(host.n_terms, 5000, dtype=np.uint64))
    setup(arr)
    check(arr, [Or(["w0", "w2", "s1"], mm=2), And(["t0", "w0"]), "w1"], ["lang", "tail"], "shard")


def test_phrase_rows_span_two_groups():
    """test_phrase_rows_span_two_groups' ~2M-doc batch, whose phrase rows need two launch groups."""
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
    arr.set_facet("m", np.where(rng.random(n) < 0.05, -1, rng.integers(0, 300, n)), 300)
    queries = [Or([["pa", "pb"]] * 63 + ["x"], mm=1 + i % 2) for i in range(9)]   # 567 phrase rows
    check(arr, queries, ["m"], "2M docs")


def test_fields_topk():
    """A facet on a column no clause reads, one on a second name of a clause's column, and where=."""
    from searcharray_b200 import Bool, DisMax, Field, Or, SearchArray, fields_topk
    ha, _ = synth_corpus()
    hb, _ = fb_corpus()
    frame = pd.DataFrame({A: SearchArray.from_host_index(ha), B: SearchArray.from_host_index(hb)})
    frame["fa2"] = frame[A]
    cols = facet_columns()
    frame[A].array.set_facet("lang", *cols["lang"])
    frame[B].array.set_facet("tail", *cols["tail"])
    frame[B].array.set_facet("wide", *cols["wide"])

    def score(c):
        return frame[c.field].array.score(c.clause)
    codes = {(A, "lang"): cols["lang"], ("fa2", "lang"): cols["lang"], (B, "tail"): cols["tail"],
             (B, "wide"): cols["wide"]}
    only_a = [Or([Field(A, "w0"), Field(A, "s1")]), Bool(must=[Field(A, "w1")], must_not=[Field(A, "t3")])]
    mixed = only_a + [Bool(should=[DisMax([Field(A, "w0"), Field(B, "b1")], tie=0.3), Field("fa2", "w2")])]
    rng = np.random.default_rng(6)
    for qs, facets, where in ((only_a, [(B, "tail"), (B, "wide")], None),
                              (mixed, [("fa2", "lang"), (B, "wide"), (A, "lang")], None),
                              (mixed, [(B, "tail")], rng.random(N) < 0.4), (only_a, [], None)):
        d0, s0 = fields_topk(frame, qs, k=10, where=where)
        d, s, hits = fields_topk(frame, qs, k=10, where=where, facets=facets)
        assert np.array_equal(d, d0) and np.array_equal(s.view(np.uint32), s0.view(np.uint32))
        for i, q in enumerate(qs):
            dense = compose_nested(score, q)
            if where is not None:
                dense = np.where(where, dense, np.float32(0))
            assert_counts(hits, i, dense, lambda f: codes[f], facets, f"fields {q!r} {facets}")


def test_tmdb():
    """Title and overview queries on the TMDB corpus, counted by original language and release decade."""
    from searcharray_b200 import And, Bool, Or, SearchArray
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    fz = np.load(os.path.join(GOLDEN, "tmdb_facets.npz"))
    cols = {"lang": fz["original_language"], "decade": fz["decade"]}
    queries = {"title_tokens": [Or(["Star", "Wars"]), "the", And(["of", "the"]), ["Star", "Wars"]],
               "overview_tokens": [Or(["love", "war"], mm=1), Bool(must=["a"], should=["young"], must_not=["the"]),
                                   "family", Or(["zzzzunknown"])]}
    for field, qs in queries.items():
        arr = SearchArray.from_host_index(load_field(z, field))
        for name, codes in cols.items():
            arr.set_facet(name, codes, int(codes.max()) + 1)
        hits = check(arr, qs, ["lang", "decade"], f"tmdb {field}")
        assert hits.total.max() > 100
