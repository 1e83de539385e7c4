"""GPU: every branch of the device edismax (sa_edismax.cu, driven by solr._run_device) against oracle.solr.edismax,
bit for bit: the score vector's dtype and bits, and edismax_topk's ids, float64 score bits and padding at
k = 1, 10, 16, 17, 32 (16 / 17 sit on either side of sa_topk_slots' 128 / 256 switch).

The synthetic corpus has 5 full 8192-doc tiles and a partial sixth, so the combine kernels' padding, the tile
collector past tile 0 and the filtered lists of every tile are read.  Per field: common terms (c0, c1, c2, >= 1,024
words: tile directory and tf table), rare ones (r1, r2: binary search over words), terms confined to tile 0 (t0, t0b)
and tile 3 (t3, t3b), phrase families adjacent in some docs and apart in others (pa pb pc, c0 c1, t0 t0b, t3 t3b),
a same-term phrase (ss ss) and `lone`, whose docs hold no other query term: under mm = 2 its list filtered to
qf > 0 is empty (the `missing` branch of sa_multi_phrases).  body has long docs, title short ones, tag tokenises a
query to its first two tokens, so a longer query is field-centric; f3 .. f8 make 8 distinct indexes."""
import ctypes
import json
import os

import numpy as np
import pandas as pd
import pytest

from _tmdb_index import load_field
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

TILE = 8192
N_DOCS = 5 * TILE + 300
KS = (1, 10, 16, 17, 32)
LONE = np.arange(5, N_DOCS, 97)          # docs holding `lone` and no other query term, in every field
WS8 = ["body", "title", "f3", "f4", "f5", "f6", "f7", "f8"]       # 8 distinct indexes, whitespace tokenizer


def first_two(text):
    return text.split()[:2]


def synth_field(seed, long):
    from searcharray_b200.indexing import index_from_term_postings
    from searcharray_b200.roaringish import encode_postings
    rng = np.random.default_rng(seed)
    n, span = N_DOCS, (250 if long else 12)
    doc_lens = (rng.integers(40, 400, n) if long else rng.integers(2, 16, n)).astype(np.float32)
    free = np.setdiff1d(np.arange(n), LONE)
    post = {}

    def put(name, docs, posns):
        d = post.setdefault(name, {})
        for doc, ps in zip(np.asarray(docs).tolist(), posns):
            d.setdefault(doc, set()).update(int(p) for p in ps)

    def pick(count, lo=0, hi=n):
        pool = free[(free >= lo) & (free < hi)]
        return np.sort(rng.choice(pool, min(count, len(pool)), replace=False))

    def rand_posns(docs):
        return [rng.integers(0, span, 1 + doc % 3).tolist() for doc in docs.tolist()]

    def follow(name, lead, docs, near, far):
        """`name` after the first position of `lead` in each of docs: `near` positions on in even docs, `far` in odd"""
        put(name, docs, [[min(post[lead][d]) + (near if d % 2 == 0 else far)] for d in docs.tolist()])

    c0 = pick(int(0.3 * n))
    put("c0", c0, rand_posns(c0))
    c1 = pick(int(0.15 * n))
    put("c1", c1, rand_posns(c1))
    follow("c1", "c0", c0[::5], 1, 7)                       # adjacent to c0 in some docs, apart in others
    c2 = pick(1700)
    put("c2", c2, rand_posns(c2))
    follow("c2", "c1", c1[::7], 1, 3)
    r1 = pick(300)
    put("r1", r1, rand_posns(r1))
    r2 = np.concatenate([pick(100, TILE, 2 * TILE), pick(100, 5 * TILE)])     # tile 1 and the partial last tile
    put("r2", r2, rand_posns(r2))
    t0 = pick(400, 0, TILE)
    put("t0", t0, rand_posns(t0))
    follow("t0b", "t0", t0[::2], 1, 5)
    t3 = pick(500, 3 * TILE, 4 * TILE)
    put("t3", t3, rand_posns(t3))
    follow("t3b", "t3", t3[::2], 1, 4)
    ph = pick(2500)
    put("pa", ph, [[10 + doc % 40] for doc in ph.tolist()])
    follow("pb", "pa", ph[ph % 5 != 0], 1, 4)
    follow("pc", "pb", ph[(ph % 5 != 0) & (ph % 3 == 0)], 1, 2)
    ss = pick(1500)
    put("ss", ss, [[20] if d % 3 == 2 else [20, 21] if d % 3 == 0 else [20, 25] for d in ss.tolist()])
    put("lone", LONE, [[3]] * len(LONE))
    names = list(post)
    words = []
    for t in names:
        docs = sorted(post[t])
        d = [doc for doc in docs for _ in post[t][doc]]
        p = [x for doc in docs for x in sorted(post[t][doc])]
        words.append(encode_postings(np.asarray(d, dtype=np.int64), np.asarray(p, dtype=np.int64)))
    return index_from_term_postings(names, words, doc_lens)


class Corpus:
    def __init__(self):
        from oracle import search as osearch
        from oracle import solr as osolr
        from searcharray_b200 import SearchArray
        from searcharray_b200.postings import ws_tokenizer
        cols, self.ofields = {}, {}

        def add(name, host, tokenizer=ws_tokenizer, **kw):
            cols[name] = SearchArray.from_host_index(host, tokenizer=tokenizer, **kw)
            avgdl = kw.get("avg_doc_length", host.avg_doc_length)
            oidx = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                                       avg_doc_length=avgdl)
            self.ofields[name] = osolr.OracleField(oidx, host.term_dict.term_to_ids, tokenizer=tokenizer)

        hosts = {}
        for i, f in enumerate(WS8):
            hosts[f] = synth_field(seed=100 + i, long=(i % 2 == 0))
            add(f, hosts[f])
        add("tag", synth_field(seed=99, long=False), tokenizer=first_two)
        add("zero", hosts["title"], avg_doc_length=0)      # its own index, avgdl 0: every score is 0
        self.frame = pd.DataFrame(cols)

    def oracle(self, ofields=None, sims=None, **kw):
        from oracle import solr as osolr
        fields = dict(self.ofields if ofields is None else ofields)
        for f, s in (sims or {}).items():
            o = fields[f]
            fields[f] = osolr.OracleField(o.index, o.term_to_id, tokenizer=o.tokenizer, k1=s.k1, b=s.b)
        return osolr.edismax(fields, **kw)


@pytest.fixture(scope="module")
def corpus():
    return Corpus()


def assert_vec(got, want, what):
    assert got.dtype == want.dtype, (what, got.dtype, want.dtype)
    bits = np.uint64 if want.dtype == np.float64 else np.uint32
    bad = np.flatnonzero(got.view(bits) != want.view(bits))
    assert len(bad) == 0, f"{what}: {len(bad)} docs differ, first {bad[:5]}: {got[bad[:5]]} want {want[bad[:5]]}"


def assert_topk(docs, scores, want, k, what):
    w = want.astype(np.float64)
    order = np.lexsort((np.arange(len(w)), -w))[:k]
    order = order[w[order] > 0]
    wd = np.full(k, 0xFFFFFFFF, dtype=np.uint32)
    ws = np.zeros(k, dtype=np.float64)
    wd[:len(order)], ws[:len(order)] = order, w[order]
    assert docs.dtype == np.uint32 and scores.dtype == np.float64
    assert np.array_equal(docs, wd), f"{what} k={k}: ids {docs} want {wd}"
    assert np.array_equal(scores.view(np.uint64), ws.view(np.uint64)), f"{what} k={k}: scores {scores} want {ws}"


def check(corpus, what, frame=None, ofields=None, sims=None, ks=KS, matches=True, **kw):
    """edismax and edismax_topk on `frame` (default: the corpus) against the oracle on `ofields`."""
    from searcharray_b200.solr import edismax, edismax_topk
    frame = corpus.frame if frame is None else frame
    want = corpus.oracle(ofields, sims, **kw)
    assert (np.count_nonzero(want) > 0) == matches, (what, np.count_nonzero(want))
    skw = dict(kw, similarity=sims) if sims else kw
    got, _ = edismax(frame, **skw)
    assert_vec(got, want, what)
    for k in ks:
        d, s = edismax_topk(frame, k=k, **skw)
        assert_topk(d, s, want, k, what)
    return want


# ------------------------------------------------------------------ term-centric combine
TERM_CENTRIC = {
    "one_field": dict(q="c0 c1 r1", qf=["body"]),
    "two_fields_tie": dict(q="c0 t3 r2", qf=["body", "title^1.0"], tie=0.3),
    "three_fields_boosts": dict(q="c1 pa t0", qf=["body^2.5", "title", "f3^0.7"], tie=1.0),
    "eight_fields": dict(q="c0 pa", qf=["body", "title^1.5", "tag", "f3", "f4^0.25", "f5", "f6", "f7"], tie=0.3),
    "eight_ws_fields": dict(q="c2 r1 t3", qf=[f + "^0.5" for f in WS8], tie=0.1, mm=2),
    "mm_int": dict(q="c0 c1 c2 r1", qf=["body", "title"], mm=2),
    "mm_pct": dict(q="c0 c1 c2 r1", qf=["body", "title"], mm="75%"),
    "mm_negative": dict(q="c0 c1 c2 r1", qf=["body", "title"], mm="-1"),
    "mm_conditional": dict(q="c0 c1 c2 r1", qf=["body", "title"], mm="2<75%"),
    "mm_conditional_low": dict(q="c0 t0", qf=["body", "title"], mm="2<75%"),
    "mm_above_count": dict(q="c0 c1 c2", qf=["body", "title"], mm=5),
    "q_op_and": dict(q="c0 c1 pa", qf=["body", "title"], q_op="AND"),
    "duplicates": dict(q="c1 c1 r1", qf=["body", "title^2"], mm=3, tie=0.3),
    "unknown_token": dict(q="c0 zzz t3", qf=["body", "title"], mm=2),
    "tile_confined": dict(q="t0 t3", qf=["body", "title"], mm=1),
}


@pytest.mark.parametrize("name", list(TERM_CENTRIC))
def test_term_centric_combine(corpus, name):
    """edismax_combine_terms_kernel: 1, 2, 3 and 8 fields, boosts absent / ^1.0 / fractional, tie 0 / 0.3 / 1.0,
    every mm form, duplicate and unknown tokens."""
    from searcharray_b200.solr import _Plan, default_bm25
    kw = TERM_CENTRIC[name]
    plan = _Plan(corpus.frame, kw["q"], kw["qf"], kw.get("mm"), None, None, None, kw.get("tie", 0.0),
                 kw.get("q_op", "OR"), default_bm25)
    assert plan.term_centric and plan.device_ok()
    check(corpus, name, **kw)


def phrase_launches(arrays):
    from searcharray_b200 import _lib
    out = {"phrase": 0, "total": 0}
    for a in {id(a._shared): a for a in arrays}.values():
        st = _lib.SaStats()
        _lib.check(_lib.lib().sa_stats_get(a._device().handle, ctypes.byref(st)))
        out["phrase"] += st.phrase_kernel_launches + st.phrase_tile_launches
        out["total"] += st.total_launches
    return out


def reset_stats(arrays):
    from searcharray_b200 import _lib
    for a in arrays:
        _lib.check(_lib.lib().sa_stats_reset(a._device().handle))


def test_unknown_tokens_only_stop_after_qf(corpus):
    """A query of unknown tokens matches nothing: _run_device returns after sa_multi_qf, before any filter or phrase
    launch, and every result is zero / padding."""
    from searcharray_b200.solr import edismax
    arrays = [corpus.frame[f].array for f in ("body", "title")]
    phases = dict(pf=["body", "title"], pf2=["body"], pf3=["title"])
    counts = {}
    for q, extra in (("zzz yyy xxx", {}), ("zzz yyy xxx", phases), ("pa pb pc", phases)):
        edismax(corpus.frame, q=q, qf=["body", "title"], **extra)           # warm: norm tables, buffers
        reset_stats(arrays)
        edismax(corpus.frame, q=q, qf=["body", "title"], **extra)
        counts[(q, bool(extra))] = phrase_launches(arrays)
    assert counts[("zzz yyy xxx", True)] == counts[("zzz yyy xxx", False)], counts
    assert counts[("zzz yyy xxx", True)]["phrase"] == 0 and counts[("pa pb pc", True)]["phrase"] > 0, counts
    check(corpus, "unknown only", matches=False, q="zzz yyy", qf=["body", "title"], **phases)


# ------------------------------------------------------------------ field-centric combine
FIELD_CENTRIC = {
    "two_fields_mm": dict(q="c0 pa pb", qf=["body", "tag"], mm="2"),
    "mm_clamped_per_field": dict(q="c0 c1 pa", qf=["body", "title", "tag"], mm=3),
    "boosts_tie": dict(q="c1 t3 zzz r1", qf=["body^1.5", "title", "tag^0.5"], mm="75%", tie=0.3),
    "tie_one": dict(q="pa pb pc", qf=["body", "tag^2"], tie=1.0),
    "negative_mm": dict(q="c0 c1 c2 t0", qf=["title^0.5", "tag"], mm="-1", tie=0.7),
    "eight_fields": dict(q="c0 c2 t3", qf=["body", "title", "tag", "f3", "f4", "f5", "f6^3", "f7"], tie=0.2),
}


@pytest.mark.parametrize("name", list(FIELD_CENTRIC))
def test_field_centric_combine(corpus, name):
    """edismax_combine_fields_kernel: float32 per-field sums, the per-field mm clamp, boosts and tie."""
    from searcharray_b200.solr import _Plan, default_bm25
    kw = FIELD_CENTRIC[name]
    plan = _Plan(corpus.frame, kw["q"], kw["qf"], kw.get("mm"), None, None, None, kw.get("tie", 0.0), "OR",
                 default_bm25)
    assert not plan.term_centric and plan.device_ok()
    want = check(corpus, name, **kw)
    assert want.dtype == np.float32


# ------------------------------------------------------------------ phases
LONG_Q = "c0 c1 pa pb pc ss ss r1 t0 t0b t3 t3b c2 zzz pa pb"       # SA_MAX_PHRASE_TERMS tokens
PHASES = {
    "pf_one_field": dict(q="pa pb pc", qf=["body"], pf=["body"]),
    "pf2_across_fields": dict(q="pa pb pc c0", qf=["body", "title"], pf2=["body", "title^2"], tie=0.3),
    "pf2_repeat_last": dict(q="pa pb", qf=["body", "title"], pf2=["title^0.5"]),
    "pf3_across_fields": dict(q="pa pb pc", qf=["body", "title"], pf3=["body^0.5", "title"]),
    "all_phases": dict(q="pa pb pc c1", qf=["body^2", "title"], pf=["title"], pf2=["body"], pf3=["body", "title^3"],
                       mm="50%", tie=0.3),
    "common_terms": dict(q="c0 c1 c2", qf=["body", "title"], pf=["body", "title"], pf2=["body", "title"],
                         pf3=["body"]),
    "tile_confined": dict(q="t0 t0b t3 t3b", qf=["body", "title"], pf=["body"], pf2=["body", "title"],
                          pf3=["title"]),
    "same_term": dict(q="ss ss r1", qf=["body", "title"], pf=["body"], pf2=["body", "title"]),
    "missing_filtered_list": dict(q="lone c0 c1", qf=["body", "title"], mm=2, pf=["body"], pf2=["body", "title"],
                                  pf3=["title"]),
    "unknown_in_phrase": dict(q="pa zzz pb", qf=["body"], pf=["body"], pf2=["body"], pf3=["body"]),
    "field_centric": dict(q="pa pb pc", qf=["body", "tag"], pf=["body", "tag"], pf2=["tag", "body"], pf3=["body"],
                          tie=0.3),
    "sixteen_tokens": dict(q=LONG_Q, qf=["body", "title"], mm="50%", pf=["body", "title"], pf2=["body", "title"],
                           pf3=["body", "title^0.5"]),
}


@pytest.mark.parametrize("name", list(PHASES))
def test_phrase_phases(corpus, name):
    """pf / pf2 / pf3 on one field and across fields on the lists filtered to qf > 0: sa_multi_filter,
    sa_multi_phrases (one launch per field, every regime and the missing branch) and sa_multi_add_phase."""
    check(corpus, name, **PHASES[name])


def test_missing_filtered_list_is_empty(corpus):
    """`lone` docs hold one query term: under mm = 2 none of them matches, so lone's filtered list is empty."""
    want = corpus.oracle(**PHASES["missing_filtered_list"])
    assert np.all(want[LONE] == 0) and np.count_nonzero(want) > 0
    assert len(LONE) > 0 and corpus.frame["body"].array.docfreq("lone") == len(LONE)


def test_similarity_per_field(corpus):
    """Different sparse-safe k1 / b per field in qf and the phrase phases."""
    from searcharray_b200 import bm25_similarity
    sims = {"body": bm25_similarity(k1=1.2, b=0.75), "title": bm25_similarity(k1=0.6, b=0.3),
            "f3": bm25_similarity(k1=2.0, b=0.9)}
    check(corpus, "sims term-centric", sims=sims, q="pa pb c0", qf=["body", "title", "f3"], pf2=["body", "title", "f3"],
          pf=["f3"], tie=0.3)
    check(corpus, "sims field-centric", sims=dict(sims, tag=bm25_similarity(k1=0.9, b=0.1)), q="pa pb pc",
          qf=["body", "title", "tag"], pf=["tag"], pf3=["title"], mm="2")


def test_zero_average_doc_length(corpus):
    """A field with avgdl 0 scores 0 everywhere (reference similarity.py:31-32), in qf and in pf."""
    of = corpus.ofields["zero"]
    for toks in (["c0"], ["pa", "pb"]):
        assert not np.any(of.score(toks)), toks
    check(corpus, "zero term-centric", q="pa pb c0", qf=["body", "zero"], pf=["body", "zero"], pf2=["zero"], tie=0.5)
    check(corpus, "zero field-centric", q="pa pb c0", qf=["zero", "tag"], pf=["zero", "tag"])
    check(corpus, "zero alone", matches=False, q="pa pb", qf=["zero"], pf=["zero"])


# ------------------------------------------------------------------ two names of one index
@pytest.fixture(scope="module")
def shared(corpus):
    frame = pd.DataFrame({f: corpus.frame[f].array for f in ("body", "title", "tag")})
    frame["body2"] = frame["body"]
    assert frame["body2"].array._shared is frame["body"].array._shared      # one sa_index
    assert all(frame[f].array.rows is None for f in frame.columns)          # whole columns: the device path
    ofields = dict(corpus.ofields, body2=corpus.ofields["body"])
    return frame, ofields


def test_shared_index_similarities(corpus, shared):
    """Two column names of one device index under different similarities: each name's rows keep its own
    parameters until the combine and the phase sums read them."""
    from searcharray_b200 import bm25_similarity
    frame, ofields = shared
    sims = {"body": bm25_similarity(k1=1.2, b=0.75), "body2": bm25_similarity(k1=0.6, b=0.3)}
    kw = dict(frame=frame, ofields=ofields, sims=sims)
    check(corpus, "shared qf", q="c0 pa pb", qf=["body", "body2"], tie=0.3, **kw)
    check(corpus, "shared qf pf", q="c0 pa pb", qf=["body", "body2^2"], pf=["body"], pf2=["body2"], tie=0.3, **kw)
    check(corpus, "shared field-centric", q="c0 pa pb", qf=["body", "body2", "tag"], pf2=["body2", "body"], **kw)


def test_shared_index_phrase_rows(corpus, shared):
    """pf on one name and pf2 / pf3 on the other, in both call orders, under one similarity: every phase entry reads
    its own name's phrase rows."""
    frame, ofields = shared
    kw = dict(frame=frame, ofields=ofields)
    check(corpus, "pf body pf2 body2", q="pa pb pc", qf=["body", "body2"], pf=["body"], pf2=["body2"], **kw)
    check(corpus, "pf body2 pf2 body", q="pa pb pc", qf=["body", "body2"], pf=["body2"], pf2=["body"], **kw)
    check(corpus, "pf3 body pf body2", q="pa pb pc c0", qf=["body", "body2"], pf3=["body"], pf=["body2"], **kw)
    check(corpus, "all on both", q="c0 c1 c2", qf=["body2", "title", "body"], pf=["body", "body2"],
          pf2=["body2", "title"], pf3=["body", "body2"], tie=0.3, **kw)


# ------------------------------------------------------------------ the most the device path admits
def test_eight_fields_pf2_nine_tokens(corpus):
    """pf2 on 8 fields of 9 tokens: one sa_multi_add_phase of 72 entries."""
    q = "c0 c1 pa pb pc c2 r1 ss t3"
    check(corpus, "8 x 9 pf2", q=q, qf=WS8, pf2=WS8, mm="50%", tie=0.3)


def test_eight_fields_sixteen_tokens_every_phase(corpus):
    """8 fields x 16 tokens with pf, pf2 and pf3 on every field: 30 phrase rows per field, 128 pf2 entries."""
    from searcharray_b200.solr import _Plan, default_bm25
    qf = [f + "^0.5" if i % 3 == 0 else f for i, f in enumerate(WS8)]
    plan = _Plan(corpus.frame, LONG_Q, qf, None, qf, qf, qf, 0.3, "OR", default_bm25)
    assert plan.device_ok() and [len(e) for _, e in plan.phase_entries()] == [8, 128, 112]
    check(corpus, "8 x 16 pf pf2 pf3", ks=(10, 17), q=LONG_Q, qf=qf, pf=qf, pf2=qf, pf3=qf, mm="25%", tie=0.3)


# ------------------------------------------------------------------ state other calls leave behind
def test_after_row_filters_and_batched_topk(corpus):
    """A sliced score installs a row filter on body's index; search_topk and fields_topk run on the same indexes
    between edismax and edismax_topk.  None of it may leak into the device edismax."""
    from searcharray_b200 import Field, Or, fields_topk
    from searcharray_b200.solr import edismax, edismax_topk
    frame = corpus.frame
    kw = dict(q="pa pb c0", qf=["body", "title^2"], pf=["body"], pf2=["body", "title"], tie=0.3)
    want = corpus.oracle(**kw)
    mask = np.arange(N_DOCS) % 3 == 1
    frame["body"].array[mask].score("c0")
    got, _ = edismax(frame, **kw)
    assert_vec(got, want, "after a sliced score")
    for k in KS:
        frame["title"].array[mask].score(["pa", "pb"])
        frame["body"].array.search_topk(["c1", ["pa", "pb"]], k=k)
        fields_topk(frame, [Or([Field("body", "c0"), Field("title", "pa")])], k=k)
        d, s = edismax_topk(frame, k=k, **kw)
        assert_topk(d, s, want, k, "after search_topk / fields_topk")
        got, _ = edismax(frame, **kw)
        assert_vec(got, want, f"interleaved k={k}")


# ------------------------------------------------------------------ composed path (views)
@pytest.mark.parametrize("kw", [
    dict(q="pa pb c0", qf=["body", "title^2"], pf=["body"], pf2=["body", "title"], pf3=["title"], tie=0.3, mm=2),
    dict(q="pa pb pc", qf=["body", "tag"], pf=["body", "tag"], pf2=["body"], tie=0.3),
], ids=["term_centric", "field_centric"])
def test_sliced_frame_composed(corpus, kw):
    """A view takes _run_composed (device_ok is False): GPU .score calls on the view, the reference's numpy
    combination.  Bit for bit against the oracle on the sliced indexes; edismax_topk refuses views."""
    from oracle import solr as osolr
    from searcharray_b200.solr import edismax, edismax_topk
    mask = (np.arange(N_DOCS) % 7 != 3) & (np.arange(N_DOCS) < 4 * TILE + 1000)
    frame = corpus.frame[mask]
    ofields = {f: osolr.OracleField(o.index.sliced(mask), o.term_to_id, tokenizer=o.tokenizer)
               for f, o in corpus.ofields.items()}
    want = corpus.oracle(ofields, **kw)
    assert np.count_nonzero(want) > 0
    got, _ = edismax(frame, **kw)
    assert_vec(got, want, "composed")
    with pytest.raises(NotImplementedError):
        edismax_topk(frame, k=10, **kw)


# ------------------------------------------------------------------ TMDB
TMDB_FIELDS = ["title_tokens^1.0", "overview_tokens^0.5"]
TMDB_KWARGS = {
    "qf_only": dict(qf=TMDB_FIELDS, tie=0.0),
    "pf_mm100": dict(qf=TMDB_FIELDS, pf=TMDB_FIELDS, mm="100%"),
    "pf2_pf3_and": dict(qf=TMDB_FIELDS, pf2=TMDB_FIELDS, pf3=TMDB_FIELDS, tie=1.0, q_op="AND"),
}


@pytest.fixture(scope="module")
def tmdb():
    from oracle import search as osearch
    from oracle import solr as osolr
    from searcharray_b200 import SearchArray
    z = np.load(os.path.join(GOLDEN, "tmdb_index.npz"))
    cols, ofields = {}, {}
    for name in ("title_tokens", "overview_tokens"):
        host = load_field(z, name)
        cols[name] = SearchArray.from_host_index(host)
        oidx = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                                   avg_doc_length=host.avg_doc_length)
        ofields[name] = osolr.OracleField(oidx, host.term_dict.term_to_ids)
    with open(os.path.join(GOLDEN, "tmdb.json")) as f:
        g = json.load(f)
    return pd.DataFrame(cols), ofields, g


@pytest.mark.parametrize("name", list(TMDB_KWARGS) + ["golden_kwargs"])
def test_tmdb(tmdb, name):
    """The 8 golden TMDB edismax queries (27,846 docs) under more kwargs sets, bit for bit against the oracle."""
    from oracle import solr as osolr
    from searcharray_b200.solr import edismax, edismax_topk
    frame, ofields, g = tmdb
    kw = g["edismax_kwargs"] if name == "golden_kwargs" else TMDB_KWARGS[name]
    assert len(g["edismax"]) == 8
    for r in g["edismax"]:
        want = osolr.edismax(ofields, q=r["q"], **kw)
        got, _ = edismax(frame, q=r["q"], **kw)
        assert_vec(got, want, (name, r["q"]))
        for k in (10, 17):
            d, s = edismax_topk(frame, r["q"], k=k, **kw)
            assert_topk(d, s, want, k, (name, r["q"]))
