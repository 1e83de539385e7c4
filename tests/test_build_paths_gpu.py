"""The device index build (sa_build.cu: sa_op_build_index, SearchArray.index(..., gpu_build=True)) against the CPU
oracle: every term's slice equals oracle.search.encode of that term's (doc, posn) pairs, and doc_lens /
avg_doc_length equal the host build's.  Covers the radix sort's end_bit (vocabularies around powers of two up to
2^17 + 1), terms absent from the triples, repeated triples, a doc of MAX_POSN tokens, empty docs, truncation, scoring
on the built array, and the entry point's refusals of triples that do not fit a posting word."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MAX_POSN = (1 << 18) - 1


def build_c(terms, docs, posns, n_terms, n_triples=None):
    """sa_op_build_index through ctypes -> (words, term offsets, term lengths)"""
    from searcharray_b200 import _lib
    t = np.ascontiguousarray(terms, dtype=np.uint32)
    d = np.ascontiguousarray(docs, dtype=np.uint32)
    p = np.ascontiguousarray(posns, dtype=np.uint32)
    n = len(t) if n_triples is None else n_triples
    words = np.zeros(max(len(t), 1), dtype=np.uint64)
    offs = np.full(max(n_terms, 1), 7, dtype=np.uint64)
    lens = np.full(max(n_terms, 1), 7, dtype=np.uint64)
    n_words = ctypes.c_uint64(0)
    _lib.check(_lib.lib().sa_op_build_index(_lib.p_u32(t), _lib.p_u32(d), _lib.p_u32(p), n, n_terms, 0,
                                            _lib.p_u64(words), ctypes.byref(n_words), _lib.p_u64(offs), _lib.p_u64(lens)))
    return words[:n_words.value], offs[:n_terms], lens[:n_terms]


def check_slices(words, offs, lens, terms, docs, posns, n_terms):
    """every term's slice against oracle.search.encode of its (doc, posn) pairs in document order; absent terms
    have offset 0 and length 0; the slices tile `words` in term-id order"""
    from oracle import search as osearch
    terms = np.asarray(terms, dtype=np.int64)
    order = np.argsort(terms, kind="stable")
    bounds = np.searchsorted(terms[order], np.arange(n_terms + 1))
    docs, posns = np.asarray(docs)[order], np.asarray(posns)[order]
    at = 0
    for t in range(n_terms):
        a, b = bounds[t], bounds[t + 1]
        if a == b:
            assert offs[t] == 0 and lens[t] == 0, (t, offs[t], lens[t])
            continue
        want = osearch.encode(docs[a:b], posns[a:b])
        assert offs[t] == at and lens[t] == len(want), (t, offs[t], lens[t], at, len(want))
        got = words[at:at + len(want)]
        assert np.array_equal(got, want), (t, np.flatnonzero(got != want)[:4])
        at += len(want)
    assert at == len(words)


def random_triples(rng, n_terms, n_docs, per_doc):
    """triples in document order (docs ascending, positions ascending within a doc); every term id occurs"""
    lens = rng.integers(0, 2 * per_doc, size=n_docs)
    docs = np.repeat(np.arange(n_docs), lens)
    posns = np.concatenate([np.arange(k) for k in lens]) if len(lens) else np.zeros(0, dtype=np.int64)
    terms = rng.integers(0, n_terms, size=len(docs))
    terms[rng.permutation(len(terms))[:n_terms]] = np.arange(n_terms)   # every id at least once
    return terms, docs, posns


@pytest.mark.parametrize("n_terms", [1, 2, 3, 4, 5, 16, 17, 256, 257, 4096, 4097, 1 << 16, (1 << 16) + 1,
                                     1 << 17, (1 << 17) + 1])
def test_vocabulary_sizes(n_terms):
    """the sort key is end_bit = ceil(log2(n_terms)) bits wide: the largest ids need its top bit"""
    rng = np.random.default_rng(n_terms)
    n_docs = max(50, 3 * n_terms // 40)
    terms, docs, posns = random_triples(rng, n_terms, n_docs, 40)
    assert len(terms) >= n_terms and terms.max() == n_terms - 1
    check_slices(*build_c(terms, docs, posns, n_terms), terms, docs, posns, n_terms)


def test_absent_terms_and_repeated_triples():
    rng = np.random.default_rng(5)
    terms, docs, posns = random_triples(rng, 300, 400, 30)
    terms = terms % 300
    used = terms * 2 + 1                                           # every even id and everything >= 601 is absent
    n_terms = 1000
    # repeat a third of the triples in place: the same (term, doc, posn) twice ORs the same bit
    rep = np.sort(np.concatenate([np.arange(len(used)), rng.choice(len(used), size=len(used) // 3, replace=False)]))
    t, d, p = used[rep], docs[rep], posns[rep]
    words, offs, lens = build_c(t, d, p, n_terms)
    check_slices(words, offs, lens, t, d, p, n_terms)
    assert (lens[0::2] == 0).all() and (lens[601:] == 0).all() and (lens[1:600:2] > 0).all()
    # the repeats change nothing
    w1, o1, l1 = build_c(used, docs, posns, n_terms)
    assert np.array_equal(words, w1) and np.array_equal(offs, o1) and np.array_equal(lens, l1)


def test_same_block_in_neighbouring_docs():
    """consecutive triples of one term in two docs at the same block must start two words"""
    terms = np.zeros(6, dtype=np.int64)
    docs = np.array([0, 1, 2, 2, 3, 5])
    posns = np.array([0, 0, 3, 4, 0, 17])
    check_slices(*build_c(terms, docs, posns, 1), terms, docs, posns, 1)


def same_as_host(docs, **kw):
    from searcharray_b200.indexing import build_index
    dev = build_index(docs, str.split, gpu_build=0, **kw)
    host = build_index(docs, str.split, **kw)
    assert dev.n_terms == host.n_terms and np.array_equal(dev.term_lengths, host.term_lengths)
    assert np.array_equal(dev.term_offsets, host.term_offsets) and np.array_equal(dev.words, host.words)
    assert dev.doc_lens.dtype == host.doc_lens.dtype and np.array_equal(dev.doc_lens, host.doc_lens)
    assert dev.avg_doc_length == host.avg_doc_length
    return dev


def test_max_posn_doc_and_empty_docs():
    """a doc of MAX_POSN tokens of one term between empty docs, first, inside and last"""
    from oracle import search as osearch
    long_doc = " ".join(["a"] * MAX_POSN)
    docs = ["", "b a c", "", long_doc, "", "", "c c a", ""]
    dev = same_as_host(docs)
    a = dev.term_dict.term_to_ids["a"]
    want = osearch.encode(np.concatenate([[1], np.full(MAX_POSN, 3), [6]]),
                          np.concatenate([[1], np.arange(MAX_POSN), [2]]))
    assert np.array_equal(dev.term_words(a), want)
    assert dev.doc_lens[3] == MAX_POSN and (dev.doc_lens[[0, 2, 4, 5, 7]] == 0).all()
    # the device index counts every one of those positions
    from searcharray_b200 import SearchArray
    arr = SearchArray.from_host_index(dev)
    tf = arr.termfreqs("a")
    assert np.array_equal(tf, osearch.termfreqs_dense(want, len(docs))) and tf[3] == MAX_POSN


def test_truncate():
    from searcharray_b200.indexing import build_index
    docs = ["x y", " ".join(["y"] * (MAX_POSN + 7)), "", "x"]
    with pytest.raises(ValueError):
        build_index(docs, str.split, gpu_build=0)
    dev = same_as_host(docs, truncate=True)
    assert dev.doc_lens[1] == MAX_POSN


def test_score_and_search_topk_on_the_built_array():
    from searcharray_b200 import SearchArray
    rng = np.random.default_rng(9)
    vocab = [f"t{i}" for i in range(300)]
    p = 1.0 / np.arange(1, 301)
    p /= p.sum()
    docs = [" ".join(rng.choice(vocab, size=int(rng.integers(0, 200)), p=p)) for _ in range(20_000)]
    dev = SearchArray.index(docs, gpu_build=True)
    host = SearchArray.index(docs)
    for q in ("t0", "t7", "t299", ["t0", "t1"], ["t3", "t3"]):
        s1, s2 = dev.score(q), host.score(q)
        assert np.array_equal(s1.view(np.uint32), s2.view(np.uint32)), q
    qs = ["t0", "t5", "t100", "t299"]
    d1, sc1 = dev.search_topk(qs, k=10)
    d2, sc2 = host.search_topk(qs, k=10)
    assert np.array_equal(d1, d2) and np.array_equal(np.asarray(sc1), np.asarray(sc2))


# ---------------------------------------------------------------- refusals
def test_build_index_refuses_triples_that_do_not_fit():
    from searcharray_b200._lib import SearchArrayB200Error
    ok_t, ok_d, ok_p = np.array([0, 1, 0]), np.array([0, 0, 1]), np.array([0, 1, 0])
    build_c(ok_t, ok_d, ok_p, 2)
    cases = [("n_terms", (np.array([0, 2, 0]), ok_d, ok_p, 2)),
             ("28-bit", (ok_t, np.array([0, 0, 1 << 28]), ok_p, 2)),
             ("exceeds", (ok_t, ok_d, np.array([0, 18 << 18, 0]), 2)),
             ("n_terms", (ok_t, ok_d, ok_p, 0))]
    for words, (t, d, p, n_terms) in cases:
        with pytest.raises(SearchArrayB200Error, match=words):
            build_c(t, d, p, n_terms)
    # the largest position and doc id that fit are accepted
    t, d, p = np.array([0, 0, 1]), np.array([5, (1 << 28) - 1, (1 << 28) - 1]), np.array([(18 << 18) - 1, 0, 3])
    check_slices(*build_c(t, d, p, 2), t, d, p, 2)
    # cub counts in an int: 2^31 triples are refused before any array is read
    with pytest.raises(SearchArrayB200Error, match="too many tokens"):
        build_c(ok_t, ok_d, ok_p, 2, n_triples=1 << 31)


def test_index_refuses_words_past_max_posn():
    """posting words injected through from_host_index with a block past MAX_POSN // 18 = 14,563: the first device
    call raises; block 14,563 itself is accepted and counted exactly"""
    from oracle import search as osearch
    from searcharray_b200 import SearchArray
    from searcharray_b200._lib import SearchArrayB200Error
    from searcharray_b200.indexing import index_from_term_postings
    n_docs = 3000
    rng = np.random.default_rng(13)
    ok = np.sort(rng.choice(n_docs, size=2000, replace=False)).astype(np.uint64)
    w_ok = (ok << np.uint64(36)) | (np.uint64(14_563) << np.uint64(18)) | np.uint64(0x3FFFF)
    for last_block in (14_564, (1 << 18) - 1):
        bad = w_ok.copy()
        bad[-1] = (bad[-1] & ~np.uint64(0xFFFFFFFFF)) | (np.uint64(last_block) << np.uint64(18)) | np.uint64(1)
        host = index_from_term_postings(["a", "b"], [w_ok, bad], np.full(n_docs, 10, dtype=np.float32))
        arr = SearchArray.from_host_index(host)
        with pytest.raises(SearchArrayB200Error, match="MAX_POSN"):
            arr.termfreqs("a")
    host = index_from_term_postings(["a"], [w_ok], np.full(n_docs, 10, dtype=np.float32))
    arr = SearchArray.from_host_index(host)
    assert np.array_equal(arr.termfreqs("a"), osearch.termfreqs_dense(w_ok, n_docs))
