"""GPU: the count row of one phrase or slop query (sa_phrase_row) through every entry point that writes it --
termfreqs and score (sa_phrase_freqs / sa_score_phrase; on a view termfreqs + ops.bm25_score) and the batched top-k
on views and under classic_similarity (sa_score_batch_topk_sim) -- on the index's own lists and on a view's filtered
lists, against the CPU oracle and against .score.  The corpus reaches each branch of the route: doc 0 holds every
phrase term in its first 18 positions, so the own lists sit in the span search's "literal" corner, and so do the
filtered lists of a view that keeps doc 0 but not those of one that drops it; one phrase has an unknown token, one a
term with no docs in the mask view, and one repeats a term (the same-term speculation)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

NO_DOC = 0xFFFFFFFF
N_DOCS = 20_000                   # three tiles of 8,192 docs
Z_DOCS = [3, 9_000, 17_000]       # the only docs with "z"; the mask view drops them
HEADER_MASK = np.uint64(0xFFFFFFFFFFFC0000)
PHRASES = [["a", "b"], ["b", "c", "d"], ["a", "a"], ["a", "nope"], ["a", "z"], ["c", "a", "b"]]
QUERIES = ["a", ["a", "b"], "c", ["b", "c", "d"], ["a", "a"], ["a", "nope"], "nope", ["a", "z"], ["c", "a", "b"]]


def view_keys():
    mask = np.random.default_rng(4).random(N_DOCS) < 0.4
    mask[0] = True
    mask[Z_DOCS] = False
    return {"unsliced": None, "mask_keeps_doc0": mask, "drops_doc0": slice(1, None)}


@pytest.fixture(scope="module")
def corpus():
    from oracle import search as osearch
    from searcharray_b200 import SearchArray
    rng = np.random.default_rng(17)
    vocab = ["a", "b", "c", "d"] + [f"f{i}" for i in range(8)]
    p = 1.0 / np.arange(1, len(vocab) + 1)
    p /= p.sum()
    docs = [" ".join(rng.choice(vocab, size=int(rng.integers(1, 60)), p=p)) for _ in range(N_DOCS)]
    docs[0] = "a b c d a a b f0 c a b"
    for d in Z_DOCS:
        docs[d] += " a z"
    arr = SearchArray.index(docs)
    host = arr.host
    tid = host.term_dict.term_to_ids
    for t in "abcd":                  # the own lists start at (doc 0, block 0)
        assert host.term_words(tid[t])[0] & HEADER_MASK == 0, t
    assert host.term_words(tid["z"])[0] & HEADER_MASK != 0
    oidx = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                               avg_doc_length=host.avg_doc_length)
    return arr, oidx, tid


def views_of(corpus, name):
    arr, oidx, _ = corpus
    key = view_keys()[name]
    return (arr, oidx) if key is None else (arr[key], oidx.sliced(key))


def ids_of(tid, q):
    ids = [tid.get(t) for t in ([q] if isinstance(q, str) else q)]
    return ids[0] if len(ids) == 1 else ids


@pytest.mark.parametrize("slop", [0, 2])
@pytest.mark.parametrize("name", list(view_keys()))
def test_termfreqs(corpus, name, slop):
    view, oview = views_of(corpus, name)
    tid = corpus[2]
    if name == "mask_keeps_doc0":
        assert oview.docfreq(tid["z"]) == 0
    for q in PHRASES:
        got = view.termfreqs(q, slop=slop)
        assert np.array_equal(got, oview.termfreqs(ids_of(tid, q), slop=slop)), (name, q, slop)
        if "nope" not in q and "z" not in q:
            assert got.max() > 0, (name, q, slop)


@pytest.mark.parametrize("k1,b", [(1.2, 0.75), (1.2, 1.5)])
@pytest.mark.parametrize("slop", [0, 2])
@pytest.mark.parametrize("name", list(view_keys()))
def test_score(corpus, name, slop, k1, b):
    from searcharray_b200 import bm25_similarity
    view, oview = views_of(corpus, name)
    tid = corpus[2]
    for q in PHRASES:
        got = view.score(q, similarity=bm25_similarity(k1=k1, b=b), slop=slop)
        want = oview.score(ids_of(tid, q), k1=k1, b=b, slop=slop)
        what = (name, q, slop, k1, b)
        assert np.array_equal(got > 0, want > 0), what
        assert np.array_equal(np.isnan(got), np.isnan(want)), what
        np.testing.assert_allclose(got, want, rtol=1e-5, atol=0, err_msg=str(what))


def expected_topk(dense, k):
    """The top k of a .score vector, in its own dtype: ids by (score desc, id asc) over the scores > 0."""
    dense = np.asarray(dense)
    nz = np.flatnonzero(dense > 0)
    order = nz[np.lexsort((nz, -dense[nz].astype(np.float64)))][:k]
    docs = np.full(k, NO_DOC, dtype=np.uint32)
    scores = np.zeros(k, dtype=dense.dtype)
    docs[:len(order)] = order
    scores[:len(order)] = dense[order]
    return docs, scores


def bits(a):
    return a.view(np.uint64 if a.dtype == np.float64 else np.uint32)


# BM25 on an unsliced array takes the fused batch path, which writes no count rows
@pytest.mark.parametrize("slop", [0, 2])
@pytest.mark.parametrize("name,sim_name", [(n, s) for n in view_keys() for s in ("bm25", "classic")
                                           if (n, s) != ("unsliced", "bm25")])
def test_search_topk(corpus, name, slop, sim_name):
    from searcharray_b200 import bm25_similarity, classic_similarity
    view, _ = views_of(corpus, name)
    sim = bm25_similarity() if sim_name == "bm25" else classic_similarity()
    dense = [view.score(q, similarity=sim, slop=slop) for q in QUERIES]
    for k in (1, 10):
        docs, scores = view.search_topk(QUERIES, k=k, similarity=sim, slop=slop)
        for i, q in enumerate(QUERIES):
            wd, ws = expected_topk(dense[i], k)
            what = (name, sim_name, q, slop, k)
            assert scores.dtype == ws.dtype, what
            assert np.array_equal(docs[i], wd), what
            assert np.array_equal(bits(scores[i]), bits(ws)), what
