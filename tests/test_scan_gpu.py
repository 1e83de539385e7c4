"""GPU: the exclusive scans of sa_scan.cuh at sizes where the one-CTA scans run more than one round and carry a sum
from one round to the next.  That carry is reached only beyond 1,024 scan blocks: set ops on more than
2^20 + 1,024 elements, device builds of more than 2^20 tokens, an index of more than 2^20 posting words (the tf
table's block counts), and a filtered list of more than 256 x 2,048 words (the filter's chunk counts)."""
import numpy as np
import pytest

from test_build_gpu import same_index

pytestmark = pytest.mark.gpu

BIG = (1 << 20) + 1024
SIZES = [0, 1, 1023, 1024, 1025, BIG + 1, 2 * BIG + 777]


def eq(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a, b), (a[:8], b[:8])


def sorted_words(rng, n):
    """n sorted words with runs of equal high parts (so heads are neither all nor none of the elements)."""
    hi = np.cumsum(rng.integers(0, 2, n, dtype=np.uint64))
    lo = rng.integers(0, 1 << 18, n, dtype=np.uint64)
    return np.sort((hi << np.uint64(36)) | (lo << np.uint64(18)) | rng.integers(0, 1 << 18, n, dtype=np.uint64))


@pytest.mark.parametrize("n", SIZES)
def test_compacting_ops_across_scan_rounds(n):
    from searcharray_b200 import ops
    rng = np.random.default_rng(n)
    a = sorted_words(rng, n)
    eq(ops.unique(a, 36), np.unique(a >> np.uint64(36)))
    eq(ops.unique(a), np.unique(a))

    msb = np.uint64(0x0000000FFFFC0000)
    lo, hi = (1 << 18) * 1000, (1 << 18) * 150000
    v = a & msb
    eq(ops.payload_slice(a, int(msb), lo, hi), a[(v >= np.uint64(lo)) & (v <= np.uint64(hi))])

    ids = a >> np.uint64(36)
    counts = rng.integers(0, 40, n, dtype=np.uint64)
    got_ids, got_sums = ops.key_sum_over(ids, counts)
    want_ids, first = np.unique(ids, return_index=True)
    want_sums = np.add.reduceat(counts, first).astype(np.float32) if n else np.zeros(0, np.float32)
    eq(got_ids, want_ids)
    eq(got_sums, want_sums)


def test_device_build_beyond_1024_scan_blocks():
    from searcharray_b200.indexing import build_index
    rng = np.random.default_rng(11)
    vocab = np.array([f"w{i}" for i in range(3000)])
    lens = rng.integers(40, 90, 18_000)
    toks = vocab[np.minimum(rng.zipf(1.3, int(lens.sum())) - 1, len(vocab) - 1)]
    cuts = np.cumsum(lens)[:-1]
    docs = [" ".join(d) for d in np.split(toks, cuts)]
    assert lens.sum() > (1 << 20) + 1024
    same_index(build_index(docs, str.split, gpu_build=0), build_index(docs, str.split))


@pytest.fixture(scope="module")
def long_lists():
    """Two terms of 600,000 words each (1.2M words in the index) and a short one.  "a" has one word per doc; "b" has
    two words (blocks 0 and 2) in every other doc."""
    from searcharray_b200 import SearchArray
    from searcharray_b200.indexing import index_from_term_postings
    rng = np.random.default_rng(5)
    n_docs = 600_000
    bits = lambda k: rng.integers(1, 1 << 18, k, dtype=np.uint64)
    docs_a = np.arange(n_docs, dtype=np.uint64)
    words_a = (docs_a << np.uint64(36)) | bits(n_docs)
    docs_b = np.repeat(np.arange(0, n_docs, 2, dtype=np.uint64), 2)
    blk_b = np.tile(np.array([0, 2], dtype=np.uint64), n_docs // 2)
    words_b = (docs_b << np.uint64(36)) | (blk_b << np.uint64(18)) | bits(len(docs_b))
    words_c = (np.arange(0, n_docs, 997, dtype=np.uint64) << np.uint64(36)) | np.uint64(1)
    host = index_from_term_postings(["a", "b", "c"], [words_a, words_b, words_c],
                                    rng.integers(1, 50, n_docs).astype(np.float32))
    assert len(host.words) > (1 << 20) + 1024 and len(words_a) > 256 * 2048
    return host, SearchArray.from_host_index(host)


def host_tf(host, t):
    w = host.term_words(t)
    tf = np.bincount((w >> np.uint64(36)).astype(np.int64), weights=np.bitwise_count(w & np.uint64(0x3FFFF)),
                     minlength=host.n_docs)
    return tf.astype(np.float32)


def test_upload_tf_table_and_df_of_long_lists(long_lists):
    host, arr = long_lists
    for t, name in enumerate(["a", "b", "c"]):
        eq(arr.termfreqs(name), host_tf(host, t))
        assert int(arr.docfreq(name)) == len(np.unique(host.term_words(t) >> np.uint64(36))), name


def test_view_filter_of_long_lists(long_lists):
    host, arr = long_lists
    mask = np.random.default_rng(6).random(host.n_docs) < 0.4
    view = arr[mask]
    rows = np.flatnonzero(mask)
    for t, name in enumerate(["a", "b", "c"]):
        eq(view.termfreqs(name), arr.termfreqs(name)[rows])
        docs = np.unique(host.term_words(t) >> np.uint64(36)).astype(np.int64)
        assert int(view.docfreq(name)) == int(mask[docs].sum()), name
