"""GPU: every branch of the BM25 term scan (term_tile_kernel, sa_term.cu) and of the top-k collector it ends with,
against the CPU oracle.  termfreqs must match bit for bit, BM25 scores bit for bit (exotic parameters: the 1e-5
contract with the same NaN mask), and search_topk must return the ids of the top k by (score desc, id asc) over
the scores > 0 with the oracle's score bits, empty slots NO_DOC / 0.

Which branch a CTA takes depends on how many records or words its tile holds and on the tuning knobs that
launch_term_batch reads on every launch (SA_STAGED_NORM_MIN_RECS / _WORDS, SA_TERM_QUAD_MIN_RECS,
SA_TERM_PREFETCH_TILES).  The corpora below place those counts in tiles on purpose; the knob settings force each
branch on or off for all of them.  SA_NO_TF_TABLE and SA_TERM_QUERY_MAJOR are read once per process, so the same
checks run again in a child process (tests/_term_paths_worker.py)."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TILE = 8192
NO_DOC = 0xFFFFFFFF
REL_TOL = 1e-5
KNOB_VARS = ("SA_STAGED_NORM_MIN_RECS", "SA_STAGED_NORM_MIN_WORDS", "SA_TERM_QUAD_MIN_RECS", "SA_TERM_PREFETCH_TILES")
# "always": staged norms on every non-empty tile and four records per thread wherever >= 16 * k records exist;
# "never": gathered norms and one record per thread everywhere
KNOBS = {
    "default": {},
    "always": {"SA_STAGED_NORM_MIN_RECS": "1", "SA_STAGED_NORM_MIN_WORDS": "1", "SA_TERM_QUAD_MIN_RECS": "1"},
    "never": {"SA_STAGED_NORM_MIN_RECS": str(2 ** 31), "SA_STAGED_NORM_MIN_WORDS": str(2 ** 31),
              "SA_TERM_QUAD_MIN_RECS": str(2 ** 31)},
    "prefetch0": {"SA_TERM_PREFETCH_TILES": "0"},
    "prefetch1": {"SA_TERM_PREFETCH_TILES": "1"},
}
TOPK_KS = (1, 2, 10, 11, 16, 17, 32)
EXOTIC = ((0.0, 0.75), (1.2, 1.0), (1.2, 1.5))       # (k1, b): every one takes the ALL_DOCS kernel
MIXED_RUNS = (1, 2, 3, 4, 40)


def set_knobs(monkeypatch, setting):
    """Clears every knob, then sets the ones of `setting`."""
    for var in KNOB_VARS:
        monkeypatch.delenv(var, raising=False)
    for var, val in KNOBS[setting].items():
        monkeypatch.setenv(var, val)


# ------------------------------------------------------------------------------------------ comparisons
def assert_bits(got, want, what):
    got, want = np.asarray(got, dtype=np.float32), np.asarray(want, dtype=np.float32)
    assert got.shape == want.shape, what
    bad = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, f"{what}: {bad.size} docs differ, first {bad[:5]}: got {got[bad[:5]]}, want {want[bad[:5]]}"


def assert_contract(got, want, what):
    """Exotic parameters: same NaN mask, bits or 1e-5 relative elsewhere."""
    got, want = np.asarray(got), np.asarray(want)
    assert np.array_equal(np.isnan(got), np.isnan(want)), f"{what}: NaN mask differs"
    ok = ~np.isnan(want)
    if np.array_equal(got[ok].view(np.uint32), want[ok].view(np.uint32)):
        return
    assert np.array_equal(got[ok] > 0, want[ok] > 0), f"{what}: match mask differs"
    np.testing.assert_allclose(got[ok], want[ok], rtol=REL_TOL, atol=0, err_msg=what)


def expected_topk(dense, k, doc_base=0):
    dense = np.asarray(dense, dtype=np.float32)
    nz = np.flatnonzero(dense > 0)
    order = nz[np.lexsort((nz, -dense[nz].astype(np.float64)))][:k]
    docs = np.full(k, NO_DOC, dtype=np.uint32)
    scores = np.zeros(k, dtype=np.float32)
    docs[:len(order)] = order + doc_base
    scores[:len(order)] = dense[order]
    return docs, scores


def assert_topk(docs, scores, dense, k, what, doc_base=0):
    wd, ws = expected_topk(dense, k, doc_base)
    assert np.array_equal(np.asarray(docs, dtype=np.uint32), wd), f"{what}: ids {docs} want {wd}"
    assert np.array_equal(np.asarray(scores, dtype=np.float32).view(np.uint32), ws.view(np.uint32)), \
        f"{what}: score bits {scores} want {ws}"


def oracle_bm25(tfs, doc_lens, avgdl, idf, k1=1.2, b=0.75):
    from oracle import ops
    s = np.array(tfs, dtype=np.float32, copy=True)
    ops.bm25_score(s, np.asarray(doc_lens, dtype=np.float32), avgdl, idf, k1, b)
    return s


# ----------------------------------------------------------------------------------------- corpora
def encode_term(docs, runs, doc_base=0):
    """A doc with a run of r words holds the term at positions 0, 18, ..., 18 (r - 1): one word per position."""
    from searcharray_b200.roaringish import encode_postings
    docs = np.asarray(docs, dtype=np.int64)
    runs = np.asarray(runs, dtype=np.int64)
    d = np.repeat(docs + doc_base, runs)
    p = np.concatenate([18 * np.arange(r) for r in runs]) if len(runs) else np.zeros(0, dtype=np.int64)
    return encode_postings(d, p)


def tile_docs(rng, n_docs, tile, count):
    """`count` sorted docs of `tile`; with two or more, the first and the last doc of the tile are among them."""
    lo = tile * TILE
    size = min(TILE, n_docs - lo)
    if count == size:
        return lo + np.arange(size)
    if count < 2:
        return lo + np.sort(rng.choice(size, count, replace=False))
    inner = rng.choice(np.arange(1, size - 1), count - 2, replace=False)
    return lo + np.sort(np.concatenate([[0, size - 1], inner]))


def lane_runs(n_words):
    """Runs whose heads sit at lanes 28 and 29 of the 30-word windows the words path reads (windows start at the
    tile's first word): single-word docs up to the lane, then a run of 4, 3, 2, 40, 1, ... words."""
    targets = [(28, 4), (29, 3), (28, 2), (29, 40), (28, 1), (29, 2), (28, 3), (29, 4), (28, 40), (29, 1)]
    runs, off, i = [], 0, 0
    while off < n_words:
        lane, r = targets[i % len(targets)]
        while off % 30 != lane:
            runs.append(1)
            off += 1
        runs.append(r)
        off += r
        i += 1
    return runs


def mixed_corpus():
    """4 * 8192 + 517 docs (five tiles, a short last one), doc lengths 0..299 with some zeros, and terms whose
    tiles hold the record / word counts where the kernel's branches switch:
      0, 1, k-1 / k / k+1 for k = 10 and 32, 47 / 48 / 49 (staged norms), 159 / 161 (16 k +- 1 for k = 10),
      511 / 512 / 513 (four records per thread; 16 k +- 1 for k = 32), every doc of a full and of the short tile,
      and >= 1,024 words (staged norms on the words path).
    "_1" terms have one word per doc (words = records); "_r" terms runs of 1, 2, 3, 4 and 40 words.  Terms of fewer
    than 1,024 words have no tile directory and no tf table: their tiles are found by binary search.  `lanes` (tf
    table) and `lanes_s` (binary search) start runs at lanes 28 and 29 of a window, in 4-window and in 1-window
    passes.  `edge` holds only the first and the last doc of every tile."""
    from searcharray_b200.indexing import index_from_term_postings
    rng = np.random.default_rng(2018)
    n = 4 * TILE + 517
    doc_lens = rng.integers(0, 300, n).astype(np.float32)
    doc_lens[::97] = 0
    counts = {"full": [TILE, 0, 1, 9, 517], "c1": [10, 11, 31, 32, 33], "c2": [47, 48, 49, 159, 160],
              "c3": [161, 511, 512, 513, 0], "w1100": [0, 1100, 0, 2, 0]}
    terms = {}
    for name, per_tile in counts.items():
        docs = np.concatenate([tile_docs(rng, n, t, c) for t, c in enumerate(per_tile)])
        mixed = np.asarray(MIXED_RUNS)[rng.integers(0, len(MIXED_RUNS), len(docs))]
        if name != "full":
            terms[name + "_1"] = (docs, np.ones(len(docs), dtype=np.int64))
        if name != "w1100":
            terms[name + "_r"] = (docs, mixed)
    for name, layout in (("lanes", {1: 1300, 3: 150}), ("lanes_s", {0: 200, 4: 100})):
        docs, runs = [], []
        for t, n_words in layout.items():
            r = lane_runs(n_words)
            docs.append(tile_docs(rng, n, t, len(r)))
            runs += r
        terms[name] = (np.concatenate(docs), np.asarray(runs))
    edge = np.sort(np.concatenate([[t * TILE, min(n, (t + 1) * TILE) - 1] for t in range(5)]))
    terms["edge"] = (edge, np.resize([1, 2], len(edge)))
    names = list(terms)
    host = index_from_term_postings(names, [encode_term(*terms[t]) for t in names], doc_lens)
    return host, names


class Case:
    """A SearchArray over a host index, its oracle and memoised oracle results."""

    def __init__(self, host, names, **kw):
        from oracle import search as osearch
        from searcharray_b200 import SearchArray
        self.host, self.names = host, names
        self.arr = SearchArray.from_host_index(host, **kw)
        self.oidx = osearch.OracleIndex({t: host.term_words(t) for t in range(host.n_terms)}, host.doc_lens,
                                        avg_doc_length=host.avg_doc_length)
        self._memo = {}

    def want(self, key, fn):
        if key not in self._memo:
            self._memo[key] = fn()
        return self._memo[key]


@pytest.fixture(scope="module")
def mixed():
    return Case(*mixed_corpus())


def view_mask(n):
    mask = np.random.default_rng(7).random(n) < 0.7
    mask[[0, n - 1]] = True
    return mask


def check_mixed(case, what):
    """Every entry point of the term scan on the mixed corpus under the knobs now set."""
    from searcharray_b200 import bm25_similarity
    arr, o = case.arr, case.oidx
    mask = view_mask(len(arr))
    view, ov = arr[mask], o.sliced(mask)
    for t, name in enumerate(case.names):
        tag = f"{what} {name}"
        assert_bits(arr.termfreqs(name), case.want(("tf", t), lambda: o.termfreqs(t)), tag + " termfreqs")
        assert_bits(arr.score(name), case.want(("s", t), lambda: o.score(t)), tag + " score")
        assert_bits(arr.score(name, min_posn=18), case.want(("smin", t), lambda: o.score(t, min_posn=18)),
                    tag + " score min_posn=18")
        assert_bits(arr.score(name, max_posn=35), case.want(("smax", t), lambda: o.score(t, max_posn=35)),
                    tag + " score max_posn=35")
        for k1, b in EXOTIC:
            assert_contract(arr.score(name, similarity=bm25_similarity(k1=k1, b=b)),
                            case.want(("x", t, k1, b), lambda: o.score(t, k1=k1, b=b)), f"{tag} score k1={k1} b={b}")
        assert_bits(view.termfreqs(name), case.want(("vtf", t), lambda: ov.termfreqs(t)), tag + " view termfreqs")
        assert_bits(view.score(name), case.want(("vs", t), lambda: ov.score(t)), tag + " view score")
    queries = case.names + ["missing"]
    for k1, b in ((1.2, 0.75),) + EXOTIC:
        dense = [case.want(("s", t), lambda: o.score(t)) if (k1, b) == (1.2, 0.75) else
                 case.want(("x", t, k1, b), lambda: o.score(t, k1=k1, b=b)) for t in range(len(case.names))]
        dense.append(np.zeros(len(arr), dtype=np.float32))
        for k in TOPK_KS:
            docs, scores = arr.search_topk(queries, k=k, similarity=bm25_similarity(k1=k1, b=b))
            for qi, name in enumerate(queries):
                assert_topk(docs[qi], scores[qi], dense[qi], k, f"{what} search_topk {name} k={k} k1={k1} b={b}")


def test_oracle_bm25_matches_float64(mixed):
    """Common-mode guard: the oracle's float32 BM25 against the same formula evaluated in float64."""
    from oracle.search import compute_idf
    o = mixed.oidx
    t = mixed.names.index("c3_r")
    tf = o.termfreqs(t).astype(np.float64)
    idf = np.float32(compute_idf(o.corpus_size, [o.docfreq(t)]))
    dl = o.doc_lens.astype(np.float64)
    k1, b, avgdl = (np.float64(np.float32(x)) for x in (1.2, 0.75, o.avg_doc_length))
    want = tf / (tf + k1 * ((1 - b) + b * (dl / avgdl))) * np.float64(idf)
    got = o.score(t).astype(np.float64)
    assert np.count_nonzero(got) > 1000
    np.testing.assert_allclose(got, want, rtol=4 * np.finfo(np.float32).eps, atol=0)


@pytest.mark.parametrize("setting", list(KNOBS))
def test_branch_matrix(mixed, monkeypatch, setting):
    """termfreqs, score (default, min_posn / max_posn: FILTER, exotic: ALL_DOCS), search_topk at k = 1 ... 32 and
    termfreqs / score on a mask view (filtered lists: the words path) under one knob setting.  The tile counts of
    mixed_corpus put every branch on both sides of its default threshold; "always" and "never" move the thresholds
    of the staged norms and of the four-records-per-thread path below and above every tile; the prefetch distance 0
    turns the L2 prefetch off, 1 prefetches the very next tile (the short last one included)."""
    set_knobs(monkeypatch, setting)
    check_mixed(mixed, setting)


def test_branch_matrix_no_tf_table_query_major():
    """The branch matrix in a process with SA_NO_TF_TABLE=1 (every term on the words path: directory or binary
    search) and SA_TERM_QUERY_MAJOR=1 (the (tiles, queries) grid), under the default, "always" and "never" knobs."""
    env = dict(os.environ, SA_NO_TF_TABLE="1", SA_TERM_QUERY_MAJOR="1")
    for var in KNOB_VARS:
        env.pop(var, None)
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_term_paths_worker.py")
    r = subprocess.run([sys.executable, worker], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.strip().splitlines()[-1] == "OK", r.stdout[-3000:]


# ----------------------------------------------------------------------------- batches and their stats
def stats(arr):
    from searcharray_b200 import _lib
    st = _lib.SaStats()
    _lib.check(_lib.lib().sa_stats_get(arr._device().handle, ctypes.byref(st)))
    return st


def run_batch(arr, queries, k, idfs=None, runs=1):
    """queries through sa_batch_upload / execute / download, `runs` executes of one upload.  Returns per run
    (docs, scores, n_overflow) and the term / top-k kernel launches of the whole call."""
    from searcharray_b200 import _lib
    from searcharray_b200.similarity import compute_idf, default_bm25
    terms, starts, qidf = arr._topk_queries(queries, lambda dfs: compute_idf(arr.corpus_size, dfs))
    idfs = np.asarray(qidf if idfs is None else idfs, dtype=np.float32)
    L, h = _lib.lib(), arr._device().handle
    out = []
    with arr._shared["lock"]:
        _lib.check(L.sa_stats_reset(h))
        _lib.check(L.sa_batch_upload(h, _lib.p_u32(terms), _lib.p_u32(starts), _lib.p_f32(idfs), len(queries), 0,
                                     arr.avg_doc_length, default_bm25.k1, default_bm25.b, k))
        for _ in range(runs):
            docs = np.empty((len(queries), k), dtype=np.uint32)
            scores = np.empty((len(queries), k), dtype=np.float32)
            n_over = ctypes.c_uint32(0)
            _lib.check(L.sa_batch_execute(h))
            _lib.check(L.sa_batch_download(h, _lib.p_u32(docs), _lib.p_f32(scores), ctypes.byref(n_over)))
            out.append((docs, scores, n_over.value))
    st = stats(arr)
    return out, st.term_kernel_launches, st.topk_kernel_launches


# ------------------------------------------------------------------------------------------------ ties
TIE_TILES = 40
SPARSE_STEP = 41


def ties_corpus():
    """40 tiles of docs of one length.  `sparse`: tf 1 in every 41st doc (~200 per tile); `dense`: tf 1 in every doc;
    `top{c}`: `sparse` with c of its docs, spread over different tiles, at tf 2 (c = k - 1, k, k + 1 for k = 10, 32)."""
    from searcharray_b200.indexing import index_from_term_postings
    n = TIE_TILES * TILE
    sparse = np.arange(0, n, SPARSE_STEP)
    terms = {"sparse": (sparse, np.ones(len(sparse), dtype=np.int64)),
             "dense": (np.arange(n), np.ones(n, dtype=np.int64))}
    for c in (9, 10, 11, 31, 32, 33):
        runs = np.ones(len(sparse), dtype=np.int64)
        # the c docs: one per tile, tiles 3, 10, 17, ... (mod 40), at varying offsets within their tile
        tiles = (3 + 7 * np.arange(c)) % TIE_TILES + TIE_TILES * (np.arange(c) // TIE_TILES)
        picks = [np.searchsorted(sparse, t * TILE + 97 * (i + 1)) for i, t in enumerate(tiles)]
        runs[picks] = 2
        assert len(set(picks)) == c
        terms[f"top{c}"] = (sparse, runs)
    names = list(terms)
    host = index_from_term_postings(names, [encode_term(*terms[t]) for t in names], np.full(n, 50.0, dtype=np.float32))
    return host, names


@pytest.fixture(scope="module")
def ties():
    return Case(*ties_corpus())


def check_batch(case, queries, k, n_overflow, term_launches):
    (res,), tl, kl = run_batch(case.arr, queries, k)
    docs, scores, n_over = res
    for qi, name in enumerate(queries):
        t = case.names.index(name)
        assert_topk(docs[qi], scores[qi], case.want(("s", t), lambda: case.oidx.score(t)), k, f"{name} k={k}")
    assert n_over == n_overflow, (queries, k, n_over)
    assert (tl, kl) == (term_launches, term_launches), (queries, k, tl, kl)


@pytest.mark.parametrize("setting", ["default", "never"])
def test_sparse_ties(ties, monkeypatch, setting):
    """~200 tied docs per tile, fewer than the 256 slots at k = 32: no tile overflows, but all 40 tiles' maxima are
    the top score, so the select keeps ~8,000 survivors and takes its radix path (> 4,096).  At k = 10 (128 slots)
    each tile takes the tie retry instead, which keeps about k docs per tile: no re-run either.  "default" stages
    the norms (>= 48 records: the retry reads the negated tile), "never" gathers them (the plain tile)."""
    set_knobs(monkeypatch, setting)
    for k in (10, 32):
        check_batch(ties, ["sparse"], k, n_overflow=0, term_launches=1)


@pytest.mark.parametrize("setting", ["default", "never"])
def test_dense_ties(ties, monkeypatch, setting):
    """Every doc ties.  The tie retry's doc bound is the k-th smallest of the threads' smallest tied docs that the
    warps publish, 8 per warp: thread t's smallest is tile position 4 t, so the bound lands at position 412 for
    k = 32 and at 132 for k = 10, and a tile keeps 413 / 133 docs, more than its 256 / 128 slots.  Every such query
    therefore takes the host re-run (one more term launch and one more select), whose select sees every doc and
    takes the radix path.  n_overflow is 1: the one dense query.  The ordinary query of the batch stays exact."""
    set_knobs(monkeypatch, setting)
    for k in (10, 32):
        check_batch(ties, ["dense", "sparse"], k, n_overflow=1, term_launches=2)


@pytest.mark.parametrize("setting", ["default", "never"])
def test_two_level_ties(ties, monkeypatch, setting):
    """k - 1, k and k + 1 docs at the top score in different tiles, above ~8,000 docs tied at the second score: the
    result is the top docs in id order, then the lowest ids of the second level.  No query overflows."""
    set_knobs(monkeypatch, setting)
    for k, cs in ((10, (9, 10, 11)), (32, (31, 32, 33))):
        check_batch(ties, [f"top{c}" for c in cs], k, n_overflow=0, term_launches=1)


# ------------------------------------------------------------------------------- exact re-run of a term
def rerun_corpus():
    """Tile 0 holds the term `hot` in every doc, so its record i is doc i.  With one record per thread, thread t
    holds records t + 256 j; the 992 docs of threads 0-30 have tf 5, the other docs tf 1.  Docs have lengths
    10-20, so the high scores differ.  `a` and `b` are ordinary terms."""
    from searcharray_b200.indexing import index_from_term_postings
    rng = np.random.default_rng(5)
    n = 2 * TILE + 100
    hot_docs = np.arange(TILE)
    runs = np.ones(TILE, dtype=np.int64)
    runs[(hot_docs % 256) < 31] = 5
    terms = {"hot": (hot_docs, runs)}
    for name, df in (("a", 3000), ("b", 700)):
        docs = np.sort(rng.choice(n, df, replace=False))
        terms[name] = (docs, np.asarray(MIXED_RUNS)[rng.integers(0, 5, df)])
    names = list(terms)
    host = index_from_term_postings(names, [encode_term(*terms[t]) for t in names],
                                    rng.integers(10, 21, n).astype(np.float32))
    return host, names


def test_term_rerun_exact(monkeypatch):
    """SA_TERM_QUAD_MIN_RECS=2^31 forces one record per thread.  The tile bound is the k-th largest thread maximum
    (k = 32: 8 per warp, of which warp 0 alone holds high ones; k = 10: 4 per warp), so it is the low score; all
    8,192 docs reach it, and the tie retry still keeps the 992 high docs strictly above it -- more than the slots.
    The query takes the exact host re-run on both executes; the other queries stay exact."""
    monkeypatch.setenv("SA_TERM_QUAD_MIN_RECS", str(2 ** 31))
    case = Case(*rerun_corpus())
    queries = ["hot", "a", "b"]
    dense = [case.oidx.score(t) for t in range(3)]
    hot_tf = case.oidx.termfreqs(0)
    assert np.count_nonzero(dense[0] > dense[0][hot_tf == 1].max()) == 992
    for k in (10, 32):
        res, tl, kl = run_batch(case.arr, queries, k, runs=2)
        for run, (docs, scores, n_over) in enumerate(res):
            assert n_over >= 1, (k, run)
            for qi, name in enumerate(queries):
                assert_topk(docs[qi], scores[qi], dense[qi], k, f"{name} k={k} run={run}")
        # each execute: one term launch and one select, plus one of each per re-run query
        assert tl == kl == 2 + sum(r[2] for r in res), (k, tl, kl)


# --------------------------------------------------------------------------------------- shard, raw idf
def test_shard_doc_base():
    """A BM25 shard whose first doc is 1,000,003 (not a tile multiple) with the global corpus size, average doc
    length and document frequencies: score bits from the global idf, search_topk ids absolute."""
    from oracle.search import compute_idf
    from searcharray_b200 import SearchArray
    from searcharray_b200.indexing import index_from_term_postings
    rng = np.random.default_rng(3)
    base, n = 1_000_003, 3 * TILE + 77
    dfs = (5, 300, 2500, 9000)
    terms = []
    for df in dfs:
        docs = np.sort(rng.choice(n, df, replace=False))
        terms.append((docs, np.asarray(MIXED_RUNS)[rng.integers(0, 5, df)]))
    doc_lens = rng.integers(1, 200, n).astype(np.float32)
    names = [f"s{i}" for i in range(len(dfs))]
    host = index_from_term_postings(names, [encode_term(d, r, doc_base=base) for d, r in terms], doc_lens)
    local = index_from_term_postings(names, [encode_term(d, r) for d, r in terms], doc_lens)
    corpus, avgdl = 4_000_000, 93.25
    gdf = np.asarray([df + 1000 * (i + 1) for i, df in enumerate(dfs)], dtype=np.uint64)
    arr = SearchArray.from_host_index(host, doc_base=base, corpus_size=corpus, avg_doc_length=avgdl, global_df=gdf)
    from oracle import search as osearch
    dense = []
    for i, name in enumerate(names):
        tf = osearch.termfreqs_dense(local.term_words(i), n)
        assert_bits(arr.termfreqs(name), tf, name + " termfreqs")
        assert int(arr.docfreq(name)) == int(gdf[i])
        dense.append(oracle_bm25(tf, doc_lens, avgdl, compute_idf(corpus, [gdf[i]])))
        assert_bits(arr.score(name), dense[-1], name + " score")
    for k in (1, 10, 32):
        docs, scores = arr.search_topk(names, k=k)
        for i, name in enumerate(names):
            assert_topk(docs[i], scores[i], dense[i], k, f"{name} k={k}", doc_base=base)


def test_raw_batch_negative_idf(mixed):
    """One negative idf in a raw batch turns the whole chunk into ALL_DOCS; each query is the top k of its own
    scores under its own idf, and the negative one ranks nothing."""
    case = mixed
    queries = ["full_r", "c1_r", "c3_1", "lanes"]
    idfs = np.asarray([1.75, -0.5, 2.25, 0.875], dtype=np.float32)
    dense = [oracle_bm25(case.oidx.termfreqs(case.names.index(q)), case.host.doc_lens, case.host.avg_doc_length, idf)
             for q, idf in zip(queries, idfs)]
    for k in (10, 32):
        ((docs, scores, _),), _, _ = run_batch(case.arr, queries, k, idfs=idfs)
        for qi, name in enumerate(queries):
            assert_topk(docs[qi], scores[qi], dense[qi], k, f"{name} idf={idfs[qi]} k={k}")
        assert np.all(docs[1] == NO_DOC) and np.all(scores[1] == 0)


# --------------------------------------------------------------------------------------------- tf = 2^18
MAX_TF = 1 << 18


def big_tf_case(doc):
    """3 * 8192 + 10 docs; `big` holds every position 0 .. 2^18 - 1 of `doc` (tf 2^18, doc length 2^18) and tf
    1-3 in 2,000 other docs; `other` is an ordinary term."""
    from searcharray_b200.indexing import index_from_term_postings
    from searcharray_b200.roaringish import encode_postings
    rng = np.random.default_rng(18)
    n = 3 * TILE + 10
    doc_lens = rng.integers(1, 100, n).astype(np.float32)
    doc_lens[doc] = MAX_TF
    small = np.sort(rng.choice(np.setdiff1d(np.arange(n), [doc]), 2000, replace=False))
    runs = rng.integers(1, 4, len(small))
    d = np.concatenate([np.repeat(small, runs), np.full(MAX_TF, doc)])
    p = np.concatenate([np.concatenate([18 * np.arange(r) for r in runs]), np.arange(MAX_TF)])
    o = np.lexsort((p, d))
    other = np.sort(rng.choice(n, 500, replace=False))
    host = index_from_term_postings(["big", "other"], [encode_postings(d[o], p[o]), encode_term(other, np.ones(500))],
                                    doc_lens)
    case = Case(host, ["big", "other"])
    assert case.oidx.termfreqs(0)[doc] == MAX_TF
    return case


BIG_DOC = TILE + 1234          # an interior tile offset


@pytest.fixture(scope="module")
def big():
    return big_tf_case(BIG_DOC)


def test_tf_2_18_tf_table(big):
    """Unsliced termfreqs / score: the term has a tf table (19 tf bits)."""
    assert_bits(big.arr.termfreqs("big"), big.oidx.termfreqs(0), "termfreqs")
    assert_bits(big.arr.score("big"), big.oidx.score(0), "score")


def test_tf_2_18_all_docs(big):
    """score with b = 1.0: the ALL_DOCS kernel, which reads the words."""
    from searcharray_b200 import bm25_similarity
    got = big.arr.score("big", similarity=bm25_similarity(b=1.0))
    assert_contract(got, big.oidx.score(0, b=1.0), "score b=1.0")
    assert got[BIG_DOC] > 0


def test_tf_2_18_filter(big):
    """min_posn = 18 (FILTER, the words path): tf 2^18 - 18 = 262,126."""
    got = big.arr.termfreqs("big", min_posn=18)
    assert got[BIG_DOC] == MAX_TF - 18
    assert_bits(got, big.oidx.termfreqs(0, min_posn=18), "termfreqs min_posn=18")


def test_tf_2_18_view(big):
    """termfreqs / score on a view that keeps the doc: the filtered list goes through the words path."""
    mask = view_mask(len(big.arr))
    mask[BIG_DOC] = True
    view, ov = big.arr[mask], big.oidx.sliced(mask)
    assert_bits(view.termfreqs("big"), ov.termfreqs(0), "view termfreqs")
    assert_bits(view.score("big"), ov.score(0), "view score")


def test_tf_2_18_view_topk(big):
    """view.search_topk against view.score: the doc of tf 2^18 ranks first."""
    mask = view_mask(len(big.arr))
    mask[BIG_DOC] = True
    view = big.arr[mask]
    dense = view.score("big")
    docs, scores = view.search_topk(["big"], k=10)
    assert docs[0][0] == np.count_nonzero(mask[:BIG_DOC])
    assert_topk(docs[0], scores[0].astype(np.float32), dense, 10, "view search_topk")


def test_tf_2_18_at_tile_offset_8191():
    """The doc of tf 2^18 at the last offset of its tile, unsliced (ALL_DOCS, FILTER) and as position 8191 of a view:
    a packed head that carried tf into the doc bits would land one float past the shared tile."""
    from searcharray_b200 import bm25_similarity
    doc = 2 * TILE + TILE - 1
    case = big_tf_case(doc)
    arr, o = case.arr, case.oidx
    assert_contract(arr.score("big", similarity=bm25_similarity(b=1.0)), o.score(0, b=1.0), "score b=1.0")
    assert_bits(arr.termfreqs("big", min_posn=18), o.termfreqs(0, min_posn=18), "termfreqs min_posn=18")
    mask = np.zeros(len(arr), dtype=bool)
    mask[2 * TILE:] = True
    view, ov = arr[mask], o.sliced(mask)
    assert_bits(view.termfreqs("big"), ov.termfreqs(0), "view termfreqs")
    assert view.termfreqs("big")[TILE - 1] == MAX_TF
    assert_bits(view.score("big"), ov.score(0), "view score")
