"""GPU: every branch of exact phrase matching (slop 0: phrase_kernel, the search regime, and phrase_tile_kernel, the
conjunction regime, sa_phrase.cu / sa_phrase_warp.cuh) and of span search (slop > 0, sa_span.cu) against the CPU
oracle.  termfreqs must match bit for bit, BM25 scores bit for bit (b = 1.0: the 1e-5 contract with the same NaN
mask), and search_topk must return the oracle's top k by (score desc, id asc) over the scores > 0, empty slots
NO_DOC / 0.

Which regime runs a phrase is chosen on the host per query (sa_phrase_use_conjunction) from the list lengths and
SA_PHRASE_STAGE_RATIO; whether a span query gets the conjunction prefilter from SA_SPAN_CONJ_RATIO.  Both are read on
every call, so each knob setting below forces the regimes in this process.  Every case asserts the branch it took
through the launch counters (sa_stats.phrase_tile_launches / phrase_kernel_launches) and, in batches, n_overflow, so
a threshold change that moves a case to another branch fails here instead of silently covering nothing.

The corpus (phrase_corpus) places docs and positions on purpose; its docstring lists what each family reaches."""
import numpy as np
import pytest

from test_term_paths_gpu import NO_DOC, TILE, assert_bits, assert_contract, assert_topk, run_batch, stats

pytestmark = pytest.mark.gpu

SUB = 1024                          # docs of a tile one warp of the conjunction regime owns
N_DOCS = 40 * TILE + 517            # 40 full tiles and a short one
SHARD_BASE = 1_000_003
RATIO_VARS = ("SA_PHRASE_STAGE_RATIO", "SA_SPAN_CONJ_RATIO")
# unset: the default 50; "0": the search regime only (no span prefilter); 2**40: the conjunction regime (the span
# prefilter) wherever the candidate estimate allows, rare x common phrases included
RATIOS = {"default": None, "search": "0", "conj": str(2 ** 40)}
TOPK_KS = (1, 10, 32)


def set_ratio(monkeypatch, setting):
    for var in RATIO_VARS:
        if RATIOS[setting] is None:
            monkeypatch.delenv(var, raising=False)
        else:
            monkeypatch.setenv(var, RATIOS[setting])


# ------------------------------------------------------------------------------------------------- corpus
class Postings:
    """(doc, position) pairs per term; `words()` encodes each term's sorted, de-duplicated pairs."""

    def __init__(self):
        self.pairs = {}

    def add(self, term, docs, posns):
        docs, posns = np.broadcast_arrays(np.atleast_1d(np.asarray(docs, dtype=np.int64)),
                                          np.asarray(posns, dtype=np.int64))
        self.pairs.setdefault(term, []).append(np.stack([docs, posns]))

    def plant(self, phrase, doc, start):
        """phrase[i] at position start + i of doc."""
        for i, t in enumerate(phrase):
            self.add(t, doc, start + i)

    def words(self, term, doc_base=0):
        from searcharray_b200.roaringish import encode_postings
        p = np.unique(np.concatenate(self.pairs[term], axis=1), axis=1)     # sorted by (doc, posn)
        return encode_postings(p[0] + doc_base, p[1])


def sub0(tile, sub):
    return tile * TILE + sub * SUB


F = [f"f{i}" for i in range(16)]
# plant sub-ranges (tile, warp) where the background of every f term is left out, so that what the warp sees there is
# exactly what is planted
LANE_SUB, RES_SUB, XLEFT_SUB, XRIGHT_SUB, XLEFT3_SUB, PLAIN3_SUB = (3, 2), (4, 5), (6, 1), (6, 6), (7, 3), (7, 4)
P16_SUBS = [(9 + i, 2) for i in range(10)]
OVF_SUB = (12, 7)
ABSENT_TILE, FEW_TILE, LATE_TILE = 39, 38, 37      # f1 absent; f0 and f1 absent; f2 absent
R_TILE = 5                                         # the rare term's 254 lead docs and its 255 / 256 straddle
MID5 = ["f3", "f4", "f0", "f1", "f2"]              # shortest (f0) at 2: middle-out, split 2
GIVEUP_DOCS = (1500, 20000)                        # span doc groups that fill the 512-slot table


def p16_variants():
    """16-term phrases over F (f0 is the shortest list, f1 the next): LR driven from the carry (f0 first) and from
    the other list (f0 second), RL from the carry (f0 last) and from the other list (f0 next to last), middle-out."""
    rest = F[2:]
    return {"p16_lr": ["f0", "f1"] + rest, "p16_lr_o": ["f1", "f0"] + rest,
            "p16_rl": rest[::-1] + ["f1", "f0"], "p16_rl_o": rest[::-1] + ["f0", "f1"],
            "p16_mid": rest[:7] + ["f0", "f1"] + rest[7:]}


def phrase_corpus(doc_base=0):
    """N_DOCS docs, lengths 0..299 with every 97th 0, and these term families:

    f0..f15   balanced lists at 2.5 % + 0.15 % * i of the docs (f0 the shortest), one position each in 0..59, all
              >= 1,024 words (tile directory).  Default ratio: the conjunction regime for every phrase over them.
              Planted matches: inside one 18-position word and across words (position 17 -> 18) at docs 0 (block
              1), 1023 / 1024, 8191 / 8192, 3 * 8192 - 1 / 3 * 8192, the last doc and in the short tile;
              LANE_SUB: 31 one-word matching docs, then a doc whose four words sit at driver lanes 31 .. 34, then
              14 more (46 result docs: res[1]); XLEFT_SUB / XRIGHT_SUB: "f0 f1" where f0 (f1) has an extra word, so
              the warp's first step drives from the other list (the carry); XLEFT3_SUB / PLAIN3_SUB the same for the
              RL chain of "f2 f1 f0"; "f0 f1 f2" across words with f0 also in the next word (`next_handles`);
              "f0 f1 f2" alone (the right half of the middle-out MID5) in many docs; 16-term phrases in P16_SUBS.
              f1 is absent from ABSENT_TILE, f0 and f1 from FEW_TILE, f2 from LATE_TILE.
    m         ~600 words: no tile directory (binary search), mixed with f terms in "f3 m f4".
    o0, o1    balanced, but OVF_SUB holds 70 docs with "o0 o1": more candidates than the warp's compaction area
              (60 words at n = 2), so the conjunction regime flags the query and it re-runs in the search regime.
    r, c      r: ~1,150 words (254 lead docs in R_TILE without c, then a doc with five words at driver threads
              254 .. 258 of the search regime's bigram_step, then ~850 spread docs); c: 30 % of the docs.  "r c"
              and "c r" take the search regime by default and the conjunction regime under 2**40.
    s, s2     one list under two names: runs of 2 .. 5 consecutive positions (one crossing 17 -> 18).  "s s2" is
              guessed different-term, the pair statistics say same-term: a re-run with the flipped guess.
    g0, g1    GIVEUP_DOCS: g0 in 40 blocks, g1 (the last term) in 520 / 680 positions next to them, which fill the
              span search's 512-slot table: it compacts and gives up on the doc group; two plain matches after.
    L0..L2    every list starts in doc 0, block 0: the span search's literal corner."""
    from searcharray_b200.indexing import index_from_term_postings
    rng = np.random.default_rng(1913)
    n = N_DOCS
    P = Postings()
    doc_lens = rng.integers(0, 300, n).astype(np.float32)
    doc_lens[::97] = 0

    # ---- backgrounds
    excluded = np.zeros(n, dtype=bool)
    excluded[0] = True
    for t, s in [LANE_SUB, RES_SUB, XLEFT_SUB, XRIGHT_SUB, XLEFT3_SUB, PLAIN3_SUB, OVF_SUB] + P16_SUBS:
        excluded[sub0(t, s):sub0(t, s) + SUB] = True
    tile_of = np.arange(n) // TILE
    for i, t in enumerate(F):
        keep = (rng.random(n) < 0.025 + 0.0015 * i) & ~excluded
        if t in ("f0", "f1"):
            keep &= tile_of != FEW_TILE
        if t == "f1":
            keep &= tile_of != ABSENT_TILE
        if t == "f2":
            keep &= tile_of != LATE_TILE
        d = np.flatnonzero(keep)
        P.add(t, d, rng.integers(0, 60, len(d)))
    for t, density in (("o0", 0.03), ("o1", 0.03), ("s", 0.02)):
        d = np.flatnonzero((rng.random(n) < density) & ~excluded)
        P.add(t, d, rng.integers(0, 60, len(d)))
    d = np.flatnonzero((rng.random(n) < 0.0018) & ~excluded)
    P.add("m", d, rng.integers(0, 60, len(d)))

    # ---- f: edges, inside a word (start 3) and across words (start 17); doc 0 in block 1 (not the literal corner)
    edges = [1023, 1024, TILE - 1, TILE, 3 * TILE - 1, 3 * TILE, n - 1, 40 * TILE + 5, 40 * TILE + 300]
    P.plant(["f0", "f1"], 0, 20)
    P.plant(["f0", "f1", "f2"], 0, 35)
    for j, d in enumerate(edges):
        P.plant(["f0", "f1"], d, 17 if j % 2 else 3)
        P.plant(["f0", "f1", "f2"], d, 40 if j % 2 else 16)
        P.plant(["f2", "f1", "f0"], d, 70)
        P.plant(MID5, d, 100 + 17 * (j % 2))
        P.plant(["f3", "m", "f4"], d, 130)
    # res[1] and the warp-iteration carry: 31 docs, the straddling doc, 14 more
    base = sub0(*LANE_SUB)
    for j in range(31):
        P.plant(["f0", "f1"], base + 3 * j, 3)
    for b in range(4):
        P.plant(["f0", "f1"], base + 100, 5 + 18 * b)
    for j in range(14):
        P.plant(["f0", "f1"], base + 200 + 5 * j, 17)
    # more than 32 result docs, one word each
    base = sub0(*RES_SUB)
    for j in range(45):
        P.plant(["f0", "f1"], base + 7 * j + 1, 9)
    # first step driven from either side in the conjunction regime: extra words of one term in its candidate docs
    for j in range(6):
        d = sub0(*XLEFT_SUB) + 50 * j
        P.plant(["f0", "f1"], d, 4)
        P.add("f0", d, 200)
        d = sub0(*XRIGHT_SUB) + 50 * j
        P.plant(["f0", "f1"], d, 4)
        P.add("f1", d, 200)
        d = sub0(*XLEFT3_SUB) + 50 * j
        P.plant(["f2", "f1", "f0"], d, 8)
        P.add("f0", d, 220)
        d = sub0(*PLAIN3_SUB) + 50 * j
        P.plant(["f2", "f1", "f0"], d, 8 + 17 * (j % 2))
    # next_handles: an across-word match whose rhs word is also paired by the next lhs word
    hit = rng.choice(np.flatnonzero(~excluded & (tile_of < 36)), 40, replace=False)
    for d in hit[:20]:
        P.plant(["f0", "f1", "f2"], d, 17)
        P.add("f0", d, 30)
    # the right half of MID5 alone
    for d in hit[20:]:
        P.plant(["f0", "f1", "f2"], d, 50)
    # 16-term phrases, inside one word (start 1) and across words (start 10)
    for (name, ph), (t, s) in zip(sorted(p16_variants().items()) * 2, P16_SUBS):
        for j in range(3):
            P.plant(ph, sub0(t, s) + 100 * j + 7, 1 if j != 1 else 10)
    # ---- the overflowing sub-range
    for j in range(70):
        P.plant(["o0", "o1"], sub0(*OVF_SUB) + 13 * j, 5)
    # ---- rare x common
    c_docs = np.flatnonzero(rng.random(n) < 0.3)
    lead = R_TILE * TILE + np.arange(254)
    c_docs = np.setdiff1d(c_docs, lead)
    P.add("c", c_docs, rng.integers(0, 60, len(c_docs)))
    P.add("r", lead, 7)
    straddle = R_TILE * TILE + 300
    for b in range(5):
        P.add("r", straddle, 1 + 18 * b)
        P.add("c", straddle, 2 + 18 * b)
    spread = np.setdiff1d(rng.choice(n, 850, replace=False), np.arange(R_TILE * TILE, R_TILE * TILE + 400))
    P.add("r", spread, rng.integers(0, 60, len(spread)))
    for d in spread[::4]:
        P.plant(["r", "c"], d, 61)
        P.plant(["c", "r"], d, 80)
    # ---- same term: runs of 2 .. 5 positions, one across 17 -> 18
    same = rng.choice(np.flatnonzero(~excluded), 400, replace=False)
    for j, d in enumerate(same):
        start, run = [(3, 2), (10, 3), (30, 4), (40, 5), (16, 3)][j % 5]
        P.add("s", np.full(run, d), start + np.arange(run))
        if j % 3 == 0:
            P.plant(["f5", "s", "s"], d, 100)
            P.plant(["s", "s", "f6"], d, 120)
    # ---- every case phrase at 12 more docs, inside a word or across words
    free = np.flatnonzero(~excluded & ((np.arange(n) < R_TILE * TILE) | (np.arange(n) >= R_TILE * TILE + 400)))
    for name in ("f1 f0", "f2 f0 f1", "lr5", "rl5", "rl5_c", "c f9 r", "mid5", "f3 m f4"):
        for j, d in enumerate(rng.choice(free, 12, replace=False)):
            P.plant(CASES[name][0], d, (3, 17, 30)[j % 3])
    # ---- span table: in GIVEUP_DOCS g0 opens every one of 40 blocks and g1, the last term, fills 13 (17) more
    #      positions of each, so > 512 of its positions survive the candidate slicing; the table fills, compaction
    #      frees nothing, and the walk gives up on the rest of the doc group.  Each is followed by another doc group
    #      of g1 (a plain match), so the reference stays defined.
    blocks = 18 * np.arange(40)
    for d, per_block in zip(GIVEUP_DOCS, (13, 17)):
        P.add("g0", d, blocks)
        P.add("g1", d, (blocks[:, None] + np.arange(1, per_block + 1)).ravel())
    for d in (9000, 33000):
        P.plant(["g0", "g1"], d, 5)
        P.plant(["g0", "g1"], d, 17)
    # ---- literal corner: every list starts in doc 0, block 0
    for i in range(3):
        d = np.sort(rng.choice(np.arange(1, 3000), 300, replace=False))
        P.add(f"L{i}", d, rng.integers(0, 40, len(d)))
        P.add(f"L{i}", 0, [2 + i, 5 + 2 * i])
    P.plant(["L0", "L1", "L2"], 0, 9)

    names = sorted(P.pairs) + ["s2"]
    lists = [P.words(t, doc_base) for t in names[:-1]]
    lists.append(lists[names.index("s")])
    return index_from_term_postings(names, lists, doc_lens), names


class Case:
    """The SearchArray of the corpus (a shard at doc_base), the oracle of the unsharded corpus and memoised results."""

    def __init__(self, doc_base=0):
        from oracle import search as osearch
        from searcharray_b200 import SearchArray
        self.host, self.names = phrase_corpus(doc_base)
        self.doc_base = doc_base
        self.arr = SearchArray.from_host_index(self.host, doc_base=doc_base)
        if doc_base:
            local, _ = phrase_corpus(0)
        else:
            local = self.host
        self.oidx = osearch.OracleIndex({t: local.term_words(t) for t in range(local.n_terms)}, local.doc_lens,
                                        avg_doc_length=local.avg_doc_length)
        self._memo = {}

    def ids(self, phrase):
        return [self.names.index(t) if t in self.names else None for t in phrase]

    def want(self, key, fn):
        if key not in self._memo:
            self._memo[key] = fn()
        return self._memo[key]

    def tf(self, phrase):
        return self.want(("tf",) + tuple(phrase), lambda: self.oidx.termfreqs(self.ids(phrase)))

    def score(self, phrase, b=0.75):
        return self.want(("s", b) + tuple(phrase), lambda: self.oidx.score(self.ids(phrase), b=b))


@pytest.fixture(scope="module")
def corpus():
    return Case()


# --------------------------------------------------------------------------------------------- the cases
# name -> (tokens, regime under the default ratio, what happens after the first launch)
#   regime "conj" / "search";  after: None, "overflow" (a warp sub-range overflows its compaction area: the
#   conjunction regime bounces the query), "guess" (the same-term guess is wrong: one re-run), "missing"
CASES = {
    "f0 f1": (["f0", "f1"], "conj", None),
    "f1 f0": (["f1", "f0"], "conj", None),
    "f0 f1 f2": (["f0", "f1", "f2"], "conj", None),
    "f2 f0 f1": (["f2", "f0", "f1"], "conj", None),
    "f2 f1 f0": (["f2", "f1", "f0"], "conj", None),
    "mid5": (MID5, "conj", None),
    "lr5": (["f0", "f1", "f2", "f3", "f4"], "conj", None),
    "rl5": (["f4", "f3", "f2", "f0", "f1"], "conj", None),
    "rl5_c": (["f4", "f3", "f2", "f1", "f0"], "conj", None),
    "f3 m f4": (["f3", "m", "f4"], "conj", None),
    "o0 o1": (["o0", "o1"], "conj", "overflow"),
    "r c": (["r", "c"], "search", None),
    "c r": (["c", "r"], "search", None),
    "c f9 r": (["c", "f9", "r"], "search", None),
    "s s": (["s", "s"], "conj", None),
    "s s s": (["s", "s", "s"], "conj", None),
    "f5 s s": (["f5", "s", "s"], "conj", None),
    "s s f6": (["s", "s", "f6"], "conj", None),
    "s s2": (["s", "s2"], "conj", "guess"),
    "missing": (["f0", "nope"], "search", "missing"),
}
CASES.update({name: (ph, "conj", None) for name, ph in p16_variants().items()})


def expected_launches(setting, regime, after):
    """(phrase_tile_launches, phrase_kernel_launches) of one termfreqs / score call."""
    if after == "missing":
        return 0, 0
    conj = setting == "conj" or (setting == "default" and regime == "conj")
    if not conj:
        return 0, 2 if after == "guess" else 1
    # the conjunction launch; a bounce restarts in the search regime from the planned guess, which a wrong guess
    # makes run twice (that guess, then the flipped one)
    return 1, {None: 1, "overflow": 2, "guess": 3}[after]


def launches(arr):
    st = stats(arr)
    return st.phrase_tile_launches, st.phrase_kernel_launches


def reset(arr):
    from searcharray_b200 import _lib
    _lib.check(_lib.lib().sa_stats_reset(arr._device().handle))


def test_cases_cover_the_branches(corpus):
    """The corpus does what the cases claim, checked on the oracle's counts: matches at every edge doc, > 32 matching
    docs in RES_SUB and LANE_SUB, a count of 4 in the straddling doc, the overflowing sub-range, MID5's right half
    alone, every list length relation the plans depend on, and more than 512 positions of g1, the last term of the
    "g0 g1" span, in each of GIVEUP_DOCS after the span search's candidate slicing (the 512-slot table fills there),
    with the reference defined."""
    from oracle.search import _span_candidates
    c = corpus
    enc = [c.host.term_words(c.names.index(t)) for t in ("g0", "g1")]
    posns, lengths = _span_candidates([e.copy() for e in enc])
    last = posns[int(lengths[1]):int(lengths[2])]
    last_doc = (last >> np.uint64(36)).astype(np.int64)
    popcount = np.asarray([bin(int(w) & 0x3FFFF).count("1") for w in last])
    for d in GIVEUP_DOCS:
        assert popcount[last_doc == d].sum() > 512, d
        assert last_doc.max() > d, d                       # a later doc group of g1: the walk can skip to it
    for slop in (1, 2, 3, 4):
        tf, und = span_want(c, SPANS["g0 g1"], slop)
        assert und == 0 and np.all(tf[list(GIVEUP_DOCS)] > 0), slop
    tf = c.tf(["f0", "f1"])
    for d in [0, 1023, 1024, TILE - 1, TILE, 3 * TILE - 1, 3 * TILE, N_DOCS - 1, 40 * TILE + 5]:
        assert tf[d] >= 1, d
    for sub in (RES_SUB, LANE_SUB):
        assert np.count_nonzero(tf[sub0(*sub):sub0(*sub) + SUB]) > 32, sub
    assert tf[sub0(*LANE_SUB) + 100] == 4
    assert c.tf(["r", "c"])[R_TILE * TILE + 300] == 5
    assert np.count_nonzero(c.tf(["o0", "o1"])[sub0(*OVF_SUB):sub0(*OVF_SUB) + SUB]) == 70
    right = c.tf(["f0", "f1", "f2"])
    assert np.count_nonzero((right > 0) & (c.tf(MID5) == 0)) > 10
    lens = {t: len(c.host.term_words(c.names.index(t))) for t in c.names}
    assert all(lens[F[i]] < lens[F[i + 1]] for i in range(15)) and lens["f0"] >= 1024
    assert lens["m"] < 1024 <= lens["r"] and lens["r"] * 50 < lens["c"]
    for name, (ph, _, _) in CASES.items():
        if name != "missing":
            assert c.tf(ph).any(), name


# --------------------------------------------------------------------------------------- single queries
@pytest.mark.parametrize("setting", list(RATIOS))
def test_phrase_single(corpus, monkeypatch, setting):
    """termfreqs, score and score with b = 1.0 of every case, each with the regime and the re-runs it must take."""
    from searcharray_b200 import bm25_similarity
    set_ratio(monkeypatch, setting)
    arr = corpus.arr
    for name, (ph, regime, after) in CASES.items():
        want = expected_launches(setting, regime, after)
        reset(arr)
        assert_bits(arr.termfreqs(ph), corpus.tf(ph), f"{setting} {name} termfreqs")
        assert launches(arr) == want, (setting, name, launches(arr), want)
        reset(arr)
        assert_bits(arr.score(ph), corpus.score(ph), f"{setting} {name} score")
        assert launches(arr) == want, (setting, name, "score", launches(arr), want)
        assert_contract(arr.score(ph, similarity=bm25_similarity(b=1.0)), corpus.score(ph, b=1.0),
                        f"{setting} {name} score b=1.0")


def test_phrase_17_terms_refused(corpus):
    from searcharray_b200._lib import SearchArrayB200Error
    ph = F + ["c"]
    for call in (lambda: corpus.arr.termfreqs(ph), lambda: corpus.arr.search_topk([ph], k=10)):
        with pytest.raises(SearchArrayB200Error, match="terms"):
            call()


@pytest.mark.parametrize("setting", list(RATIOS))
def test_phrase_view(corpus, monkeypatch, setting):
    """A mask view filters the lists: always the search regime, whatever the ratio."""
    set_ratio(monkeypatch, setting)
    mask = np.random.default_rng(7).random(N_DOCS) < 0.7
    mask[[0, 1023, 1024, TILE - 1, N_DOCS - 1]] = True
    view, ov = corpus.arr[mask], corpus.oidx.sliced(mask)
    for name, (ph, _, after) in CASES.items():
        ids = corpus.ids(ph)
        reset(corpus.arr)
        assert_bits(view.termfreqs(ph), ov.termfreqs(ids), f"{setting} {name} view termfreqs")
        assert launches(corpus.arr) == expected_launches("search", "search", after), (setting, name)
        assert_bits(view.score(ph), ov.score(ids), f"{setting} {name} view score")


# ------------------------------------------------------------------------------------------------ batches
BATCH = list(CASES) + ["f7", "c", "nope"]


def batch_queries(names):
    return [CASES[q][0] if q in CASES else q for q in names]


def dense_of(corpus, q):
    if q in CASES:
        return corpus.score(CASES[q][0])
    t = corpus.names.index(q) if q in corpus.names else None
    return corpus.want(("term", q), lambda: corpus.oidx.score(t) if t is not None else np.zeros(N_DOCS, np.float32))


def expected_redo(setting, names):
    """n_overflow of the first and of later executes of one upload: overflowing queries re-run on every execute, a
    wrong guess once (the re-run writes the flipped guess back)."""
    ovf = sum(1 for q in names if q in CASES and CASES[q][2] == "overflow" and
              (setting == "conj" or (setting == "default" and CASES[q][1] == "conj")))
    guess = sum(1 for q in names if q in CASES and CASES[q][2] == "guess")
    return ovf + guess, ovf


def any_conj(setting, names):
    return any(q in CASES and CASES[q][2] != "missing" and
               (setting == "conj" or (setting == "default" and CASES[q][1] == "conj")) for q in names)


@pytest.mark.parametrize("setting", list(RATIOS))
def test_phrase_batch(corpus, monkeypatch, setting):
    """search_topk at k = 1, 10, 32 over every case, term queries and an unknown token in one batch (both regimes
    side by side), and one upload executed twice: the second execute keeps the guess the first one's re-run flipped."""
    set_ratio(monkeypatch, setting)
    arr, qs = corpus.arr, batch_queries(BATCH)
    for k in TOPK_KS:
        docs, scores = arr.search_topk(qs, k=k)
        for i, q in enumerate(BATCH):
            assert_topk(docs[i], scores[i], dense_of(corpus, q), k, f"{setting} {q} k={k}")
    res, _, _ = run_batch(arr, qs, 10, runs=2)
    tile, _ = launches(arr)
    assert (tile > 0) == any_conj(setting, BATCH), (setting, tile)
    assert [r[2] for r in res] == list(expected_redo(setting, BATCH)), (setting, [r[2] for r in res])
    for docs, scores, _ in res:
        for i, q in enumerate(BATCH):
            assert_topk(docs[i], scores[i], dense_of(corpus, q), 10, f"{setting} {q} two executes")


@pytest.mark.parametrize("setting", list(RATIOS))
def test_phrase_batch_256(corpus, monkeypatch, setting):
    """256 queries: the search regime splits the doc range into chunks of several tiles (phrase_doc_chunks)."""
    set_ratio(monkeypatch, setting)
    names = (BATCH * 16)[:256]
    res, _, _ = run_batch(corpus.arr, batch_queries(names), 10)
    docs, scores, n_over = res[0]
    tile, _ = launches(corpus.arr)
    assert (tile > 0) == any_conj(setting, names), (setting, tile)
    assert n_over == expected_redo(setting, names)[0], (setting, n_over)
    for i, q in enumerate(names):
        assert_topk(docs[i], scores[i], dense_of(corpus, q), 10, f"{setting} {q} [{i}]")


@pytest.mark.parametrize("setting", list(RATIOS))
def test_phrase_bool_clause(corpus, monkeypatch, setting):
    """A phrase clause of a Bool goes through sa_phrase_row, which may take the conjunction regime:
    s = score(phrase) + score(f7), ranked where the phrase scores > 0 and f8 does not occur.  Each phrase clause runs
    once, in the regime and with the re-runs its termfreqs takes (test_phrase_single)."""
    from searcharray_b200.query import Bool
    from searcharray_b200.similarity import default_bm25
    set_ratio(monkeypatch, setting)
    f7, f8 = dense_of(corpus, "f7"), dense_of(corpus, "f8")
    names = ["f0 f1", "mid5", "r c", "o0 o1", "s s2", "p16_mid", "f3 m f4"]
    qs = [Bool(must=[CASES[q][0]], should=["f7"], must_not=["f8"]) for q in names]
    per_clause = [expected_launches(setting, CASES[q][1], CASES[q][2]) for q in names]
    want = tuple(int(x) for x in np.sum(per_clause, axis=0))
    for k in (10, 32):
        reset(corpus.arr)
        docs, scores, n_redone = corpus.arr._search_topk_bool(qs, k, default_bm25, 0)   # search_topk's Bool route
        assert n_redone == 0 and launches(corpus.arr) == want, (setting, k, n_redone, launches(corpus.arr), want)
        for i, q in enumerate(names):
            ph = corpus.score(CASES[q][0])
            s = (ph + f7).astype(np.float32)
            s[(ph <= 0) | (f8 > 0)] = 0
            assert_topk(docs[i], scores[i], s, k, f"{setting} Bool {q} k={k}")


@pytest.fixture(scope="module")
def shard():
    return Case(SHARD_BASE)


@pytest.mark.parametrize("setting", ["default", "search"])
def test_phrase_shard(corpus, shard, monkeypatch, setting):
    """The corpus as a shard at doc_base 1,000,003 (not a tile multiple): the same counts and scores, search_topk
    ids absolute."""
    set_ratio(monkeypatch, setting)
    for name, (ph, regime, after) in CASES.items():
        reset(shard.arr)
        assert_bits(shard.arr.termfreqs(ph), corpus.tf(ph), f"shard {name} termfreqs")
        assert launches(shard.arr) == expected_launches(setting, regime, after), (setting, name)
        assert_bits(shard.arr.score(ph), corpus.score(ph), f"shard {name} score")
    docs, scores = shard.arr.search_topk(batch_queries(BATCH), k=32)
    for i, q in enumerate(BATCH):
        assert_topk(docs[i], scores[i], dense_of(corpus, q), 32, f"shard {q}", doc_base=SHARD_BASE)


# ------------------------------------------------------------------------------------------- span search
SPANS = {
    "f0 f1": ["f0", "f1"], "f0 f1 f2": ["f0", "f1", "f2"], "mid5": MID5, "p16_mid": p16_variants()["p16_mid"],
    "f3 m f4": ["f3", "m", "f4"], "r c": ["r", "c"], "s s": ["s", "s"], "g0 g1": ["g0", "g1"],
    "literal": ["L0", "L1", "L2"], "missing": ["f0", "nope"],
}
# prefilter under the default ratio: balanced lists that all have a tile directory
SPAN_PREFILTER = {"f0 f1", "f0 f1 f2", "mid5", "p16_mid", "s s"}


def span_want(corpus, ph, slop):
    """The oracle's counts and how many docs the reference leaves undefined (its 512-slot table overflows there)."""
    from oracle import ops as oops

    def run():
        tf = corpus.oidx.termfreqs(corpus.ids(ph), slop=slop)
        return tf, oops.last_span_undefined
    return corpus.want(("span", slop) + tuple(ph), run)


def assert_span(corpus, ph, got, want, und, what):
    """Bit for bit, except where the reference is undefined: then only docs that hold every term of the phrase (the
    only ones whose span table can overflow) may differ, at most `und` of them."""
    if not und:
        assert_bits(got, want, what)
        return
    holders = np.ones(len(want), dtype=bool)
    for t in set(ph):
        holders &= corpus.tf([t]) > 0
    assert_bits(got[~holders], want[~holders], what + " (docs without every term)")
    bad = np.count_nonzero(got[holders] != want[holders])
    assert bad <= und, f"{what}: {bad} docs differ, {und} undefined"


def span_prefilter(setting, name):
    """Whether a span query gets span_cand_kernel: never for the literal corner, an unknown token or a list without a
    tile directory (m, g0, g1); r x c only under 2**40."""
    if name == "r c":
        return setting == "conj"
    return setting != "search" and name in SPAN_PREFILTER


@pytest.mark.parametrize("setting", list(RATIOS))
def test_span_single(corpus, monkeypatch, setting):
    """termfreqs at slop 1 .. 4 with the prefilter forced on, off, and by default.  Launches: span_cand_kernel
    (prefilter) 1, phase 1 3 (span_presence / scan / write), the literal corner 2, phase 2 1."""
    set_ratio(monkeypatch, setting)
    for name, ph in SPANS.items():
        for slop in (1, 2, 3, 4):
            want, und = span_want(corpus, ph, slop)
            reset(corpus.arr)
            got = corpus.arr.termfreqs(ph, slop=slop)
            assert_span(corpus, ph, got, want, und, f"{setting} {name} slop={slop}")
            if name == "missing":
                n = 0
            elif name == "literal":
                n = 2 + 1
            else:
                n = (1 if span_prefilter(setting, name) else 0) + 3 + 1
            assert launches(corpus.arr) == (0, n), (setting, name, slop, launches(corpus.arr), n)
    # 16 terms fork past the reference's table in every doc that holds the phrase: there only the launches and the
    # docs without every term are checked
    assert span_want(corpus, SPANS["p16_mid"], 1)[1] > 0


@pytest.mark.parametrize("setting", list(RATIOS))
def test_span_batch(corpus, shard, monkeypatch, setting):
    """The fused span batch (search_topk with slop on the whole array) on the corpus and on the shard: the top k of
    the oracle's BM25 of the span counts; with 256 queries its tile pass runs chunks of several tiles."""
    set_ratio(monkeypatch, setting)
    names = list(SPANS) + ["f7"]
    qs = [SPANS.get(q, q) for q in names]
    for slop in (1, 3):
        dense = []
        for q in names:
            if q == "f7":
                dense.append(dense_of(corpus, "f7"))
                continue
            # a 16-term span forks past the reference's 512-slot table in every candidate doc: undefined there
            tf, und = span_want(corpus, SPANS[q], slop)
            assert (und > 0) == (q == "p16_mid"), (q, und)
            dense.append(None if und else
                         corpus.want(("span_s", slop, q), lambda: corpus.oidx.score(corpus.ids(SPANS[q]), slop=slop)))
        for arr, base in ((corpus.arr, 0), (shard.arr, SHARD_BASE)):
            reset(arr)
            docs, scores = arr.search_topk(qs, k=10, slop=slop)
            for i, q in enumerate(names):
                # on the shard the L lists start at doc 1,000,003: not the literal corner (shard_literal_spans)
                if dense[i] is not None and not (base and q == "literal"):
                    assert_span_topk(docs[i], scores[i], dense[i], 10, f"{setting} span {q} slop={slop} base={base}",
                                     base)
            pre = any(span_prefilter(setting, q) for q in names if q in SPANS)
            literal = 0 if base else 2
            assert launches(arr) == (0, int(pre) + 3 + literal + 1 + 2), (setting, slop, base, launches(arr))
        big = (qs * 26)[:256]
        docs, scores = corpus.arr.search_topk(big, k=10, slop=slop)
        for i in range(256):
            if dense[i % len(names)] is not None:
                assert_span_topk(docs[i], scores[i], dense[i % len(names)], 10, f"{setting} span256 [{i}] slop={slop}", 0)


def test_shard_literal_spans(shard):
    """The literal corner replays the reference's underflow at header 0, which only doc 0 has.  On the shard the same
    lists start at doc 1,000,003, so they take the ordinary span path: the counts are the oracle's on the shard's
    absolute ids, not those of the unsharded corpus, and no literal launch runs."""
    from oracle import ops as oops, search as osearch
    ph = SPANS["literal"]
    enc = [shard.host.term_words(shard.names.index(t)) for t in ph]
    for slop in (1, 2, 3, 4):
        keys, cnts = osearch.span_search([e.copy() for e in enc], slop)
        assert oops.last_span_undefined == 0
        want = np.zeros(N_DOCS, dtype=np.float32)
        want[keys.astype(np.int64) - SHARD_BASE] = cnts
        reset(shard.arr)
        assert_bits(shard.arr.termfreqs(ph, slop=slop), want, f"shard literal slop={slop}")
        assert launches(shard.arr) == (0, 3 + 1), slop


def assert_span_topk(docs, scores, dense, k, what, doc_base):
    """Span scores: the ids of the oracle's order, scores within 1e-5 (the batch scores the counts with the
    precomputed length norm)."""
    dense = np.asarray(dense, dtype=np.float32)
    nz = np.flatnonzero(dense > 0)
    order = nz[np.lexsort((nz, -dense[nz].astype(np.float64)))][:k]
    assert np.array_equal(docs[:len(order)], (order + doc_base).astype(np.uint32)), f"{what}: {docs} want {order}"
    np.testing.assert_allclose(scores[:len(order)], dense[order], rtol=1e-5, atol=0, err_msg=what)
    assert np.all(docs[len(order):] == NO_DOC) and np.all(scores[len(order):] == 0), what
