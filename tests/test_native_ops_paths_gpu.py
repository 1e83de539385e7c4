"""Every branch of the native set ops (sa_setops.cu) and the op exports against the CPU oracle (oracle.ops, a C
restatement of the reference's Cython ops, and oracle.search), element for element and float32 counts bit for bit.

The intersect family runs one kernel, `partner_kernel`: a CTA takes 1,024 lhs elements, finds the rhs range
[r0, r1) that can hold their partners, and stages that range through shared memory in 4,096-word blocks when it is
at most 8,192 words long, searches global memory when it is longer, and does nothing when it is empty.  Every call
here asserts how many CTAs took each path (`ops.last_path_ctas()`) against `expected_paths`, a numpy restatement of
the range computation, so a case meant for one branch cannot drift into another.

Inputs are sorted by the masked value, the admissible domain of DESIGN.md section 3.6.  intersect_with_adjacents
is compared where the reference's loop returns first occurrences: rhs masked values distinct, and no rhs value 0
when an lhs value + delta wraps past 2^64 (section 3.6 states both)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

U64 = np.uint64
ALL = 0xFFFFFFFFFFFFFFFF
HM = 0xFFFFFFFFFFFC0000                 # header: doc and block
MSB = 0x0000000FFFFC0000                # the block field alone: does not reach bit 63
LOW8 = 0xFFFFFFFFFFFFFF00
MASKS = {"hm": HM, "all": ALL, "msb": MSB, "low8": LOW8}
TILE = 1024
STAGE = 4096


def eq(got, want, what=""):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    if got.dtype == np.float32 or want.dtype == np.float32:
        assert got.dtype == want.dtype == np.float32, (what, got.dtype, want.dtype)
        bad = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
    else:
        bad = np.flatnonzero(got.astype(U64) != want.astype(U64))
    assert len(bad) == 0, (what, int(bad[0]), got[bad[0]], want[bad[0]])


def lowbit(mask):
    return mask & -mask


def field_max(mask):
    """the largest slot: slot s stands for the masked value s * lowbit(mask)"""
    return mask // lowbit(mask)


def words(slots, mask, rng):
    """words whose masked values are slots * lowbit(mask), random bits outside the mask"""
    s = np.asarray(slots, dtype=U64)
    noise = rng.integers(0, 1 << 63, size=len(s), dtype=np.int64).astype(U64) * U64(2) + U64(1)
    return (s * U64(lowbit(mask))) | (noise & U64(~mask & ALL))


# ---------------------------------------------------------------- which path each CTA takes
def expected_paths(lhs, rhs, mask, add):
    """(staged, global, empty) CTAs of one partner pass, restating partner_kernel's range: r0 = first rhs index
    whose masked value reaches the tile's first target, r1 = first one past its last target (nr on overflow)."""
    nl, nr = len(lhs), len(rhs)
    if nl == 0 or nr == 0:
        return np.zeros(3, dtype=np.int64)
    m = U64(mask)
    rv = rhs & m
    firsts = lhs[0::TILE] & m
    lasts = lhs[np.minimum(np.arange(TILE, nl + TILE, TILE), nl) - 1] & m
    out = np.zeros(3, dtype=np.int64)
    for a, b in zip(firsts.tolist(), lasts.tolist()):
        ka, kb = a + add, b + add
        r0 = nr if ka > ALL else int(np.searchsorted(rv, U64(ka), "left"))
        r1 = nr if kb >= ALL else int(np.searchsorted(rv, U64(kb), "right"))
        r1 = max(r1, r0)
        out[2 if r1 == r0 else 0 if r1 - r0 <= 8 * TILE else 1] += 1
    return out


def check_paths(want):
    from searcharray_b200 import ops
    got = ops.last_path_ctas()
    assert tuple(int(x) for x in want) == got, (tuple(int(x) for x in want), got)
    assert ops.last_staged_ctas() == got[0]
    return np.asarray(got, dtype=np.int64)


def run_family(lhs, rhs, mask, with_adjacents=True):
    """intersect (both drop modes), adjacent and intersect_with_adjacents against the oracle, with their paths.
    Returns the summed path counts."""
    from oracle import ops as oops
    from searcharray_b200 import ops
    d = lowbit(mask)
    total = np.zeros(3, dtype=np.int64)
    for drop in (True, False):
        got = ops.intersect(lhs, rhs, mask=mask, drop_duplicates=drop)
        for g, w, name in zip(got, oops.intersect(lhs, rhs, mask=U64(mask), drop_duplicates=drop), ("lhs", "rhs")):
            eq(g, w, f"intersect drop={drop} {name}")
        want = expected_paths(lhs, rhs, mask, 0)
        if not drop:
            want = want + expected_paths(rhs, lhs, mask, 0)
        total += check_paths(want)
    got = ops.adjacent(lhs, rhs, mask=mask)
    for g, w, name in zip(got, oops.adjacent(lhs, rhs, U64(mask)), ("lhs", "rhs")):
        eq(g, w, f"adjacent {name}")
    total += check_paths(expected_paths(lhs, rhs, mask, d))
    if with_adjacents:
        got = ops.intersect_with_adjacents(lhs, rhs, mask=mask)
        for g, w, name in zip(got, oops.intersect_with_adjacents(lhs, rhs, mask=U64(mask)),
                              ("lhs", "rhs", "adj lhs", "adj rhs")):
            eq(g, w, f"intersect_with_adjacents {name}")
        total += check_paths(expected_paths(lhs, rhs, mask, 0) + expected_paths(lhs, rhs, mask, d))
    return total


# ---------------------------------------------------------------- intersect family
@pytest.mark.parametrize("mname", list(MASKS))
@pytest.mark.parametrize("nl", [1, 1023, 1024, 1025, 3 * 1024 + 1])
def test_lhs_lengths(mname, nl):
    mask = MASKS[mname]
    rng = np.random.default_rng(nl * 7 + len(mname))
    span = 4 * nl + 64
    ls = np.sort(rng.choice(span, size=nl, replace=False))
    rs = np.sort(rng.choice(span, size=max(1, 3 * nl // 2), replace=False))
    run_family(words(ls, mask, rng), words(rs, mask, rng), mask)


@pytest.mark.parametrize("mname", list(MASKS))
@pytest.mark.parametrize("width", [STAGE, STAGE + 1, 2 * STAGE, 2 * STAGE + 1])
def test_partner_range_at_the_stage_block_and_the_threshold(mname, width):
    """one lhs tile whose rhs range holds exactly `width` words: 4,096 and 8,192 are staged (one and two full
    blocks), 4,097 adds a one-word block, 8,193 searches global memory.  The range starts on an odd word (the stage
    copy's head word) and, in the second call, ends at nr with nr odd."""
    mask = MASKS[mname]
    rng = np.random.default_rng(width + len(mname))
    # (start, nr): an odd start (the first staged word is not 16-byte aligned) with the range ending inside rhs, and
    # a range that ends at an odd nr
    for start, nr in ((1001, 1001 + width + 500), (1001 + width % 2, 1001 + width % 2 + width)):
        assert start % 2 == 1 or nr % 2 == 1
        rs = np.arange(nr)
        inner = np.sort(rng.choice(np.arange(start + 1, start + width - 1), size=TILE - 2, replace=False))
        ls = np.concatenate([[start], inner, [start + width - 1]])
        lhs, rhs = words(ls, mask, rng), words(rs, mask, rng)
        paths = expected_paths(lhs, rhs, mask, 0)
        assert tuple(paths) == ((1, 0, 0) if width <= 2 * STAGE else (0, 1, 0))
        run_family(lhs, rhs, mask)
        # adjacency targets are one slot higher: the same width, shifted by one word
        if nr > start + width:
            assert tuple(expected_paths(lhs, rhs, mask, lowbit(mask))) == tuple(paths)


@pytest.mark.parametrize("mname", list(MASKS))
def test_runs_across_a_stage_block_and_a_cta_tile(mname):
    """an rhs run of equal masked values that straddles the boundary between two stage blocks (the first copy is in
    the first block), one that starts on the boundary, and an lhs run that straddles a CTA tile, so that the first
    element of the second tile is not a first occurrence"""
    mask = MASKS[mname]
    rng = np.random.default_rng(11 + len(mname))
    rs = np.arange(12_000)
    rs = np.concatenate([rs[:STAGE - 3], np.full(7, STAGE - 3), rs[STAGE - 2:2 * STAGE], np.full(5, 2 * STAGE),
                         rs[2 * STAGE + 1:]])                      # runs over staged words 4,093..4,099 and 8,192..
    # lhs: a run of 4,093 over indices 1,018..1,029 (tile boundary 1,024), one of 8,192 over 2,046..2,050 (2,048)
    # a starts at 1, so tile 0's range starts at rhs word 1 and its second stage block at word 4,097: inside the run
    a = np.concatenate([[1], np.sort(rng.choice(np.arange(2, STAGE - 3), size=TILE - 7, replace=False))])
    b = np.sort(rng.choice(np.arange(STAGE - 2, 2 * STAGE), size=2 * TILE - 2 - (TILE + 6), replace=False))
    c = np.sort(rng.choice(np.arange(2 * STAGE + 1, 11_000), size=3 * TILE - (2 * TILE + 3), replace=False))
    ls = np.concatenate([a, np.full(12, STAGE - 3), b, np.full(5, 2 * STAGE), c])
    assert (ls[TILE - 6:TILE + 6] == STAGE - 3).all() and (ls[2 * TILE - 2:2 * TILE + 3] == 2 * STAGE).all()
    lhs, rhs = words(ls, mask, rng), words(rs, mask, rng)
    run_family(lhs, rhs, mask, with_adjacents=False)
    # intersect_with_adjacents on the lhs runs, rhs distinct
    rd = np.unique(rs)
    run_family(lhs, words(rd, mask, rng), mask)
    # the lhs run's second-tile copies are not reported in drop mode
    from searcharray_b200 import ops
    li, _ = ops.intersect(lhs, words(rd, mask, rng), mask=mask)
    assert TILE not in set(li.tolist()) and TILE - 6 in set(li.tolist())


@pytest.mark.parametrize("mname", list(MASKS))
def test_tiles_with_empty_ranges(mname):
    """tiles whose targets all lie before rhs, between two rhs values, and after rhs: no partner range at all"""
    mask = MASKS[mname]
    rng = np.random.default_rng(23 + len(mname))
    gap_lo, gap_hi = 100_000, 200_000
    rs = np.concatenate([np.arange(5000, 6000), [gap_lo], np.arange(gap_hi, gap_hi + 1000)])
    ls = np.concatenate([np.arange(0, TILE), np.arange(5000, 5000 + TILE), np.arange(gap_lo + 10, gap_lo + 10 + TILE),
                         np.arange(300_000, 300_000 + TILE)])     # before rhs, staged, between two rhs values, after
    lhs, rhs = words(ls, mask, rng), words(rs, mask, rng)
    for add in (0, lowbit(mask)):
        assert tuple(expected_paths(lhs, rhs, mask, add)) == (1, 0, 3)
    run_family(lhs, rhs, mask)


@pytest.mark.parametrize("mname", list(MASKS))
def test_adjacent_delta_past_the_top_of_the_field(mname):
    """lhs holds the largest masked value: + delta overflows u64 (masks reaching bit 63) or carries out of the
    masked field (MSB); nothing may pair with it, and the tile's range ends at nr"""
    mask = MASKS[mname]
    rng = np.random.default_rng(31 + len(mname))
    top = field_max(mask)
    ls = np.array([1, 2, 5, top - 1, top], dtype=object)
    rs = np.array([0, 2, 3, 6, top - 2, top], dtype=object)
    lhs = words(np.array(ls, dtype=U64), mask, rng)
    rhs = words(np.array(rs, dtype=U64), mask, rng)
    run_family(lhs, rhs, mask, with_adjacents=(mask == MSB))
    # the reference's intersect_with_adjacents can pair the top value with an rhs 0 across the wrap: compare it
    # without an rhs 0
    run_family(lhs, rhs[1:], mask)
    from searcharray_b200 import ops
    li, _ = ops.adjacent(lhs, rhs, mask=mask)
    assert len(lhs) - 1 not in set(li.tolist())
    # a whole tile of top values: its range starts and ends at nr
    big = words(np.full(TILE, top, dtype=U64), mask, rng)
    assert tuple(expected_paths(big, rhs, mask, lowbit(mask))) == (0, 0, 1)
    run_family(big, rhs[1:], mask)


def test_every_path_runs():
    """one call per path, and one whose tiles take all three"""
    mask = HM
    rng = np.random.default_rng(41)
    rs = np.arange(0, 40_000)
    tiles = [np.arange(100, 100 + TILE),                                          # staged: range of 1,024
             np.sort(rng.choice(np.arange(2000, 20_000), size=TILE, replace=False)),  # global: ~18,000
             np.arange(50_000, 50_000 + TILE)]                                    # empty: past rhs
    lhs = words(np.concatenate(tiles), mask, rng)
    rhs = words(rs, mask, rng)
    assert tuple(expected_paths(lhs, rhs, mask, 0)) == (1, 1, 1)
    total = np.zeros(3, dtype=np.int64)
    for t in tiles:
        total += run_family(words(t, mask, rng), rhs, mask)
    total += run_family(lhs, rhs, mask)
    assert (total > 0).all(), total


def test_large_random_lists_under_every_mask():
    """posting-like lists of 200,000 and 150,000 words under each mask (sorted by that mask's value)"""
    rng = np.random.default_rng(43)
    for mname, mask in MASKS.items():
        top = min(field_max(mask), 1 << 40)
        ls = np.sort(rng.choice(min(top, 600_000), size=200_000, replace=False))
        rs = np.sort(rng.choice(min(top, 600_000), size=150_000, replace=False))
        run_family(words(ls, mask, rng), words(rs, mask, rng), mask)


# ---------------------------------------------------------------- merges
def merge_cases(rng):
    a = np.sort(rng.choice(1 << 40, size=50_000, replace=False)).astype(U64)
    b = np.sort(rng.choice(1 << 40, size=30_000, replace=False)).astype(U64)
    e = np.array([], dtype=U64)
    sub = np.sort(rng.choice(a, size=20_000, replace=False))
    dl = np.sort(np.concatenate([a, a[::7], a[::11]]))                 # duplicates inside lhs
    dr = np.sort(np.concatenate([sub, sub[::5], sub[::3], b[:100]]))  # duplicates inside rhs, shared with lhs
    return {"lhs empty": (e, b), "rhs empty": (a, e), "both empty": (e, e), "rhs inside lhs": (a, sub),
            "random": (a, b), "lhs dups": (dl, sub), "rhs dups": (a, dr), "both dups": (dl, dr),
            "one each": (a[:1], a[:1]), "one vs three": (a[:1], np.repeat(a[:1], 3)),
            "three vs one": (np.repeat(a[:1], 3), a[:1])}


def test_merge():
    from oracle import ops as oops
    from searcharray_b200 import ops
    rng = np.random.default_rng(51)
    for name, (l, r) in merge_cases(rng).items():
        for drop in (False, True):
            got = ops.merge(l, r, drop_duplicates=drop)
            eq(got, oops.merge(l, r, drop_duplicates=drop), f"{name} drop={drop}")
        if name == "rhs inside lhs":
            eq(ops.merge(l, r, drop_duplicates=True), l, name)          # nothing of rhs kept


def test_sort_merge_counts():
    from oracle import ops as oops
    from searcharray_b200 import ops
    rng = np.random.default_rng(53)
    for name, (l, r) in merge_cases(rng).items():
        lc = rng.random(len(l)).astype(np.float32) * np.float32(1000)
        rc = rng.random(len(r)).astype(np.float32)
        for gi, wi, what in zip(ops.sort_merge_counts(l, lc, r, rc), oops.sort_merge_counts(l, lc, r, rc),
                                ("ids", "counts")):
            eq(gi, wi, f"{name} {what}")
    # shared ids whose float32 sum rounds: 2^24 + 1 -> 2^24, 0.1 + 0.2, 1e8 + 3
    l = np.array([1, 2, 3, 9], dtype=U64)
    r = np.array([1, 2, 3, 4], dtype=U64)
    lc = np.array([2.0 ** 24, 0.1, 1e8, 5], dtype=np.float32)
    rc = np.array([1.0, 0.2, 3.0, 7], dtype=np.float32)
    gi, gc = ops.sort_merge_counts(l, lc, r, rc)
    wi, wc = oops.sort_merge_counts(l, lc, r, rc)
    eq(gi, wi); eq(gc, wc)
    assert gc[0] == np.float32(2.0 ** 24) and gc[1] == np.float32(0.1) + np.float32(0.2)


# ---------------------------------------------------------------- grouped ops and unique
def grouped_ids(rng, n):
    """sorted ids with runs that straddle 256-thread and 1,024-element blocks"""
    ids = np.repeat(np.arange(n), rng.integers(1, 4, size=n))
    ids[250:262] = ids[250]
    ids[1020:1030] = ids[1020]
    ids[2040:2310] = ids[2040]                                     # one run over a 256 boundary and a 1,024 boundary
    return np.maximum.accumulate(ids).astype(U64)


def test_popcount_reduce_at_and_key_sum_over():
    from oracle import ops as oops
    from searcharray_b200 import ops
    rng = np.random.default_rng(61)
    ids = grouped_ids(rng, 40_000)
    pay = rng.integers(0, 1 << 62, size=len(ids), dtype=np.int64).astype(U64)
    pay[rng.random(len(ids)) < 0.3] = 0                            # zero-sum groups
    cnt = rng.integers(0, 1 << 40, size=len(ids), dtype=np.int64).astype(U64)
    cnt[pay == 0] = 0
    for fn, ofn, v in ((ops.popcount_reduce_at, oops.popcount_reduce_at, pay), (ops.key_sum_over, oops.key_sum_over, cnt)):
        gi, gc = fn(ids, v)
        wi, wc = ofn(ids, v)
        eq(gi, wi); eq(gc, wc)
        assert (gc == 0).any()
    # popcount sum 2^24 + 1 in one group (rounds to 2^24), next to a group of 2^24 - 1
    ones = np.full(1 << 18, ALL, dtype=U64)
    pay = np.concatenate([ones, [U64(1)], ones[:-1], [U64((1 << 63) - 1)]])
    ids = np.concatenate([np.zeros((1 << 18) + 1), np.ones(1 << 18)]).astype(U64)
    gi, gc = ops.popcount_reduce_at(ids, pay)
    wi, wc = oops.popcount_reduce_at(ids, pay)
    eq(gi, wi); eq(gc, wc)
    assert gc[0] == np.float32(2.0 ** 24)
    # key sums at 2^24 + 1, 2^53 + 1 and past 2^64 (wraps to 1)
    ids = np.array([0, 0, 1, 1, 2, 2, 3, 3, 3], dtype=U64)
    cnt = np.array([1 << 24, 1, 1 << 53, 1, ALL, 2, 1 << 63, 1 << 63, 5], dtype=U64)
    gi, gc = ops.key_sum_over(ids, cnt)
    wi, wc = oops.key_sum_over(ids, cnt)
    eq(gi, wi); eq(gc, wc)
    assert list(gc) == [np.float32(2 ** 24), np.float32(2.0 ** 53), np.float32(1), np.float32(5)]


def test_unique():
    from oracle import ops as oops
    from searcharray_b200 import ops
    rng = np.random.default_rng(67)
    a = np.sort(rng.integers(0, 1 << 63, size=100_000, dtype=np.int64).astype(U64) * U64(2))
    a = np.sort(np.concatenate([a, a[::3], np.full(3000, a[5000])]))
    for shift in (0, 36, 63):
        eq(ops.unique(a, shift), oops.unique(a, shift), f"rshift {shift}")
    assert len(ops.unique(a, 63)) == 2


# ---------------------------------------------------------------- slicing
def test_payload_slice():
    from oracle import ops as oops
    from searcharray_b200 import ops
    rng = np.random.default_rng(71)
    a = rng.integers(0, 1 << 63, size=60_000, dtype=np.int64).astype(U64)
    a[::5] |= U64(1 << 63)
    for m in (MSB, 0, ALL, HM):
        vals = (a & U64(m))
        mid = int(np.median(vals)) if m else 0
        for lo, hi in ((0, ALL), (mid, mid), (mid + 1, mid), (ALL, 0), (int(vals[7]), int(vals[7])), (1, 2 << 18)):
            eq(ops.payload_slice(a, m, lo, hi), oops.payload_slice(a, U64(m), lo, hi), (hex(m), lo, hi))
    assert len(ops.payload_slice(a, 0, 0, 0)) == len(a) and len(ops.payload_slice(a, 0, 1, ALL)) == 0


def test_as_dense():
    """duplicate indices: the last value wins.  Indices >= size are dropped (the reference writes past its
    buffer there), so the oracle sees only the in-range part."""
    from oracle import ops as oops
    from searcharray_b200 import ops
    rng = np.random.default_rng(73)
    idx = np.sort(rng.integers(0, 50_000, size=80_000)).astype(U64)
    val = rng.random(len(idx)).astype(np.float32)
    eq(ops.as_dense(idx, val, 50_000), oops.as_dense(idx, val, 50_000))
    size = 30_000
    inside = idx < U64(size)
    got = ops.as_dense(idx, val, size)
    eq(got, oops.as_dense(idx[inside], val[inside], size))
    eq(ops.as_dense(idx, val, 0), np.zeros(0, dtype=np.float32))


# ---------------------------------------------------------------- popcount64_reduce
def one_doc_words(doc, tf):
    """a doc's words, blocks 0, 1, ... full (18 positions) except the last: exactly tf positions"""
    full, rest = divmod(tf, 18)
    bits = [0x3FFFF] * full + ([(1 << rest) - 1] if rest else [])
    blk = np.arange(len(bits), dtype=U64)
    return (U64(doc) << U64(36)) | (blk << U64(18)) | np.array(bits, dtype=U64)


def test_popcount64_reduce_past_the_19_bit_tf():
    """a doc with 524,304 positions (29,128 words of 0x3FFFF) counts 524,304, not its low 19 bits (16)"""
    from oracle import ops as oops
    from searcharray_b200 import ops
    w = one_doc_words(3, 524_304)
    assert len(w) == 29_128
    ids, cnt = ops.popcount64_reduce(w)
    wi, wc = oops.popcount64_reduce(w, 36, 0x3FFFF)
    assert list(wc) == [524_304.0]
    eq(ids, wi); eq(cnt, wc)


def test_popcount64_reduce():
    from oracle import ops as oops
    from searcharray_b200 import ops
    rng = np.random.default_rng(79)
    parts = [one_doc_words(0, 3), one_doc_words(1, (1 << 19) - 1), one_doc_words(2, 1 << 19),
             one_doc_words(5, 524_304), one_doc_words(6, 17)]
    # docs over several 8,192-doc tiles, some with words that carry no position bits
    docs = np.sort(rng.choice(np.arange(7, 40_000), size=5000, replace=False))
    for d in docs:
        nb = int(rng.integers(1, 4))
        blk = np.sort(rng.choice(14_000, size=nb, replace=False)).astype(U64)
        bits = rng.integers(0, 1 << 18, size=nb).astype(U64)
        if d % 7 == 0:
            bits[:] = 0
        parts.append((U64(d) << U64(36)) | (blk << U64(18)) | bits)
    top = (1 << 28) - 1
    parts += [one_doc_words(top - 2, 40), one_doc_words(top - 1, 1 << 19), one_doc_words(top, 1)]
    w = np.concatenate(parts)
    ids, cnt = ops.popcount64_reduce(w)
    wi, wc = oops.popcount64_reduce(w, 36, 0x3FFFF)
    eq(ids, wi); eq(cnt, wc)
    assert (cnt == 0).any() and cnt[1] == (1 << 19) - 1 and cnt[2] == 1 << 19
    # near the top of the doc-id space on its own (the old one-tile index was placed at min_doc)
    w = np.concatenate(parts[-3:])
    ids, cnt = ops.popcount64_reduce(w)
    wi, wc = oops.popcount64_reduce(w, 36, 0x3FFFF)
    eq(ids, wi); eq(cnt, wc)


# ---------------------------------------------------------------- bigram_freqs
def posting(rng, n_docs, p, max_block, sticky=None):
    """a random posting list: per doc 1-4 distinct blocks < max_block; `sticky` = (other list, share): reuse that
    share of the other list's headers so that the two lists meet"""
    docs = np.flatnonzero(rng.random(n_docs) < p).astype(U64)
    nb = rng.integers(1, 5, size=len(docs))
    d = np.repeat(docs, nb)
    blk = np.concatenate([np.sort(rng.choice(max_block, size=k, replace=False)) for k in nb]).astype(U64)
    w = (d << U64(36)) | (blk << U64(18)) | rng.integers(1, 1 << 18, size=len(d)).astype(U64)
    if sticky is not None:
        other, share = sticky
        pick = other[rng.random(len(other)) < share]
        hdr = pick & U64(HM)
        nxt = hdr + U64(1 << 18)                                   # the next block: adjacency across 17 -> 18
        ok = ((nxt >> U64(18)) & U64(0x3FFFF)) != U64(0)
        extra = np.concatenate([hdr | U64(1), nxt[ok] | U64(1)])    # bit 0: the position after the other's bit 17
        w = np.concatenate([w, extra])
        w = w[np.argsort(w, kind="stable")]
        keep = np.concatenate([[True], (w[1:] & U64(HM)) != (w[:-1] & U64(HM))])
        w = w[keep]                                                # one word per header
    return w


@pytest.mark.parametrize("max_block", [14_564, 1 << 18])
def test_bigram_freqs(max_block):
    """random lists of 10^5 words and more, both continuation modes; blocks up to 14,563 (MAX_POSN) or past it"""
    from oracle import search as osearch
    from searcharray_b200 import ops
    rng = np.random.default_rng(max_block)
    lhs = posting(rng, 60_000, 0.7, max_block)
    rhs = posting(rng, 60_000, 0.6, max_block, sticky=(lhs, 0.5))
    lhs[rng.random(len(lhs)) < 0.2] |= U64(1 << 17)                # bit 17 set: phrases that cross into the next block
    assert len(lhs) > 100_000 and len(rhs) > 100_000
    if max_block > 14_564:
        assert ((lhs >> U64(18)) & U64(0x3FFFF)).max() > 14_563
    cases = [(lhs, rhs), (lhs, lhs.copy()), (rhs, lhs)]
    for a, b in cases:
        for cont_rhs, cont in ((True, osearch.RHS), (False, osearch.LHS)):
            (gi, gc), gn = ops.bigram_freqs(a, b, cont_rhs=cont_rhs)
            (wi, wc), wn = osearch.bigram_freqs(a.copy(), b.copy(), cont)
            eq(gi, np.asarray(wi, dtype=U64), "ids"); eq(gc, np.asarray(wc, dtype=np.float32), "counts")
            eq(gn, np.asarray(wn, dtype=U64), "next")
            assert len(gi) > 1000
