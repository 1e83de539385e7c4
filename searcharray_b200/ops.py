"""Device implementations of the reference's native ops on raw host arrays (parity tests and
the Similarity protocol entry point).  Thin ctypes calls -- all arithmetic runs in CUDA."""
import ctypes

import numpy as np

from . import _lib


def bm25_score(term_freqs, doc_lens, avg_doc_lens, idf, k1, b, device=0):
    """searcharray.bm25.bm25_score (reference bm25/bm25.pyx:28-41): in place on term_freqs."""
    tf = term_freqs
    if tf.dtype != np.float32 or not tf.flags.c_contiguous:
        raise ValueError("term_freqs must be contiguous float32")
    dl = np.ascontiguousarray(doc_lens, dtype=np.float32)
    if len(dl) != len(tf):
        raise ValueError("doc_lens and term_freqs must have the same length")
    _lib.check(_lib.lib().sa_op_bm25_score(_lib.p_f32(tf), _lib.p_f32(dl), len(tf), float(avg_doc_lens),
                                           float(idf), float(k1), float(b), device))
    return tf


def popcount64_reduce(words, device=0):
    """reference roaringish/popcount.pyx:271-278 with key_shift=36, value_mask=0x3FFFF."""
    w = np.ascontiguousarray(words, dtype=np.uint64)
    if len(w) == 0:
        return np.array([]), np.array([])
    keys = np.empty(len(w), dtype=np.uint64)
    cnts = np.empty(len(w), dtype=np.float32)
    n = ctypes.c_uint64(0)
    _lib.check(_lib.lib().sa_op_popcount64_reduce(_lib.p_u64(w), len(w), device, _lib.p_u64(keys),
                                                  _lib.p_f32(cnts), ctypes.byref(n)))
    return keys[:n.value].copy(), cnts[:n.value].copy()


def bigram_freqs(lhs, rhs, cont_rhs=True, device=0):
    """reference phrase/bigram_freqs.py:213-307 -> ((doc ids, counts), continuation words)."""
    lhs = np.ascontiguousarray(lhs, dtype=np.uint64)
    rhs = np.ascontiguousarray(rhs, dtype=np.uint64)
    cap = 2 * min(len(lhs), len(rhs)) + 2
    ids = np.empty(cap, dtype=np.uint64)
    cnts = np.empty(cap, dtype=np.float32)
    nxt = np.empty(cap, dtype=np.uint64)
    n_ids, n_next = ctypes.c_uint64(0), ctypes.c_uint64(0)
    _lib.check(_lib.lib().sa_op_bigram_freqs(_lib.p_u64(lhs), len(lhs), _lib.p_u64(rhs), len(rhs),
                                             1 if cont_rhs else 0, device, _lib.p_u64(ids), _lib.p_f32(cnts),
                                             ctypes.byref(n_ids), _lib.p_u64(nxt), ctypes.byref(n_next)))
    return (ids[:n_ids.value].copy(), cnts[:n_ids.value].copy()), nxt[:n_next.value].copy()


# ---- the reference's sorted-set ops on the device (sa_setops.cu): same call shapes as
#      searcharray.roaringish.{intersect, adjacent, intersect_with_adjacents, merge, sort_merge_counts,
#      unique, popcount64, popcount_reduce_at, key_sum_over, payload_slice, as_dense}
ALL_BITS = 0xFFFFFFFFFFFFFFFF


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


def _n():
    return ctypes.c_uint64(0)


def intersect(lhs, rhs, mask=ALL_BITS, drop_duplicates=True, device=0):
    """reference intersect.pyx:278-320 -> (lhs_idx, rhs_idx); ValueError if mask == 0."""
    if mask == 0:
        raise ValueError("Mask cannot be zero")
    lhs, rhs = _u64(lhs), _u64(rhs)
    li, ri = np.empty(len(lhs), dtype=np.uint64), np.empty(len(rhs), dtype=np.uint64)
    nl, nr = _n(), _n()
    _lib.check(_lib.lib().sa_op_intersect(_lib.p_u64(lhs), len(lhs), _lib.p_u64(rhs), len(rhs), int(mask),
                                          1 if drop_duplicates else 0, device, _lib.p_u64(li), _lib.p_u64(ri),
                                          ctypes.byref(nl), ctypes.byref(nr)))
    return li[:nl.value].copy(), ri[:nr.value].copy()


def adjacent(lhs, rhs, mask=ALL_BITS, device=0):
    """reference intersect.pyx:323-343"""
    if mask == 0:
        raise ValueError("Mask cannot be zero")
    lhs, rhs = _u64(lhs), _u64(rhs)
    cap = min(len(lhs), len(rhs))
    li, ri = np.empty(cap, dtype=np.uint64), np.empty(cap, dtype=np.uint64)
    n = _n()
    _lib.check(_lib.lib().sa_op_adjacent(_lib.p_u64(lhs), len(lhs), _lib.p_u64(rhs), len(rhs), int(mask), device,
                                         _lib.p_u64(li), _lib.p_u64(ri), ctypes.byref(n)))
    return li[:n.value].copy(), ri[:n.value].copy()


def intersect_with_adjacents(lhs, rhs, mask=ALL_BITS, device=0):
    """reference intersect.pyx:346-390 -> (lhs_idx, rhs_idx, adj_lhs_idx, adj_rhs_idx)"""
    if mask == 0:
        raise ValueError("Mask cannot be zero")
    lhs, rhs = _u64(lhs), _u64(rhs)
    cap = min(len(lhs), len(rhs))
    li, ri, lai, rai = (np.empty(cap, dtype=np.uint64) for _ in range(4))
    n, na = _n(), _n()
    _lib.check(_lib.lib().sa_op_intersect_with_adjacents(_lib.p_u64(lhs), len(lhs), _lib.p_u64(rhs), len(rhs), int(mask),
                                                         device, _lib.p_u64(li), _lib.p_u64(ri), ctypes.byref(n),
                                                         _lib.p_u64(lai), _lib.p_u64(rai), ctypes.byref(na)))
    return li[:n.value].copy(), ri[:n.value].copy(), lai[:na.value].copy(), rai[:na.value].copy()


def merge(lhs, rhs, drop_duplicates=False, device=0):
    """reference merge.pyx:137-158"""
    lhs, rhs = _u64(lhs), _u64(rhs)
    out = np.empty(len(lhs) + len(rhs), dtype=np.uint64)
    n = _n()
    _lib.check(_lib.lib().sa_op_merge(_lib.p_u64(lhs), len(lhs), _lib.p_u64(rhs), len(rhs), 1 if drop_duplicates else 0,
                                      device, _lib.p_u64(out), ctypes.byref(n)))
    return out[:n.value].copy()


def sort_merge_counts(lhs_ids, lhs_counts, rhs_ids, rhs_counts, device=0):
    """reference merge.pyx:211-232"""
    li, ri = _u64(lhs_ids), _u64(rhs_ids)
    lc = np.ascontiguousarray(lhs_counts, dtype=np.float32)
    rc = np.ascontiguousarray(rhs_counts, dtype=np.float32)
    ids = np.empty(len(li) + len(ri), dtype=np.uint64)
    cnt = np.empty(len(li) + len(ri), dtype=np.float32)
    n = _n()
    _lib.check(_lib.lib().sa_op_sort_merge_counts(_lib.p_u64(li), _lib.p_f32(lc), len(li), _lib.p_u64(ri), _lib.p_f32(rc),
                                                  len(ri), device, _lib.p_u64(ids), _lib.p_f32(cnt), ctypes.byref(n)))
    return ids[:n.value].copy(), cnt[:n.value].copy()


def unique(arr, rshift=0, device=0):
    """reference unique.pyx:139-145"""
    arr = _u64(arr)
    out = np.empty(len(arr), dtype=np.uint64)
    n = _n()
    _lib.check(_lib.lib().sa_op_unique(_lib.p_u64(arr), len(arr), int(rshift), device, _lib.p_u64(out), ctypes.byref(n)))
    return out[:n.value].copy()


def popcount64(arr, device=0):
    """reference popcount.pyx:120-122"""
    arr = _u64(arr)
    out = np.empty(len(arr), dtype=np.uint64)
    _lib.check(_lib.lib().sa_op_popcount64(_lib.p_u64(arr), len(arr), device, _lib.p_u64(out)))
    return out


def _grouped(fn, ids, vals, device):
    ids, vals = _u64(ids), _u64(vals)
    if len(ids) != len(vals):
        raise ValueError("ids and values must have the same length")
    io = np.empty(len(ids), dtype=np.uint64)
    co = np.empty(len(ids), dtype=np.float32)
    n = _n()
    _lib.check(fn(_lib.p_u64(ids), _lib.p_u64(vals), len(ids), device, _lib.p_u64(io), _lib.p_f32(co), ctypes.byref(n)))
    return io[:n.value].copy(), co[:n.value].copy()


def popcount_reduce_at(ids, payload, device=0):
    """reference popcount.pyx:150-165 (zero-count groups kept)"""
    return _grouped(_lib.lib().sa_op_popcount_reduce_at, ids, payload, device)


def key_sum_over(ids, count, device=0):
    """reference popcount.pyx:195-204"""
    return _grouped(_lib.lib().sa_op_key_sum_over, ids, count, device)


def payload_slice(arr, msb_mask, min_payload, max_payload, device=0):
    """reference roaringish_ops.pyx:46-68 (compares the UNSHIFTED masked word, quirk vi)"""
    arr = _u64(arr)
    out = np.empty(len(arr), dtype=np.uint64)
    n = _n()
    _lib.check(_lib.lib().sa_op_payload_slice(_lib.p_u64(arr), len(arr), int(msb_mask), int(min_payload), int(max_payload),
                                              device, _lib.p_u64(out), ctypes.byref(n)))
    return out[:n.value].copy()


def as_dense(indices, values, size, device=0):
    """reference roaringish_ops.pyx:84-98"""
    idx = _u64(indices)
    val = np.ascontiguousarray(values, dtype=np.float32)
    if len(idx) != len(val):
        raise ValueError("indices and values must have the same length")
    out = np.empty(int(size), dtype=np.float32)
    _lib.check(_lib.lib().sa_op_as_dense(_lib.p_u64(idx), _lib.p_f32(val), len(idx), int(size), device, _lib.p_f32(out)))
    return out


def last_staged_ctas():
    return int(_lib.lib().sa_op_last_staged_ctas())


def last_path_ctas():
    """CTAs of this thread's last intersect-family call by path: (TMA-staged, global search, empty rhs range)."""
    out = np.zeros(3, dtype=np.uint64)
    _lib.lib().sa_op_last_path_ctas(_lib.p_u64(out))
    return tuple(int(x) for x in out)
