"""Loads one field of tests/golden/tmdb_index.npz (make_golden_tmdb_index.py) back into a HostIndex; shared by
the CPU and GPU TMDB tests."""
import numpy as np


def load_field(z, name):
    from searcharray_b200.indexing import HostIndex, TermDict
    lengths, offsets = z[name + ".lengths"], z[name + ".offsets"]
    words = z[name + ".delta"].copy()
    # undo the per-term delta coding: cumulative sum inside each term's slice
    starts = offsets[lengths > 0].astype(np.int64)
    csum = np.cumsum(words, dtype=np.uint64)
    base = np.zeros(len(words), dtype=np.uint64)
    order = np.argsort(starts)
    s_sorted = starts[order]
    before = np.where(s_sorted > 0, csum[np.maximum(s_sorted, 1) - 1], np.uint64(0))
    seg_len = np.diff(np.concatenate((s_sorted, [len(words)])))
    base = np.repeat(before, seg_len)
    words = csum - base
    td = TermDict()
    for t in bytes(z[name + ".terms"]).decode("utf-8").split("\n"):
        td.add_term(t)
    return HostIndex(words, offsets, lengths, z[name + ".doc_lens"], td,
                     avg_doc_length=z[name + ".avg_doc_length"][()])
