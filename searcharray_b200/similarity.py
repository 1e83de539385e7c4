"""Similarity plug-ins, mirroring reference searcharray/similarity.py.

`Similarity` is the same callable protocol (similarity.py:8-16).  `bm25_similarity(k1, b)`
returns a callable object that ALSO carries (k1, b): SearchArray.score recognises it and runs
the fused GPU kernel (postings -> tf -> BM25 in one launch) instead of calling it on a host
vector.  Any other callable is treated as a user plug-in and receives the GPU-computed dense
term-frequency vector on the host, exactly like the reference.
"""
from typing import Protocol

import numpy as np


class Similarity(Protocol):
    def __call__(self, term_freqs, doc_freqs, doc_lens, avg_doc_lens, num_docs) -> np.ndarray:
        ...


def compute_idf(num_docs, dfs):
    """reference similarity.py:19-21 -- float64 on the host (negligible, SURVEY section 8a row 6)."""
    dfs = np.asarray(dfs)
    return np.sum(np.log(1 + (num_docs - dfs + 0.5) / (dfs + 0.5)))


class Bm25Similarity:
    """BM25 as in Lucene 9 (reference similarity.py:24-38), evaluated on the GPU."""
    kind = 3                  # SA_SIM_BM25: search_topk on a view (sa_score_batch_topk_sim)
    out_dtype = np.float32

    def __init__(self, k1=1.2, b=0.75):
        self.k1 = k1
        self.b = b

    def __call__(self, term_freqs, doc_freqs, doc_lens, avg_doc_lens, num_docs):
        # Protocol entry point for callers that already hold a host tf vector (e.g. an
        # edismax-style combiner): still the CUDA op, never numpy.
        from . import ops
        if avg_doc_lens == 0:
            return np.zeros_like(term_freqs)
        idf = compute_idf(num_docs, doc_freqs)
        return ops.bm25_score(term_freqs, doc_lens, avg_doc_lens, idf, self.k1, self.b)

    def __repr__(self):
        return f"bm25_similarity(k1={self.k1}, b={self.b})"


def bm25_similarity(k1: float = 1.2, b: float = 0.75) -> Bm25Similarity:
    return Bm25Similarity(k1, b)


default_bm25 = bm25_similarity()


class _DeviceSimilarity:
    """A non-default similarity of the reference (similarity.py:41-89) evaluated by a CUDA kernel
    (sa_op_similarity).  Same callable protocol; SearchArray.score hands it the GPU-computed
    term-frequency vector like any user plug-in."""
    kind = None
    out_dtype = np.float64

    def __init__(self, k1=1.2, b=0.75):
        self.k1, self.b = k1, b

    def _idf(self, doc_freqs, num_docs):
        return 0.0

    def __call__(self, term_freqs, doc_freqs, doc_lens, avg_doc_lens, num_docs):
        import ctypes
        from . import _lib
        tf = np.ascontiguousarray(term_freqs, dtype=np.float32)
        if self.kind != 2 and avg_doc_lens == 0:       # similarity.py:49-50, 66-67 (classic has no such branch)
            return np.zeros_like(tf)
        dl = np.ascontiguousarray(doc_lens, dtype=np.float32)
        if len(dl) != len(tf):
            raise ValueError("term_freqs and doc_lens differ in length")
        out = np.empty(len(tf), dtype=self.out_dtype)
        _lib.check(_lib.lib().sa_op_similarity(self.kind, _lib.p_f32(tf), _lib.p_f32(dl), len(tf),
                                               float(np.float32(avg_doc_lens)), float(self._idf(doc_freqs, num_docs)),
                                               float(self.k1), float(self.b), 0, out.ctypes.data_as(ctypes.c_void_p)))
        return out


class Bm25Impact(_DeviceSimilarity):
    """BM25 without the idf (reference bm25_impact, similarity.py:41-54): float32."""
    kind = 0
    out_dtype = np.float32

    def __repr__(self):
        return f"bm25_impact(k1={self.k1}, b={self.b})"


class Bm25Legacy(_DeviceSimilarity):
    """BM25 before LUCENE-8563, (k1 + 1) in the numerator (reference similarity.py:57-72): float64."""
    kind = 1

    def _idf(self, doc_freqs, num_docs):
        return compute_idf(num_docs, doc_freqs)

    def __repr__(self):
        return f"bm25_legacy_similarity(k1={self.k1}, b={self.b})"


class ClassicSimilarity(_DeviceSimilarity):
    """Lucene classic TF-IDF (reference similarity.py:75-89): float64."""
    kind = 2

    def __init__(self):
        super().__init__(0.0, 0.0)

    def _idf(self, doc_freqs, num_docs):
        return np.log((num_docs + 1) / (np.sum(np.asarray(doc_freqs), axis=0) + 1)) + 1

    def __repr__(self):
        return "classic_similarity()"


def bm25_impact(k1: float = 1.2, b: float = 0.75) -> Bm25Impact:
    return Bm25Impact(k1, b)


def bm25_legacy_similarity(k1: float = 1.2, b: float = 0.75) -> Bm25Legacy:
    return Bm25Legacy(k1, b)


def classic_similarity() -> ClassicSimilarity:
    return ClassicSimilarity()
