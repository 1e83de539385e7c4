"""searcharray_b200 -- SearchArray's scoring hot path on NVIDIA H100 (sm_90a).

Term-at-a-time BM25 over roaringish posting words and the positional phrase / slop matcher as
hand-written CUDA kernels behind the reference's SearchArray.index / .score / .termfreqs
surface.  Host code is Python (numpy / pandas); the kernels are reached through the C ABI in
include/searcharray_b200.h via ctypes.  No PyTorch, no Triton, no CPU fallback.
"""
from .postings import Hits, SearchArray, Terms, TermsDtype, ws_tokenizer  # noqa: F401
from .similarity import (Similarity, bm25_similarity, bm25_impact, bm25_legacy_similarity,  # noqa: F401
                         classic_similarity, compute_idf, default_bm25)
from .indexing import HostIndex, TermDict, TermMissingError  # noqa: F401
from .query import And, Bool, Boost, DisMax, Feature, Field, In, Or, Range, Rescore  # noqa: F401
from .solr import fields_score_docs, fields_topk  # noqa: F401
