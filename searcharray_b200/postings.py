"""SearchArray -- the reference's search surface, backed by the CUDA kernels.

Mirrors the Search API of reference searcharray/postings.py (`SearchArray.index` :249-300,
`termfreqs` :607-638, `docfreq` :640-647, `doclengths` :649-650, `score` :652-680,
`positions` :682-687, `_phrase_freq` :689-708): same names, argument meaning, return types
(dense float32[len(self)] numpy vectors) and error behaviour (TypeError / ValueError, unknown
terms -> zeros).  The postings live in HBM (one `sa_index` handle per array); every
`.score/.termfreqs` is one C-ABI call into libsearcharray_b200.so.  There is no CPU path.

Host-side pandas plumbing beyond what a DataFrame column needs is out of scope
(SURVEY.md section 2 row 2).
"""
import ctypes
import numbers
import threading
import weakref
from typing import Dict, List, NamedTuple, Optional, Union

import numpy as np
import pandas as pd
from pandas.api.extensions import ExtensionArray, ExtensionDtype, register_extension_dtype
from pandas.api.types import is_list_like

from . import _lib
from .indexing import HostIndex, TermMissingError, build_index
from .roaringish import decode_positions
from .similarity import (Bm25Impact, Bm25Legacy, Bm25Similarity, ClassicSimilarity, Similarity, compute_idf,
                         default_bm25)


def ws_tokenizer(string):
    """reference postings.py:206-211"""
    if pd.isna(string):
        return []
    if not isinstance(string, str):
        raise ValueError("Expected a string")
    return string.split()


class Terms:
    """One indexed doc: term -> positions (a light stand-in for reference postings.py:57-160)."""

    def __init__(self, postings, doc_len=0):
        self.postings = postings
        self.doc_len = doc_len

    def terms(self):
        return ((t, len(p)) for t, p in self.postings.items())

    def termfreq(self, token):
        return len(self.postings.get(token, ()))

    def positions(self, token=None):
        if token is None:
            return self.postings
        return self.postings.get(token)

    def __len__(self):
        return len(self.postings)

    def __eq__(self, other):
        return isinstance(other, Terms) and self.doc_len == other.doc_len and \
            {k: list(v) for k, v in self.postings.items()} == {k: list(v) for k, v in other.postings.items()}

    def __hash__(self):
        return hash((self.doc_len, tuple(sorted(self.postings))))

    def __repr__(self):
        return f"Terms({ {k: list(map(int, v)) for k, v in self.postings.items()} })"


@register_extension_dtype
class TermsDtype(ExtensionDtype):
    """reference postings.py:163-203"""
    name = "tokenized_text_b200"
    type = Terms
    kind = "O"

    @classmethod
    def construct_from_string(cls, string):
        if not isinstance(string, str):
            raise TypeError("'construct_from_string' expects a string, got {}".format(type(string)))
        if string == cls.name:
            return cls()
        raise TypeError(f"Cannot construct a '{cls.__name__}' from '{string}'")

    @classmethod
    def construct_array_type(cls):
        return SearchArray

    @property
    def na_value(self):
        return Terms({})

    def __repr__(self):
        return "TermsDtype()"


class _PinnedPool:
    """Result vectors live in pinned host memory so the float32[N] D2H copy runs at PCIe
    rate; buffers are recycled when the numpy array that views them is garbage-collected.
    Sizes are bucketed to powers of two (so differently sized slices share buffers) and the idle
    pool is capped: beyond the cap a released buffer goes back to the driver (sa_host_free)."""

    MAX_IDLE_BYTES = 1 << 30

    def __init__(self):
        self._free = {}
        self._idle = 0
        self._lock = threading.Lock()

    @staticmethod
    def _bucket(nbytes):
        b = 4096
        while b < nbytes:
            b <<= 1
        return b

    def empty_f32(self, n):
        n = int(n)
        nbytes = self._bucket(max(n, 1) * 4)
        with self._lock:
            lst = self._free.get(nbytes)
            ptr = lst.pop() if lst else None
            if ptr is not None:
                self._idle -= nbytes
        if ptr is None:
            p = ctypes.c_void_p()
            _lib.check(_lib.lib().sa_host_alloc(ctypes.byref(p), nbytes))
            ptr = p.value
        buf = (ctypes.c_float * max(n, 1)).from_address(ptr)
        weakref.finalize(buf, self._release, nbytes, ptr)
        return np.frombuffer(buf, dtype=np.float32, count=n)

    def _release(self, nbytes, ptr):
        with self._lock:
            if self._idle + nbytes <= self.MAX_IDLE_BYTES:
                self._free.setdefault(nbytes, []).append(ptr)
                self._idle += nbytes
                return
        if _lib._lib is not None:
            _lib._lib.sa_host_free(ctypes.c_void_p(ptr))


_pool = _PinnedPool()

_TILE_DOCS, _TILE_THREADS = 8192, 256          # SA_TILE_DOCS, SA_TERM_THREADS (csrc/sa_term.cuh)


def pack_where(where, n, n_queries):
    """The `where=` mask of search_topk / fields_topk over n docs for n_queries queries, checked before any device
    work -- a dtype other than bool raises TypeError, a shape other than (n,) or (n_queries, n) ValueError -- and
    packed as the `_where` entry points take it: uint32[R, SA_WHERE_WORDS(n)], R = 1 (one mask for the batch) or
    n_queries.  Bits are in the tile kernels' owner order (include/searcharray_b200.h): bit 4 j + e of word
    t * 256 + i is doc t * 8192 + 4 (i + 256 j) + e; bits past n are 0."""
    w = np.asarray(where)
    if w.dtype != np.bool_:
        raise TypeError(f"where must be a boolean mask (dtype bool), not dtype {w.dtype}")
    if w.shape != (n,) and w.shape != (n_queries, n):
        raise ValueError(f"where must have shape ({n},) or ({n_queries}, {n}) (one mask per query), not {w.shape}")
    rows = w.reshape(1 if w.ndim == 1 else n_queries, n)
    n_tiles = -(-n // _TILE_DOCS)
    padded = np.zeros((rows.shape[0], n_tiles * _TILE_DOCS), dtype=bool)
    padded[:, :n] = rows
    # [row, tile, j, i, e] -> [row, tile, i, j, e]: thread i's 32 docs, bit 4 j + e
    owner = padded.reshape(rows.shape[0], n_tiles, 32 // 4, _TILE_THREADS, 4).transpose(0, 1, 3, 2, 4)
    packed = np.packbits(owner.reshape(rows.shape[0], n_tiles * _TILE_THREADS, 32), axis=-1, bitorder="little")
    return np.ascontiguousarray(packed).view("<u4").reshape(rows.shape[0], n_tiles * _TILE_THREADS).astype(
        np.uint32, copy=False)


def _where_args(bits):
    """A packed mask as the C calls take it: (where_bits, where_stride); one row is the batch's mask, None no mask."""
    if bits is None:
        return None, 0
    return _lib.p_u32(bits), (bits.shape[1] if bits.shape[0] > 1 else 0)


def _where_part(bits, sel):
    """The packed mask of the queries `sel` selects (a one-row mask is every query's)."""
    return bits if bits is None or bits.shape[0] == 1 or sel.all() else np.ascontiguousarray(bits[sel])


class Hits(NamedTuple):
    """The hit and facet counts of a batched top-k call with `facets=` (SearchArray.search_topk, solr.fields_topk).
    total[q]: how many docs query q ranks (all of them, not only the top k).  facets[name][q, b]: how many of those
    docs have code b in facet `name`."""
    total: np.ndarray                   # int64[Q]
    facets: Dict[object, np.ndarray]    # name -> int64[Q, n_buckets]


class _Counts:
    """The counts of one sa_score_batch_topk_bool / sa_multi_score_batch_topk_bool call: per facet its key in
    Hits.facets, its field slot, its slot on that field's index and its bucket count, and the uint32 outputs the call
    fills."""

    def __init__(self, facets, arrays, n_queries):
        """facets: (key, field slot, name) triples, the name set on arrays[field slot] (ValueError otherwise)."""
        found = [arrays[field]._facet_slot(name) for _, field, name in facets]
        self.keys, self.n_buckets = [key for key, _, _ in facets], [nb for _, nb in found]
        self.fields = np.asarray([field for _, field, _ in facets], dtype=np.uint32)
        self.slots = np.asarray([slot for slot, _ in found], dtype=np.uint32)
        self.total = np.zeros(n_queries, dtype=np.uint32)
        self.counts = np.zeros((n_queries, sum(self.n_buckets)), dtype=np.uint32)

    @staticmethod
    def args(counts):
        """The trailing arguments of the boolean entry points for `counts`, a _Counts or None (out_total NULL: no
        counting)."""
        if counts is None:
            return 0, None, None, None, None
        if not counts.keys:
            return 0, None, None, _lib.p_u32(counts.total), None
        return (len(counts.keys), _lib.p_u32(counts.fields), _lib.p_u32(counts.slots), _lib.p_u32(counts.total),
                _lib.p_u32(counts.counts))

    def hits(self):
        ends = np.cumsum(self.n_buckets)
        return Hits(self.total.astype(np.int64), {key: self.counts[:, e - nb:e].astype(np.int64)
                                                  for key, nb, e in zip(self.keys, self.n_buckets, ends)})


def check_facet_keys(facets, what):
    """facets= as a list of distinct keys, at most SA_BOOL_MAX_FACETS (ValueError), before any device work."""
    from .query import SA_BOOL_MAX_FACETS
    if isinstance(facets, (str, tuple)) or not is_list_like(facets):
        raise TypeError(f"facets is a list of {what}, not {facets!r}")
    facets = list(facets)
    if len(facets) > SA_BOOL_MAX_FACETS:
        raise ValueError(f"at most {SA_BOOL_MAX_FACETS} facets in one call, not {len(facets)}")
    if len(set(facets)) != len(facets):
        raise ValueError(f"facets are named once each: {facets}")
    return facets


def _check_dismax(members, clauses, clause_slot, arrays, sims, idfs=None):
    """ValueError unless the DisMax members (indices into clauses) are sparse-safe (query.check_dismax_members) under
    the k1, b and avgdl of their slot (clause_slot[i]: an index into arrays and sims) and their float32 idf.  idfs=None:
    the check before any device work, with idf 0, of the parameters alone."""
    from .query import check_dismax_members

    def params(i):
        s = clause_slot[i]
        return sims[s].k1, sims[s].b, arrays[s].avg_doc_length, 0.0 if idfs is None else idfs[i]
    check_dismax_members([(i, clauses[i]) for i in members], params)


class _PreparedBool:
    """One call of sa_score_batch_topk_bool over one SearchArray, or of sa_multi_score_batch_topk_bool over the columns
    of a solr.fields_topk plan, prepared from a flattened batch (query.BoolBatch): each clause's term ids, term starts
    and float32 idf from its own column, as that column's .score takes them, the feature and facet columns its clauses
    read and the counts it fills.  Build it and run it with the arrays' locks held (the array's lock; solr._locked for a
    multi)."""

    def __init__(self, arrays, sims, clause_slot, queries, batch, where=None, facets=None, multi=None, group=None):
        """arrays, sims: per slot its SearchArray and similarity (one array: one slot).  clause_slot: uint32 per clause
        of batch, its slot (0 for a nested clause).  batch: queries flattened (query.flatten_bool).  where: a packed
        mask (pack_where), None: no mask.  facets: (key in Hits.facets, slot, name) triples, None: no counting.
        multi: the solr._Multi over arrays for fields_topk, None for one array.  group: (slot, name) of a group column
        set on arrays[slot] (set_group) to collapse on, None: no collapsing.  A facet, feature or group name not set on
        its slot's array, an In code past its facet's buckets, and DisMax members whose idf is not sparse-safe, are
        ValueErrors, the names and codes checked before any device work."""
        from .query import Field, dismax_members
        self.arrays, self.batch, self.where = arrays, batch, where
        self.counts = None if facets is None else _Counts(facets, arrays, batch.n_queries)
        # the collapse entry point's leading arguments: the group column's slot (and its field slot on a multi)
        self.group = None if group is None else (group[0], arrays[group[0]]._group_slot(group[1]))
        clauses = batch.clauses
        feats = self.columns(clauses, clause_slot, arrays)
        text = np.asarray([i for i, c in enumerate(clauses) if c is not None and i not in feats], dtype=np.int64)
        n_terms, self.idfs = np.zeros(len(clauses), dtype=np.int64), np.zeros(len(clauses), dtype=np.float32)
        slot_terms = []
        for s, arr in enumerate(arrays):
            idx = text[clause_slot[text] == s]
            t, starts, idf = arr._topk_queries([clauses[i].clause if isinstance(clauses[i], Field) else clauses[i]
                                                for i in idx.tolist()],
                                               lambda dfs, arr=arr: compute_idf(arr.corpus_size, dfs))
            n_terms[idx], self.idfs[idx] = np.diff(starts), idf
            slot_terms.append((idx, t, starts))
        f = list(feats)
        n_terms[f], self.idfs[f] = [len(e) for e, _ in feats.values()], [param for _, param in feats.values()]
        self.c_starts = np.concatenate([[0], np.cumsum(n_terms)]).astype(np.uint32)
        # each slot's text clauses' terms from their clause's start on, each column clause's entries from its start
        self.terms = np.empty(int(self.c_starts[-1]), dtype=np.uint32)
        for idx, t, starts in slot_terms:
            first = self.c_starts[idx].astype(np.int64) - starts[:-1]
            self.terms[np.repeat(first, np.diff(starts)) + np.arange(len(t))] = t
        for i, (e, _) in feats.items():
            self.terms[self.c_starts[i]:self.c_starts[i] + len(e)] = e
        if batch.groups is not None:
            _check_dismax(dismax_members(queries), clauses, clause_slot, arrays, sims, self.idfs)
        for s in {int(clause_slot[i]) for i in feats}:
            arrays[s]._device().sync_features(arrays[s].host)
            arrays[s]._device().sync_facets(arrays[s].host)         # In clauses read facet columns
        if self.counts is not None:
            for s in set(self.counts.fields.tolist()):
                arrays[s]._device().sync_facets(arrays[s].host)
        if self.group is not None:
            arrays[self.group[0]]._device().sync_groups(arrays[self.group[0]].host)
        for arr in arrays:          # a sliced view of the same column may have left its row filter installed
            arr._apply_rows(arr._device())
        if multi is None:
            self.entry, self.handle = _lib.lib().sa_score_batch_topk_bool, arrays[0]._device().handle
            self.c_field, self.bm25 = (), (arrays[0].avg_doc_length, sims[0].k1, sims[0].b)
        else:               # the clause slots, and avgdl, k1 and b per slot (a pointer keeps its array alive)
            self.entry, self.handle = _lib.lib().sa_multi_score_batch_topk_bool, multi.handle
            self.c_field = (_lib.p_u32(clause_slot),)
            self.bm25 = tuple(_lib.p_f32(np.asarray(v, dtype=np.float32)) for v in
                              ([a.avg_doc_length for a in arrays], [s.k1 for s in sims], [s.b for s in sims]))
        self.group_args = ()
        if self.group is not None:
            lib = _lib.lib()
            self.entry = lib.sa_score_batch_topk_bool_collapse if multi is None else \
                lib.sa_multi_score_batch_topk_bool_collapse
            self.group_args = self.group[1:] if multi is None else self.group

    @staticmethod
    def columns(clauses, clause_slot, arrays):
        """The Feature, Range and In clauses as query.column_terms encodes them, each on its slot's index: {index:
        (clause entries, float32 parameter)}; ValueError for a name not set there or an In code past its buckets."""
        from .query import column_terms
        return column_terms(clauses, lambda i, c: arrays[clause_slot[i]]._feature_slot(c.name),
                            lambda i, c: arrays[clause_slot[i]]._facet_slot(c.name))

    @staticmethod
    def features(clauses, clause_slot, arrays):
        """The feature clauses as query.feature_terms encodes them, each on its slot's index: {index: (reserved term
        id, float32 parameter)}; ValueError for a name not set there."""
        from .query import feature_terms
        return feature_terms(clauses, lambda i, f: arrays[clause_slot[i]]._feature_slot(f.name))

    def run(self, k, slop):
        """Makes the call: (docs uint32[Q, k], scores float32[Q, k], queries re-run exactly), and the Hits when
        counting.  The batch's None arrays are passed as NULL, which selects the instance."""
        b = self.batch
        docs = np.empty((b.n_queries, k), dtype=np.uint32)
        scores = np.empty((b.n_queries, k), dtype=np.float32)
        n_redone = ctypes.c_uint32(0)
        opt = lambda a, p: None if a is None else p(a)      # noqa: E731
        p_w, stride = _where_args(self.where)
        _lib.check(self.entry(
            self.handle, *self.group_args, len(b.node_starts) - 1, _lib.p_u32(b.node_starts),
            opt(b.clause_node, _lib.p_u32), *self.c_field, _lib.p_u32(self.terms), _lib.p_u32(self.c_starts),
            _lib.p_f32(self.idfs), opt(b.weights, _lib.p_f32), opt(b.occurs, _lib.p_u8), opt(b.groups, _lib.p_u32),
            opt(b.ties, _lib.p_f32), _lib.p_u32(b.mm), b.n_queries, int(slop), *self.bm25, k, p_w, len(self.arrays[0]),
            stride,
            _lib.p_u32(docs), _lib.p_f32(scores), ctypes.byref(n_redone), *_Counts.args(self.counts)))
        out = docs, scores, n_redone.value
        return out if self.counts is None else out + (self.counts.hits(),)

    def score_docs(self, docs, slop):
        """Makes the score-docs call on the same descriptors (sa_score_docs_bool, sa_multi_score_docs_bool): float32
        [Q, K], the value each query ranks each of its docs with.  docs: uint32 [Q, K] (check_docs)."""
        b = self.batch
        out = np.empty(docs.shape, dtype=np.float32)
        opt = lambda a, p: None if a is None else p(a)      # noqa: E731
        entry = _lib.lib().sa_score_docs_bool if not self.c_field else _lib.lib().sa_multi_score_docs_bool
        _lib.check(entry(
            self.handle, len(b.node_starts) - 1, _lib.p_u32(b.node_starts), opt(b.clause_node, _lib.p_u32),
            *self.c_field, _lib.p_u32(self.terms), _lib.p_u32(self.c_starts), _lib.p_f32(self.idfs),
            opt(b.weights, _lib.p_f32), opt(b.occurs, _lib.p_u8), opt(b.groups, _lib.p_u32), opt(b.ties, _lib.p_f32),
            _lib.p_u32(b.mm), b.n_queries, int(slop), *self.bm25, _lib.p_u32(docs), docs.shape[1], _lib.p_f32(out)))
        return out


def _refuse_column_queries(queries):
    """TypeError for a Feature, Range or In given as a query of its own rather than as a clause."""
    from .query import Feature, In, Range
    for q in queries:
        if isinstance(q, Feature):
            raise TypeError(f"a Feature is a clause, not a query: write Bool(should=[{q!r}])")
        if isinstance(q, (Range, In)):
            raise TypeError(f"a {type(q).__name__} is a filter clause, not a query: write Bool(filter=[{q!r}]) with "
                            "a must or should clause")


def check_docs(docs, n_queries, doc_base, n_docs):
    """The docs of score_docs / fields_score_docs, checked before any device work: an integer array of shape
    (n_queries, K) (TypeError for another dtype, ValueError for another shape), each id NO_DOC or a doc of the array,
    doc_base <= id < doc_base + n_docs (ValueError).  Returns them as contiguous uint32."""
    d = np.asarray(docs)
    if d.dtype.kind not in "iu":
        raise TypeError(f"docs must be an integer array, not dtype {d.dtype}")
    if d.ndim != 2 or d.shape[0] != n_queries:
        raise ValueError(f"docs must have shape ({n_queries}, K), one row per query, not {d.shape}")
    bad = ~((d == _lib.NO_DOC) | ((d >= doc_base) & (d < doc_base + n_docs)))
    if bad.any():
        q, j = np.argwhere(bad)[0]
        raise ValueError(f"docs[{q}, {j}] = {d[q, j]} is neither NO_DOC nor a doc id in [{doc_base}, "
                         f"{doc_base + n_docs})")
    return np.ascontiguousarray(d, dtype=np.uint32)


class DeviceIndex:
    """Owns one sa_index handle (one shard in one GPU's HBM)."""

    def __init__(self, host: HostIndex, device=0, doc_base=0):
        self.handle = ctypes.c_void_p()
        self.n_docs = host.n_docs
        self._rows_set = False
        words = host.words
        words_ptr = ctypes.cast(words.ctypes.data, _lib.P_u64) if len(words) else None   # (also a read-only memmap)
        _lib.check(_lib.lib().sa_index_create(
            words_ptr, len(words), _lib.p_u64(host.term_offsets),
            _lib.p_u64(host.term_lengths), host.n_terms, _lib.p_f32(host.doc_lens), host.n_docs,
            doc_base, device, ctypes.byref(self.handle)))
        self._finalizer = weakref.finalize(self, DeviceIndex._destroy, self.handle)
        self.features = {}          # slot -> the host array last uploaded there
        self.sync_features(host)
        self.facets = {}            # slot -> the host codes last uploaded there
        self.sync_facets(host)
        self.groups = {}            # slot -> the host codes last uploaded there
        self.sync_groups(host)

    def sync_features(self, host: HostIndex):
        """Uploads every feature column of `host` that this index does not hold yet (sa_index_set_feature)."""
        for slot, values in enumerate(host.features.values()):
            if self.features.get(slot) is not values:
                _lib.check(_lib.lib().sa_index_set_feature(self.handle, slot, _lib.p_f32(values), len(values)))
                self.features[slot] = values

    def sync_facets(self, host: HostIndex):
        """Uploads every facet column of `host` that this index does not hold yet (sa_index_set_facet)."""
        for slot, (codes, n_buckets) in enumerate(host.facets.values()):
            if self.facets.get(slot) is not codes:
                _lib.check(_lib.lib().sa_index_set_facet(self.handle, slot, _lib.p_i32(codes), len(codes), n_buckets))
                self.facets[slot] = codes

    def sync_groups(self, host: HostIndex):
        """Uploads every group column of `host` that this index does not hold yet (sa_index_set_group)."""
        for slot, codes in enumerate(host.groups.values()):
            if self.groups.get(slot) is not codes:
                _lib.check(_lib.lib().sa_index_set_group(self.handle, slot, _lib.p_i32(codes), len(codes)))
                self.groups[slot] = codes

    @staticmethod
    def _destroy(handle):
        if handle and _lib._lib is not None:
            _lib._lib.sa_index_destroy(handle)

    def close(self):
        self._finalizer()


class SearchArray(ExtensionArray):
    """An ExtensionArray of tokenised text searchable with term / phrase queries on the GPU."""

    dtype = TermsDtype()

    def __init__(self, postings, tokenizer=ws_tokenizer, avoid_copies=True, device=0):
        if not is_list_like(postings):
            raise TypeError("Expected list-like object, got {}".format(type(postings)))
        self.tokenizer = tokenizer
        self.avoid_copies = avoid_copies
        self.device = device
        docs = []
        for p in postings:
            if isinstance(p, Terms):
                toks = [None] * int(p.doc_len)
                for t, posns in p.postings.items():
                    for x in posns:
                        if x >= len(toks):
                            toks.extend([None] * (x + 1 - len(toks)))
                        toks[x] = t
                docs.append(toks)
            elif isinstance(p, str) or p is None or (isinstance(p, float) and np.isnan(p)):
                docs.append(tokenizer(p))
            else:
                raise TypeError("Expected a Terms or a string")
        self._set_host(build_index(docs, lambda toks: [t for t in toks if t is not None]))

    # ------------------------------------------------------------------ construction
    def _set_host(self, host: HostIndex):
        self.host = host
        self.term_dict = host.term_dict
        self.doc_lens = host.doc_lens
        self.avg_doc_length = host.avg_doc_length
        self.corpus_size = host.n_docs
        self.rows = None                 # sliced view: local doc ids (postings.py:344-358)
        self._bm25_doc_lens = None
        # doc-range shard of a larger corpus (SURVEY 8e): absolute id of row 0, and the GLOBAL
        # statistics idf / BM25 must use (set by from_host_index; None = this array is the corpus)
        self.doc_base = 0
        self.global_df = None            # uint64[n_terms] document frequencies over all shards
        self.comm = None                 # shard.ShardComm: sums over ranks where a query needs them
        self._shared = {"dev": None, "lock": threading.RLock()}   # shared by views/copies

    @classmethod
    def index(cls, array, tokenizer=ws_tokenizer, truncate=False, batch_size=100000, avoid_copies=True,
              workers=4, cache_gt_than=25, data_dir: Optional[str] = None, autowarm=True,
              device=0, gpu_build=False) -> "SearchArray":
        """Index an array of strings (reference postings.py:249-300).  batch_size / workers /
        cache_gt_than / data_dir / autowarm are accepted for signature compatibility: the
        per-term df table the reference warms lazily is computed on the device at upload.  data_dir:
        the posting words are written to `<data_dir>/<n>.dat` and memory-mapped (reference MemoryMappedArrays); the
        upload then DMAs straight from the mapping (cudaHostRegister), and a pickle carries the file name only."""
        if not is_list_like(array):
            raise TypeError("Expected list-like object, got {}".format(type(array)))
        host = build_index(list(array), tokenizer, truncate=truncate, gpu_build=device if gpu_build else None)
        if data_dir is not None:            # reference indexing.py:228-230, 291-293: memmap the bit positions
            host.memmap(data_dir)
        return cls.from_host_index(host, tokenizer=tokenizer, avoid_copies=avoid_copies, device=device)

    @classmethod
    def from_host_index(cls, host: HostIndex, tokenizer=ws_tokenizer, avoid_copies=True, device=0,
                        doc_base=0, corpus_size=None, avg_doc_length=None, global_df=None, comm=None):
        """Wraps a prebuilt HostIndex.  For one doc-range shard of a larger corpus pass the shard's
        first absolute doc id and the global corpus size / average doc length / per-term document
        frequencies (idf must not depend on the sharding, SURVEY 8e)."""
        obj = cls.__new__(cls)
        obj.tokenizer = tokenizer
        obj.avoid_copies = avoid_copies
        obj.device = device
        obj._set_host(host)
        obj.doc_base = int(doc_base)
        if corpus_size is not None:
            obj.corpus_size = int(corpus_size)
        if avg_doc_length is not None:
            obj.avg_doc_length = avg_doc_length
        obj.global_df = None if global_df is None else np.asarray(global_df, dtype=np.uint64)
        obj.comm = comm
        return obj

    def _device(self) -> DeviceIndex:
        sh = self._shared
        if sh["dev"] is None:
            with sh["lock"]:
                if sh["dev"] is None:
                    sh["dev"] = DeviceIndex(self.host, device=self.device, doc_base=self.doc_base)
        return sh["dev"]

    def __getstate__(self):
        st = dict(self.__dict__)
        st["_shared"] = None            # device handles never travel; re-uploaded lazily
        return st

    def __setstate__(self, st):
        self.__dict__.update(st)
        self._shared = {"dev": None, "lock": threading.RLock()}

    # ------------------------------------------------------------ ExtensionArray bits
    @classmethod
    def _from_sequence(cls, scalars, dtype=None, copy=False):
        return cls(list(scalars))

    def __len__(self):
        return len(self.doc_lens) if self.rows is None else len(self.rows)

    @property
    def nbytes(self):
        return self.host.words.nbytes + self.host.doc_lens.nbytes

    def memory_usage(self, deep=False):
        return self.nbytes

    def isna(self):
        return self.doclengths() == 0

    def _row_terms(self, doc_id):
        post = {}
        key = np.uint64(doc_id + self.doc_base) << np.uint64(36)     # words carry ABSOLUTE doc ids (shards)
        nxt = np.uint64(doc_id + self.doc_base + 1) << np.uint64(36)
        for t in range(self.host.n_terms):
            w = self.host.term_words(t)
            a, b = np.searchsorted(w, key), np.searchsorted(w, nxt)
            if b > a:
                post[self.term_dict.get_term(t)] = decode_positions(w[a:b])
        return Terms(post, doc_len=int(self.host.doc_lens[doc_id]))

    def __getitem__(self, key):
        key = pd.api.indexers.check_array_indexer(self, key)
        if isinstance(key, numbers.Integral):
            n = len(self)
            if key < 0:
                key += n
            if not 0 <= key < n:
                raise IndexError("index out of bounds")
            doc = key if self.rows is None else int(self.rows[key])
            return self._row_terms(doc)
        rows = np.arange(len(self.doc_lens))[key] if self.rows is None else self.rows[key]
        view = SearchArray.__new__(SearchArray)
        view.__dict__.update(self.__dict__)
        view.rows = np.ascontiguousarray(rows, dtype=np.uint64)
        # Reference quirk: `arr.doc_lens = self.doc_lens[key]` (postings.py:353) is a STRIDED VIEW
        # for a stepped slice and bm25_score walks it contiguously (bm25.pyx:34-41), i.e. BM25 on
        # arr[a::s] sees the parent's doc_lens[a], [a+1], ...  Reproduced for parity.
        view._bm25_doc_lens = None
        if isinstance(key, slice) and key.step not in (None, 1) and len(rows):
            parent = self.doclengths()
            first = int(np.arange(len(parent))[key][0])
            if first + len(rows) <= len(parent):
                view._bm25_doc_lens = np.ascontiguousarray(parent[first:first + len(rows)])
        return view

    def take(self, indices, allow_fill=False, fill_value=None):
        idx = np.asarray(indices)
        if allow_fill and (idx < 0).any():
            raise NotImplementedError("take with fill is host-side pandas plumbing (out of scope)")
        return self[idx]

    def copy(self):
        c = SearchArray.__new__(SearchArray)
        c.__dict__.update(self.__dict__)
        return c

    @classmethod
    def _concat_same_type(cls, to_concat):
        if len(to_concat) == 1:
            return to_concat[0]
        raise NotImplementedError("concatenation re-indexes; out of scope for the scoring path")

    def __eq__(self, other):
        if isinstance(other, SearchArray):
            if len(self) != len(other):
                return False
            return np.asarray([a == b for a, b in zip(self, other)], dtype=bool)
        return NotImplemented

    # ******************************************************************************
    # Search API (reference postings.py:604-708)
    # ******************************************************************************
    def _check_token_arg(self, token):
        if isinstance(token, str):
            return token
        elif isinstance(token, list) and len(token) == 1:
            return token[0]
        elif isinstance(token, list):
            return token
        else:
            raise TypeError("Expected a string or list of strings for phrases")

    def _term_id(self, token):
        try:
            return self.term_dict.get_term_id(token)
        except TermMissingError:
            return _lib.NO_TERM

    @staticmethod
    def _payload_bounds(min_posn, max_posn):
        """RoaringishEncoder.slice argument checks (reference roaringish.py:267-282)."""
        if min_posn is None and max_posn is None:
            return 0, _lib.ALL_BITS
        if min_posn is not None and min_posn % 18 != 0:
            raise ValueError("min_payload must be a multiple of 18")
        if max_posn is not None and max_posn % 18 != 17:
            raise ValueError("max_payload must be a multiple of 18 - 1")
        lo = 0 if min_posn is None else min_posn
        hi = _lib.ALL_BITS if max_posn is None else max_posn
        return lo // 18, hi // 18

    def _apply_rows(self, dev):
        """Installs (or clears) this view's row filter on the shared device index."""
        if self.rows is None:
            if dev._rows_set:
                _lib.check(_lib.lib().sa_index_set_rows(dev.handle, None, 0))
                dev._rows_set = False
        else:
            _lib.check(_lib.lib().sa_index_set_rows(dev.handle, _lib.p_u64(self.rows), len(self.rows)))
            dev._rows_set = True

    def termfreqs(self, token: Union[List[str], str], slop: int = 0,
                  min_posn: Optional[int] = None, max_posn: Optional[int] = None) -> np.ndarray:
        token = self._check_token_arg(token)
        lo, hi = self._payload_bounds(min_posn, max_posn)
        dev = self._device()
        out = _pool.empty_f32(len(self))
        with self._shared["lock"]:
            self._apply_rows(dev)
            if isinstance(token, list):
                ids = np.asarray([self._term_id(t) for t in token], dtype=np.uint32)
                _lib.check(_lib.lib().sa_phrase_freqs(dev.handle, _lib.p_u32(ids), len(ids), int(slop),
                                                      lo, hi, _lib.p_f32(out)))
            else:
                _lib.check(_lib.lib().sa_termfreqs(dev.handle, self._term_id(token), lo, hi, _lib.p_f32(out)))
        return out

    def docfreq(self, token: str) -> int:
        if not isinstance(token, str):
            raise TypeError("Expected a string")
        tid = self._term_id(token)
        if tid == _lib.NO_TERM:
            return 0
        if self.global_df is not None and self.rows is None:
            return np.uint64(self.global_df[tid])
        dev = self._device()
        df = ctypes.c_uint64(0)
        with self._shared["lock"]:
            if self.rows is None:
                _lib.check(_lib.lib().sa_docfreq(dev.handle, tid, ctypes.byref(df)))
            else:
                self._apply_rows(dev)
                _lib.check(_lib.lib().sa_docfreq_rows(dev.handle, tid, ctypes.byref(df)))
        return np.uint64(df.value)

    def doclengths(self) -> np.ndarray:
        if self.rows is None:
            return self.doc_lens
        return self.doc_lens[self.rows.astype(np.int64)]

    def _view_bm25_doc_lens(self) -> np.ndarray:
        """The doc lengths BM25 uses on this view: the stepped-slice quirk's (see __getitem__) or the view's own.
        Shared by .score and .search_topk so that the two rank with the same lengths."""
        dl = getattr(self, "_bm25_doc_lens", None)
        return np.ascontiguousarray(self.doclengths()) if dl is None else dl

    def score(self, token: Union[str, List[str]], similarity: Similarity = default_bm25, slop: int = 0,
              min_posn: Optional[int] = None, max_posn: Optional[int] = None) -> np.ndarray:
        """Score each doc (reference postings.py:652-680).  With a bm25_similarity the whole
        chain postings -> tf -> BM25 is one fused kernel; any other callable receives the
        GPU-computed dense tf vector like the reference."""
        token = self._check_token_arg(token)
        tokens_l = [token] if isinstance(token, str) else token
        all_dfs = np.asarray([self.docfreq(t) for t in tokens_l])
        if not isinstance(similarity, Bm25Similarity):
            tfs = self.termfreqs(token, min_posn=min_posn, max_posn=max_posn, slop=slop)
            return similarity(tfs, all_dfs, self.doclengths(), self.avg_doc_length, self.corpus_size)
        lo, hi = self._payload_bounds(min_posn, max_posn)
        if self.rows is not None:
            # sliced array: tf on the filtered postings (FilteredPosns), then BM25 over the slice's
            # rows with the slice's doc lengths -- both on the GPU (reference postings.py:674-680)
            from . import ops
            tfs = self.termfreqs(token, min_posn=min_posn, max_posn=max_posn, slop=slop)
            if self.avg_doc_length == 0:
                return np.zeros_like(tfs)
            idf = compute_idf(self.corpus_size, all_dfs)
            return ops.bm25_score(tfs, self._view_bm25_doc_lens(), self.avg_doc_length, idf, similarity.k1,
                                  similarity.b, device=self.device)
        out = _pool.empty_f32(len(self))
        if self.avg_doc_length == 0:
            out[:] = 0
            return out
        idf = compute_idf(self.corpus_size, all_dfs)
        dev = self._device()
        with self._shared["lock"]:
            self._apply_rows(dev)
            if isinstance(token, list):
                ids = np.asarray([self._term_id(t) for t in token], dtype=np.uint32)
                _lib.check(_lib.lib().sa_score_phrase(dev.handle, _lib.p_u32(ids), len(ids), int(slop), idf,
                                                      self.avg_doc_length, similarity.k1, similarity.b,
                                                      lo, hi, _lib.p_f32(out)))
            else:
                _lib.check(_lib.lib().sa_score_term(dev.handle, self._term_id(token), idf, self.avg_doc_length,
                                                    similarity.k1, similarity.b, lo, hi, _lib.p_f32(out)))
        return out

    def positions(self, token: str, key=None) -> List[np.ndarray]:
        """Positions of a term per doc (reference postings.py:682-687): index-time decode, host."""
        tid = self.term_dict.get_term_id(token)
        docs = np.arange(len(self.doc_lens)) if self.rows is None else self.rows.astype(np.int64)
        if key is not None:
            docs = docs[key]
        w = self.host.term_words(tid)
        out = []
        for d in np.atleast_1d(docs):
            d = int(d) + self.doc_base                       # words carry ABSOLUTE doc ids (shards)
            a = np.searchsorted(w, np.uint64(d) << np.uint64(36))
            b = np.searchsorted(w, np.uint64(d + 1) << np.uint64(36))
            out.append(decode_positions(w[a:b]))
        return out

    # -------------------------------------------------------------------- features
    def set_feature(self, name: str, values) -> None:
        """Registers a per-document numeric column -- popularity, vote count, recency, a quality score -- for
        query.Feature clauses of search_topk and solr.fields_topk.  values: one finite number >= 0 per doc of the
        array (on a shard, per row of the shard), rounded once to float32; 0 means the doc lacks the feature.  Another
        length, NaN, inf or a negative value is a ValueError, a non-numeric dtype a TypeError, both before any device
        work.  Setting a name again replaces its values; at most 16 names per index.  Refused (ValueError) on a view,
        whose positions are not the index's docs.  The values live with the index (copies and pickles carry them) and
        go to the device when it is first used, or at once if it already is."""
        from .query import SA_MAX_FEATURES
        if not isinstance(name, str):
            raise TypeError(f"a feature name is a str, not {name!r}")
        if self.rows is not None:
            raise ValueError("set_feature on a view (arr[mask]) is not supported: set it on the whole array")
        v = np.asarray(values)
        if v.dtype.kind not in "iuf":
            raise TypeError(f"feature values are numbers (int or float), not dtype {v.dtype}")
        if v.shape != (self.host.n_docs,):
            raise ValueError(f"a feature has one value per doc: shape ({self.host.n_docs},), not {v.shape}")
        with np.errstate(over="ignore"):
            v32 = np.ascontiguousarray(v, dtype=np.float32).copy()
        if not (np.all(np.isfinite(v)) and np.all(np.isfinite(v32))) or np.any(v < 0):
            raise ValueError(f"feature values are finite and >= 0 (in float32): {name!r}")
        feats = self.host.features
        if name not in feats and len(feats) >= SA_MAX_FEATURES:
            raise ValueError(f"an index holds at most {SA_MAX_FEATURES} features")
        with self._shared["lock"]:
            feats[name] = v32
            if self._shared["dev"] is not None:
                self._shared["dev"].sync_features(self.host)

    def set_facet(self, name, codes, n_buckets=None) -> None:
        """Registers a per-document category column -- a language, a decade, a genre -- whose counts search_topk and
        solr.fields_topk return with `facets=`.  codes: one integer per doc of the array (on a shard, per row of the
        shard); a code in [0, n_buckets) is the doc's bucket, -1 means the doc has no value.  n_buckets defaults to
        max(codes) + 1, at least 1, and may be at most 1,024.  A non-integer dtype is a TypeError; another length, a
        code below -1 or >= n_buckets, more than 1,024 buckets or more than 8 names per index a ValueError, all before
        any device work.  Setting a name again replaces it.  Refused (ValueError) on a view, whose positions are not
        the index's docs.  The codes live with the index (copies and pickles carry them) and go to the device when it
        is first used, or at once if it already is."""
        from .query import SA_FACET_MAX_BUCKETS, SA_MAX_FACETS
        if not isinstance(name, str):
            raise TypeError(f"a facet name is a str, not {name!r}")
        if self.rows is not None:
            raise ValueError("set_facet on a view (arr[mask]) is not supported: set it on the whole array")
        c = np.asarray(codes)
        if c.dtype.kind not in "iu":
            raise TypeError(f"facet codes are integers, not dtype {c.dtype}")
        if c.shape != (self.host.n_docs,):
            raise ValueError(f"a facet has one code per doc: shape ({self.host.n_docs},), not {c.shape}")
        if n_buckets is None:
            n_buckets = max(int(c.max()) + 1 if len(c) else 1, 1)
        if isinstance(n_buckets, bool) or not isinstance(n_buckets, numbers.Integral):
            raise TypeError(f"n_buckets is an int, not {n_buckets!r}")
        n_buckets = int(n_buckets)
        if not 1 <= n_buckets <= SA_FACET_MAX_BUCKETS:
            raise ValueError(f"a facet has 1 to {SA_FACET_MAX_BUCKETS} buckets, not {n_buckets}")
        if len(c) and (int(c.min()) < -1 or int(c.max()) >= n_buckets):
            raise ValueError(f"facet codes are -1 (no value) or in [0, {n_buckets}): {name!r} holds "
                             f"[{int(c.min())}, {int(c.max())}]")
        facets = self.host.facets
        if name not in facets and len(facets) >= SA_MAX_FACETS:
            raise ValueError(f"an index holds at most {SA_MAX_FACETS} facets")
        with self._shared["lock"]:
            facets[name] = (np.ascontiguousarray(c, dtype=np.int32).copy(), n_buckets)
            if self._shared["dev"] is not None:
                self._shared["dev"].sync_facets(self.host)

    def set_group(self, name, codes) -> None:
        """Registers a per-document group column -- a franchise, a parent SKU, a site -- that search_topk and
        solr.fields_topk collapse on with `collapse=`, returning one document per group.  codes: one integer per doc
        of the array (on a shard, per row of the shard) in [-1, 2^31 - 1); -1 means the doc belongs to no group, and
        each such doc is a group of its own.  A non-integer dtype is a TypeError; another length, a code out of range
        or more than 4 names per index a ValueError, all before any device work.  Setting a name again replaces it.
        Refused (ValueError) on a view, whose positions are not the index's docs.  The codes live with the index
        (copies, pickles and shard slices carry them) and go to the device when it is first used, or at once if it
        already is."""
        from .query import SA_MAX_GROUPS
        if not isinstance(name, str):
            raise TypeError(f"a group name is a str, not {name!r}")
        if self.rows is not None:
            raise ValueError("set_group on a view (arr[mask]) is not supported: set it on the whole array")
        c = np.asarray(codes)
        if c.dtype.kind not in "iu":
            raise TypeError(f"group codes are integers, not dtype {c.dtype}")
        if c.shape != (self.host.n_docs,):
            raise ValueError(f"a group column has one code per doc: shape ({self.host.n_docs},), not {c.shape}")
        if len(c) and (int(c.min()) < -1 or int(c.max()) >= 2 ** 31 - 1):
            raise ValueError(f"group codes are -1 (no group) or in [0, 2^31 - 1): {name!r} holds "
                             f"[{int(c.min())}, {int(c.max())}]")
        groups = self.host.groups
        if name not in groups and len(groups) >= SA_MAX_GROUPS:
            raise ValueError(f"an index holds at most {SA_MAX_GROUPS} group columns")
        with self._shared["lock"]:
            groups[name] = np.ascontiguousarray(c, dtype=np.int32).copy()
            if self._shared["dev"] is not None:
                self._shared["dev"].sync_groups(self.host)

    def _group_slot(self, name):
        """The slot of group column `name` on this array's index; ValueError if it is not set."""
        names = list(self.host.groups)
        if name not in names:
            raise ValueError(f"group column {name!r} is not set on this array (set_group); set: {names}")
        return names.index(name)

    def _facet_slot(self, name):
        """(slot, n_buckets) of facet `name` on this array's index; ValueError if it is not set."""
        names = list(self.host.facets)
        if name not in names:
            raise ValueError(f"facet {name!r} is not set on this array (set_facet); set: {names}")
        return names.index(name), self.host.facets[name][1]

    def _feature_slot(self, name):
        """The slot of feature `name` on this array's index; ValueError if it is not set."""
        names = list(self.host.features)
        if name not in names:
            raise ValueError(f"feature {name!r} is not set on this array (set_feature); set: {names}")
        return names.index(name)

    # -------------------------------------------------- batched, HBM-resident path
    def search_topk(self, queries, k=10, similarity: Similarity = default_bm25, slop=0, where=None, facets=None,
                    rescore=None, collapse=None):
        """queries: list of str (term) or list[str] (phrase).  Returns (docs uint32[Q,k],
        scores float32[Q,k]): per query the k best scores > 0, by score descending then id ascending, empty
        slots NO_DOC / 0.  Scores never leave HBM except the top-k (sa_score_batch_topk).

        k: 1 <= k <= query.TOPK_MAX (1,024), e.g. k=1000 for first-stage retrieval ahead of a reranker; another k is a
        ValueError before any device work.  Above 32 every tile keeps its own exact top k, so the first k' results of
        a call are bit for bit those of the same call at k'.

        On a view (arr[mask], arr[a:b], arr[::s], arr.take(idx), a view of a view) the result is the top k of
        `view.score(q, similarity=similarity, slop=slop)`, and the returned ids are POSITIONS IN THE VIEW
        (0 .. len(view) - 1, the index space of view.score), not the parent's doc ids.  Views of a sharded array
        (built with a comm or a global_df) raise ValueError: their document frequencies would need a sum over
        the ranks.

        similarity: bm25_similarity, bm25_impact, bm25_legacy_similarity or classic_similarity; any other
        callable raises TypeError.  Under the last three the result is, bit for bit, the top k of
        `.score(q, similarity=similarity, slop=slop)` on the same array or view, and the scores have its dtype
        (float32 for bm25_impact, float64 for the other two, also where .score returns float32 zeros because
        avg_doc_length is 0); +inf ranks, NaN never does.

        queries may also hold boolean queries (query.Or / query.And), mixed freely with the others: per boolean query
        the top k of s = .score(c0) + .score(c1) + ... (float32, clause order) over the docs where s > 0 and at least
        mm clauses score > 0 (sa_score_batch_topk_bool).  They run on the whole array under bm25_similarity only: on
        a view they raise NotImplementedError, under another similarity TypeError.

        query.Bool(must, should, filter, must_not, mm) and query.Boost(clause, weight) clauses are accepted the same
        way: s = w0 * .score(c0) + w1 * .score(c1) + ... over must + should (float32, each product rounded), ranked
        where s > 0, every must and filter clause scores > 0, no must_not clause does and at least mm should clauses
        do.  An Or / And whose weights are all 1 runs exactly as above.

        query.DisMax(clauses, tie) is accepted as a clause of these, and as a query of its own (Bool(should=[it])):
        one clause scoring d = max_j v_j + (sum_j v_j - max_j v_j) * tie over its members' v_j = w_j * .score(c_j),
        matched where any member scores > 0 -- synonyms as
        DisMax(["film", "movie"], tie=0.1).  Its members need k1 > 0 and 0 <= b < 1 (ValueError otherwise).

        An Or / And / Bool may be a clause of another, at any depth (Or([And(["star", "wars"]), And(["star", "trek"])])):
        it scores what it would rank as a query of its own and matches where that is > 0; see query.Or.

        query.Feature, query.Range and query.In are clauses over the array's columns (set_feature, set_facet): a
        per-doc signal added to the score, a numeric range and a set of facet codes, the last two scoring 1 where they
        match.  Bool(must=[Or(["star", "wars"])], filter=[Range("year", gte=1977, lt=1990), In("lang", [en, fr])])
        ranks as the same query with the matching `where=` mask, evaluated per doc on the device with no mask copied;
        unlike a mask they also work under must_not, should (a boosted language or recency preference) and in nested
        queries.  Each is refused as a query of its own (TypeError), as a DisMax member, and for a name not set or an
        In code past the facet's buckets (ValueError), before any device work.

        where: a document filter -- a boolean array-like (a boolean pd.Series too) of shape (len(self),), one mask for
        the batch, or (len(queries), len(self)), one per query -- ranks each query only among the docs its mask
        allows, as Lucene's filter context does: the result is the top k of np.where(mask_q, S_q, 0), S_q being what
        the call without `where` ranks (.score, or the boolean composition), under the same rule, ids and dtypes.
        The mask never changes a score: idf, document frequencies, avgdl and doc lengths stay those of the whole
        array (of the view, on a view).  On a view it indexes the view's positions, on a shard the shard's rows.
        A dtype other than bool raises TypeError and another shape ValueError, before any device work; every input
        refused without `where` is refused the same way with it.  Plain BM25 queries on the unsliced array rank as
        one-clause Or queries (sa_score_batch_topk_bool); the others take sa_score_batch_topk_sim.  A
        mask per query costs len(self) / 8 bytes of host-to-device copy and device memory per query.

        facets: hit and facet counts, as Lucene's totalHits and Elasticsearch's terms aggregations return them with
        the top k.  A list of at most 4 distinct facet names (set_facet), possibly empty, returns
        (docs, scores, hits), hits a Hits: per query q, hits.total[q] == np.count_nonzero(S_q) and
        hits.facets[name][q] == np.bincount(codes[(S_q > 0) & (codes >= 0)], minlength=n_buckets), S_q being the
        dense vector the call without `facets` ranks from (`where` applied).  docs and scores are bit for bit those of
        the call without `facets`.  The counts are made where the device fold decides which docs rank; only the
        counts come back.  Every query form the boolean path takes is accepted, with or without `where`; plain
        queries then rank as one-clause Or queries through the boolean fold, which is slower than the term scan
        that ranks them without `facets`.  On a view (NotImplementedError), under another similarity than
        bm25_similarity (TypeError), and for a name not set, a name given twice or more than 4 names (ValueError),
        the call is refused before any device work.  On a shard the counts are the shard's own docs.  facets=None
        (the default) returns (docs, scores) as above.

        rescore: a query.Rescore re-ranks each query's top window by a second query scored at the window's docs
        (score_docs), Elasticsearch's `rescore`: the call above at k=rescore.window, with `where` and `facets`, then
        the top k by c = float32(query_weight * s1) + float32(rescore_weight * s2) (c desc, id asc); the scores
        returned are c, the hits pass 1's.  A rescore with another number of queries, a window outside [k, 1,024],
        a view or a similarity other than bm25_similarity is refused before any device work.  On a shard the window
        is the shard's own top window.

        collapse: the name of a group column (set_group) to return one document per group, as Elasticsearch's
        `collapse` and Solr's collapsing query parser (nullPolicy=expand) do.  Per query, of the docs with S_q > 0
        (S_q as above, `where` applied) each group's leader is its doc with the highest S_q, ties to the lower id; a
        doc whose code is -1 is a group of its own; the result is the k best leaders by (score desc, id asc), with the
        ids and float32 scores the call without `collapse` returns for them, and NO_DOC / 0 past the last group.  So
        the first k' results at k are those at k', and score_docs at the returned docs returns their scores.  With
        `facets`, hits count documents, not groups (Elasticsearch's hits.total under collapse): they equal the hits
        of the call without `collapse`.  Every query form the boolean path takes is accepted, with or without `where`
        and `facets`; plain queries then rank as one-clause Or queries through the boolean fold.  Each tile of 8,192
        docs keeps its exact k best leaders on the device, so the result is exact whatever the group sizes.  A name
        that is not a str (TypeError), a name not set (ValueError), a view (NotImplementedError), a similarity other
        than bm25_similarity (TypeError) and `collapse` with `rescore` (ValueError) are refused before any device
        work.  On a shard the groups are collapsed over the shard's own docs: shards are not merged with
        deduplication."""
        from .query import DISMAX, NESTED, OCCUR, OR_AND, bool_form, check_k, has_dismax, has_field, is_boolean
        k = check_k(k)
        if collapse is not None:
            if rescore is not None:
                raise ValueError("collapse cannot be combined with rescore")
            if not isinstance(collapse, str):
                raise TypeError(f"collapse is the name of a group column (a str), not {collapse!r}")
        if rescore is not None:
            return self._search_topk_rescore(queries, k, similarity, slop, where, facets, rescore)
        queries = list(queries)
        _refuse_column_queries(queries)
        if facets is not None:
            facets = check_facet_keys(facets, "facet names")
        bits = None if where is None else pack_where(where, len(self), len(queries))
        kind = np.asarray([bool_form(q) if is_boolean(q) else 0 for q in queries])     # 0: plain
        if facets is None and collapse is None and not kind.any():
            self._check_topk_similarity(similarity)
            if self.rows is not None or not isinstance(similarity, Bm25Similarity):
                return self._search_topk_sim(queries, k, similarity, slop, bits)
            if bits is None:
                return self._search_topk_plain(queries, k, similarity, slop)
        else:                       # the boolean path's refusals
            if any(has_field(q) for q in queries if is_boolean(q)):
                raise ValueError("a Field clause names a DataFrame column: run queries over columns with "
                                 "solr.fields_topk(frame, queries), not SearchArray.search_topk")
            if self.rows is not None:
                raise NotImplementedError("boolean queries on a view (arr[mask]) are not supported yet; "
                                          "compose .score() on the view")
            if not isinstance(similarity, Bm25Similarity):
                raise TypeError(f"boolean queries support bm25_similarity only, not {similarity!r}")
            if collapse is not None:
                self._group_slot(collapse)
        hits = None if facets is None else Hits(np.zeros(len(queries), dtype=np.int64), {
            f: np.zeros((len(queries), self._facet_slot(f)[1]), dtype=np.int64) for f in facets})
        if any(has_dismax(q) for q, kd in zip(queries, kind) if kd >= DISMAX):      # k1 / b before any device work
            _check_dismax([0], ["DisMax member"], [0], [self], [similarity])
        # one call per form present, so that each runs the lightest instance that scores it; results in query order
        docs = np.empty((len(queries), k), dtype=np.uint32)
        scores = np.empty((len(queries), k), dtype=np.float32)
        for kd in (0, OR_AND, OCCUR, DISMAX, NESTED):
            sel = kind == kd
            if not sel.any():
                continue
            part = [q for q, s in zip(queries, sel) if s]
            if kd == 0 and bits is None and facets is None and collapse is None:
                docs[sel], scores[sel] = self._search_topk_plain(part, k, similarity, slop)
                continue
            out = self._search_topk_bool(part, k, similarity, slop, _where_part(bits, sel), facets, collapse)
            docs[sel], scores[sel] = out[:2]
            if hits is not None:
                hits.total[sel] = out[3].total
                for f in facets:
                    hits.facets[f][sel] = out[3].facets[f]
        return (docs, scores) if hits is None else (docs, scores, hits)

    def score_docs(self, queries, docs, slop=0, similarity: Similarity = default_bm25):
        """The value each query ranks each of its candidate docs with, the second stage after search_topk (reranker
        features, window rescoring): out[q, j] == S_q[docs[q, j]], S_q the dense vector search_topk ranks query q from
        (.score for a term or phrase, the boolean composition for an Or / And / Bool / DisMax or nested query with
        Feature, Range and In clauses), +0 where the doc does not rank.  So score_docs(queries, search_topk(queries, k)[0]) returns
        search_topk's scores bit for bit.  It replaces `arr.score(q)[docs[q]]` without a dense row per query: every
        (query, doc) is evaluated on the device from the index's lists (sa_score_docs_bool); only phrase clauses build
        their count rows, as search_topk does.

        docs: an integer array of shape (len(queries), K), ids as search_topk returns them (global doc ids on a
        shard), NO_DOC giving 0; duplicates and any order are allowed.  Returns float32 (len(queries), K).  Another
        dtype (TypeError), another shape or an id out of range (ValueError), a view (NotImplementedError) and a
        similarity other than bm25_similarity (TypeError) are refused before any device work."""
        from .query import Or, has_field, is_boolean
        queries = list(queries)
        _refuse_column_queries(queries)
        if any(has_field(q) for q in queries if is_boolean(q)):
            raise ValueError("a Field clause names a DataFrame column: score queries over columns with "
                             "solr.fields_score_docs(frame, queries, rows), not SearchArray.score_docs")
        self._check_score_docs(similarity)
        docs = check_docs(docs, len(queries), self.doc_base, len(self))
        if docs.size == 0:
            return np.zeros(docs.shape, dtype=np.float32)
        # plain queries as one-clause Or nodes, which score as .score does: one call at the batch's heaviest form
        nodes = [q if is_boolean(q) else Or([q]) for q in queries]
        with self._shared["lock"]:
            return self._prepare_bool(nodes, similarity).score_docs(docs, slop)

    def _check_score_docs(self, similarity):
        """score_docs' refusals of the array and the similarity (the boolean path's)."""
        if self.rows is not None:
            raise NotImplementedError("score_docs on a view (arr[mask]) is not supported yet; compose .score() on "
                                      "the view")
        if not isinstance(similarity, Bm25Similarity):
            raise TypeError(f"score_docs supports bm25_similarity only, not {similarity!r}")

    def _search_topk_rescore(self, queries, k, similarity, slop, where, facets, rescore):
        """search_topk with `rescore` (query.Rescore): pass 1 at k=rescore.window, score_docs of the rescore queries
        at its docs, then the combine and order of query.rescore_window; hits are pass 1's."""
        from .query import Rescore, rescore_window
        if not isinstance(rescore, Rescore):
            raise TypeError(f"rescore is a query.Rescore, not {rescore!r}")
        queries = list(queries)
        rescore.check(len(queries), k)
        self._check_score_docs(similarity)
        out = self.search_topk(queries, rescore.window, similarity, slop, where, facets)
        s2 = self.score_docs(rescore.queries, out[0], slop=rescore.slop, similarity=similarity)
        docs, scores = rescore_window(out[0], out[1], s2, rescore.query_weight, rescore.rescore_weight, k)
        return (docs, scores) + tuple(out[2:])

    @staticmethod
    def _check_topk_similarity(similarity):
        if not isinstance(similarity, (Bm25Similarity, Bm25Impact, Bm25Legacy, ClassicSimilarity)):
            raise TypeError("search_topk supports bm25_similarity, bm25_impact, bm25_legacy_similarity and "
                            f"classic_similarity, not {similarity!r}")

    def _search_topk_plain(self, queries, k, similarity, slop):
        """search_topk of plain queries under BM25 on the whole array, without a mask or counts: the term scan of
        sa_score_batch_topk."""
        terms, starts, idfs = self._topk_queries(queries, lambda dfs: compute_idf(self.corpus_size, dfs))
        idfs = np.asarray(idfs, dtype=np.float32)
        docs = np.empty((len(idfs), k), dtype=np.uint32)
        scores = np.empty((len(idfs), k), dtype=np.float32)
        dev = self._device()
        with self._shared["lock"]:
            _lib.check(_lib.lib().sa_score_batch_topk(dev.handle, _lib.p_u32(terms), _lib.p_u32(starts),
                                                      _lib.p_f32(idfs), len(idfs), int(slop),
                                                      self.avg_doc_length, similarity.k1, similarity.b, k,
                                                      _lib.p_u32(docs), _lib.p_f32(scores)))
        return docs, scores

    def _prepare_bool(self, queries, similarity, where=None, facets=None, collapse=None):
        """Boolean queries of any forms, or plain ones (a batch of their own) as one-clause Or nodes, which score
        exactly as .score(q, slop=slop), as one sa_score_batch_topk_bool call flattened for the heaviest form among
        them (query.bool_form, flatten_bool): a _PreparedBool.  where: a packed mask (pack_where).  facets: facet names
        (check_facet_keys) whose Hits the call returns.  collapse: a group column's name, collapsed on
        (sa_score_batch_topk_bool_collapse).  Call it, and run the call, with the lock held."""
        from .query import OR_AND, bool_form, flatten_bool, is_boolean
        batch = flatten_bool(queries, max((bool_form(q) for q in queries if is_boolean(q)), default=OR_AND))
        return _PreparedBool([self], [similarity], np.zeros(len(batch.clauses), dtype=np.uint32), queries, batch,
                             where, None if facets is None else [(f, 0, f) for f in facets],
                             group=None if collapse is None else (0, collapse))

    def _search_topk_bool(self, queries, k, similarity, slop, where=None, facets=None, collapse=None):
        """_prepare_bool's call, made with the lock held: (docs, scores, queries re-run exactly), and the Hits with
        facets."""
        with self._shared["lock"]:
            return self._prepare_bool(queries, similarity, where, facets, collapse).run(k, slop)

    def _topk_queries(self, queries, idf):
        """The queries as the batched top-k entries take them: term ids, start offsets and, per query, idf(dfs) of
        its tokens' document frequencies -- .docfreq's values, on a view the slice's from one sa_docfreq_rows_batch
        over the distinct known tokens (call it with the view's rows applied and the lock held)."""
        toks = [[q] if isinstance(q, str) else list(q) for q in queries]
        ids = {t: self._term_id(t) for ts in toks for t in ts}
        if self.rows is None:
            df = {t: self.docfreq(t) for t in ids}
        else:
            # .docfreq's values: np.uint64 for a known token, 0 for an unknown one
            known = [t for t, tid in ids.items() if tid != _lib.NO_TERM]
            dfs = np.zeros(len(known), dtype=np.uint64)
            if known:
                tids = np.asarray([ids[t] for t in known], dtype=np.uint32)
                _lib.check(_lib.lib().sa_docfreq_rows_batch(self._device().handle, _lib.p_u32(tids), len(tids),
                                                            _lib.p_u64(dfs)))
            df = dict(zip(known, dfs))
        terms, starts, idfs = [], [0], []
        for ts in toks:
            terms.extend(ids[t] for t in ts)
            starts.append(len(terms))
            idfs.append(idf(np.asarray([df.get(t, 0) for t in ts])))
        return np.asarray(terms, dtype=np.uint32), np.asarray(starts, dtype=np.uint32), idfs

    def _search_topk_sim(self, queries, k, similarity, slop, where=None):
        """search_topk on a view, and under bm25_impact, bm25_legacy_similarity or classic_similarity on any array
        (sa_score_batch_topk_sim): the counts, document frequencies, doc lengths, avgdl and corpus size .score
        uses, with the idf computed here, on the host, from the same dfs.  where: a packed mask over the positions
        (pack_where)."""
        if self.rows is not None and (self.comm is not None or self.global_df is not None):
            raise ValueError("search_topk on a view of a sharded SearchArray is not supported: the slice's document "
                             "frequencies would need a sum over the ranks; use .score() on the view")
        bm25 = isinstance(similarity, Bm25Similarity)
        # BM25 ranks a view with the doc lengths .score's BM25 uses there (the stepped-slice quirk)
        dl = np.ascontiguousarray(self._view_bm25_doc_lens(), dtype=np.float32) if bm25 else None
        dev = self._device()
        with self._shared["lock"]:
            self._apply_rows(dev)
            if bm25:        # the float32 idf .score's BM25 takes
                terms, starts, idfs = self._topk_queries(queries, lambda dfs: compute_idf(self.corpus_size, dfs))
                idfs = np.asarray(idfs, dtype=np.float32)
            else:
                terms, starts, idfs = self._topk_queries(
                    queries, lambda dfs: float(similarity._idf(dfs, self.corpus_size)))
            idfs = np.asarray(idfs, dtype=np.float64)
            docs = np.full((len(idfs), k), _lib.NO_DOC, dtype=np.uint32)
            scores = np.zeros((len(idfs), k), dtype=np.float64)
            dbl = ctypes.POINTER(ctypes.c_double)
            p_w, stride = _where_args(where)
            _lib.check(_lib.lib().sa_score_batch_topk_sim(
                dev.handle, similarity.kind, _lib.p_u32(terms), _lib.p_u32(starts), idfs.ctypes.data_as(dbl),
                len(idfs), int(slop), None if dl is None else _lib.p_f32(dl), float(self.avg_doc_length),
                float(similarity.k1), float(similarity.b), k, p_w, len(self), stride, _lib.p_u32(docs),
                scores.ctypes.data_as(dbl)))
        return docs, scores.astype(similarity.out_dtype, copy=False)
