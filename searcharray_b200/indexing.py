"""Host-side index build (numpy).  Produces the upload format of the GPU index.

Mirrors what the reference builds at index time (searcharray/indexing.py:235-295: tokenize ->
(term, doc, posn) triples -> stable sort by term -> roaringish encode -> ArrayDict) and the
state SearchArray.index injects (searcharray/postings.py:293-299): term dictionary, per-term
posting words, doc_lens, avg_doc_length.  Tokenising is Python-bound and stays on the host
(out of scope for kernels: SURVEY.md section 2 rows 12-13).
"""
import numpy as np

from .roaringish import MAX_POSN, encode_grouped


class TermMissingError(KeyError):
    """reference searcharray/term_dict.py:4-7"""


class TermDict:
    """str <-> id, ids in first-seen order (reference searcharray/term_dict.py:10-59)."""

    def __init__(self):
        self.term_to_ids = {}
        self.id_to_terms = []

    def add_term(self, term):
        tid = self.term_to_ids.get(term)
        if tid is None:
            tid = len(self.id_to_terms)
            self.term_to_ids[term] = tid
            self.id_to_terms.append(term)
        return tid

    def get_term_id(self, term):
        try:
            return self.term_to_ids[term]
        except KeyError:
            raise TermMissingError(f"Term {term} not present in dictionary. Reindex to add.")

    def get_term(self, term_id):
        try:
            return self.id_to_terms[term_id]
        except IndexError:
            raise TermMissingError(f"Term at {term_id} not present in dictionary. Reindex to add.")

    def __len__(self):
        return len(self.id_to_terms)


class HostIndex:
    """Flat, upload-ready inverted index: the layout of ArrayDict.data + metadata
    (reference searcharray/phrase/memmap_arrays.py:15-53) for every term id."""

    def __init__(self, words, term_offsets, term_lengths, doc_lens, term_dict=None, avg_doc_length=None):
        self.words = np.ascontiguousarray(words, dtype=np.uint64)
        self.words_file = None
        self.term_offsets = np.ascontiguousarray(term_offsets, dtype=np.uint64)
        self.term_lengths = np.ascontiguousarray(term_lengths, dtype=np.uint64)
        self.doc_lens = np.ascontiguousarray(doc_lens, dtype=np.float32)
        self.term_dict = term_dict
        # np.mean of a float32 array, like reference indexing.py:281
        if avg_doc_length is None:
            avg_doc_length = np.mean(self.doc_lens) if len(self.doc_lens) else 0
        self.avg_doc_length = avg_doc_length
        # per-doc feature columns (SearchArray.set_feature): name -> float32[n_docs]; a name's slot on the device
        # index is its position in this dict
        self.features = {}
        # per-doc facet columns (SearchArray.set_facet): name -> (int32[n_docs] codes, -1: no value; n_buckets); a
        # name's slot on the device index is its position in this dict
        self.facets = {}
        # per-doc group columns (SearchArray.set_group): name -> int32[n_docs] codes, -1: no group; a name's slot on
        # the device index is its position in this dict
        self.groups = {}

    # ---- on-disk posting words (reference phrase/memmap_arrays.py:145-208, MemoryMappedArrays): the words
    #      array written once to `<data_dir>/<n>.dat`, mapped back read-only; pickling stores the file name
    #      and the per-term slices, not the words (reference :196-208)
    def memmap(self, data_dir):
        import os
        os.makedirs(data_dir, exist_ok=True)
        filename = os.path.join(data_dir, f"{len(os.listdir(data_dir))}.dat")     # create_filename, :8-13
        with open(filename, "wb") as f:
            self.words.tofile(f)
        self.words_file = filename
        self._map_words()
        return filename

    def _map_words(self):
        n = int(np.sum(self.term_lengths))
        self.words = np.memmap(self.words_file, dtype=np.uint64, mode="r", shape=(n,)) if n else np.empty(0, dtype=np.uint64)

    def __getstate__(self):
        st = dict(self.__dict__)
        if st.get("words_file"):
            st["words"] = None
        return st

    def __setstate__(self, st):
        self.__dict__.update(st)
        self.__dict__.setdefault("features", {})
        self.__dict__.setdefault("facets", {})
        self.__dict__.setdefault("groups", {})
        if st.get("words_file"):
            self._map_words()

    @property
    def n_terms(self):
        return len(self.term_offsets)

    @property
    def n_docs(self):
        return len(self.doc_lens)

    def term_words(self, term_id):
        o, n = int(self.term_offsets[term_id]), int(self.term_lengths[term_id])
        return self.words[o:o + n]

    def shard(self, doc_lo, doc_hi):
        """Doc-range shard [doc_lo, doc_hi): every term's sub-list (found by searching the
        doc-id key, like RoaringishEncoder.key_partition, reference roaringish.py:227-243),
        doc ids kept absolute."""
        lo_key, hi_key = np.uint64(doc_lo) << np.uint64(36), np.uint64(doc_hi) << np.uint64(36)
        parts, offs, lens = [], [], []
        total = 0
        for t in range(self.n_terms):
            w = self.term_words(t)
            a, b = np.searchsorted(w, lo_key), np.searchsorted(w, hi_key)
            parts.append(w[a:b])
            offs.append(total)
            lens.append(b - a)
            total += b - a
        words = np.concatenate(parts) if parts else np.empty(0, dtype=np.uint64)
        out = HostIndex(words, offs, lens, self.doc_lens[doc_lo:doc_hi], self.term_dict, self.avg_doc_length)
        out.features = {name: v[doc_lo:doc_hi].copy() for name, v in self.features.items()}
        out.facets = {name: (c[doc_lo:doc_hi].copy(), nb) for name, (c, nb) in self.facets.items()}
        out.groups = {name: c[doc_lo:doc_hi].copy() for name, c in self.groups.items()}
        return out


def build_index(array, tokenizer, truncate=False, gpu_build=None):
    """Strings -> HostIndex (reference indexing.py:64-145,235-295 semantics: term ids in
    first-seen order, position = token index, doc_len = number of tokens).  Tokenising is a Python loop
    and stays on the host; with `gpu_build=<device>` the sort + roaringish encode of the (term, doc, posn)
    triples runs on that GPU (sa_op_build_index, SURVEY 8f-4), otherwise in numpy."""
    term_dict = TermDict()
    all_terms, all_docs, all_posns = [], [], []
    doc_lens = np.zeros(len(array), dtype=np.float32)
    limit = MAX_POSN if truncate else None
    for doc_id, doc in enumerate(array):
        toks = tokenizer(doc)
        ids = np.fromiter((term_dict.add_term(t) for t in toks), dtype=np.int64)[:limit]
        n = len(ids)
        doc_lens[doc_id] = n
        if n:
            all_terms.append(ids)
            all_docs.append(np.full(n, doc_id, dtype=np.int64))
            all_posns.append(np.arange(n, dtype=np.int64))
    if np.any(doc_lens > MAX_POSN):
        raise ValueError(f"Document length exceeds maximum of {MAX_POSN}")
    n_terms = len(term_dict)
    if all_terms:
        terms = np.concatenate(all_terms)
        docs = np.concatenate(all_docs)
        posns = np.concatenate(all_posns)
        if gpu_build is not None:
            return _build_on_device(terms, docs, posns, n_terms, doc_lens, term_dict, gpu_build)
        order = np.argsort(terms, kind="stable")       # docs/posns already ascending
        words, uniq, offs, lens = encode_grouped(terms[order], docs[order], posns[order])
    else:
        words = np.empty(0, dtype=np.uint64)
        uniq = np.empty(0, dtype=np.int64)
        offs = lens = np.empty(0, dtype=np.uint64)
    term_offsets = np.zeros(n_terms, dtype=np.uint64)
    term_lengths = np.zeros(n_terms, dtype=np.uint64)
    term_offsets[uniq] = offs
    term_lengths[uniq] = lens
    return HostIndex(words, term_offsets, term_lengths, doc_lens, term_dict)


def _build_on_device(terms, docs, posns, n_terms, doc_lens, term_dict, device):
    import ctypes
    from . import _lib
    t32 = np.ascontiguousarray(terms, dtype=np.uint32)
    d32 = np.ascontiguousarray(docs, dtype=np.uint32)
    p32 = np.ascontiguousarray(posns, dtype=np.uint32)
    words = np.empty(len(t32), dtype=np.uint64)
    offs = np.zeros(n_terms, dtype=np.uint64)
    lens = np.zeros(n_terms, dtype=np.uint64)
    n_words = ctypes.c_uint64(0)
    _lib.check(_lib.lib().sa_op_build_index(_lib.p_u32(t32), _lib.p_u32(d32), _lib.p_u32(p32), len(t32), n_terms,
                                            int(device), _lib.p_u64(words), ctypes.byref(n_words),
                                            _lib.p_u64(offs), _lib.p_u64(lens)))
    return HostIndex(words[:n_words.value].copy(), offs, lens, doc_lens, term_dict)


def index_from_term_postings(term_names, term_words_list, doc_lens, avg_doc_length=None):
    """Inject pre-encoded postings (synthetic corpora): one sorted word list per term."""
    td = TermDict()
    offs, lens, total = [], [], 0
    for name, w in zip(term_names, term_words_list):
        td.add_term(name)
        offs.append(total)
        lens.append(len(w))
        total += len(w)
    words = np.concatenate(term_words_list) if term_words_list else np.empty(0, dtype=np.uint64)
    return HostIndex(words, offs, lens, doc_lens, td, avg_doc_length)
