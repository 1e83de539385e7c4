"""Solr-style edismax over a DataFrame of SearchArray columns -- host mirror of the reference's
`searcharray.solr` (solr.py:10-355) with the vector arithmetic on the GPU.

The query parsing, the mm mini-language and the explain string are host-side string work, as in
the reference.  Every score vector -- the per-(term, field) BM25 vectors, the phrase-phase vectors
of pf / pf2 / pf3 on the arrays sliced to the qf matches, and the combined vector -- is produced and
combined in HBM through the `sa_multi_*` entry points (include/searcharray_b200.h); only the final
vector (`edismax`) or its top-k (`edismax_topk`) comes back.  There is no CPU fallback: a custom
(non-BM25) similarity or a sliced frame still runs every `.score` on the GPU and only the final
element-wise combination in numpy, the way the reference composes it.
"""
import ctypes
import re
import threading
import weakref
from typing import Dict, List, Optional, Tuple, Union

import numpy as np
import pandas as pd

from . import _lib
from .postings import SearchArray, _check_dismax, _PreparedBool, check_docs, check_facet_keys, pack_where
from .similarity import Bm25Similarity, Similarity, compute_idf, default_bm25


# --------------------------------------------------------------------------- parsing
def parse_min_should_match(num_clauses: int, spec: str) -> int:
    """Solr's `mm` (reference solr.py:10-59): ints, negatives, percentages, `n<spec` conditionals."""
    def as_int(text):
        try:
            return int(text)
        except ValueError:
            raise ValueError("Invalid 'mm' spec. Expecting an integer.")

    spec = spec.strip()
    if "<" in spec:
        result = num_clauses
        for clause in re.sub(r"\s*<\s*", "<", spec).split():
            bound, sep, rest = clause.partition("<")
            if not sep:
                raise ValueError("Invalid 'mm' spec: '" + clause + "'. Expecting values before and after '<'")
            if num_clauses <= as_int(bound):
                return result
            result = parse_min_should_match(num_clauses, rest)
        return result
    if "%" in spec:
        calc = (num_clauses * as_int(spec[:-1])) * (1 / 100)
        result = num_clauses + int(calc) if calc < 0 else int(calc)
    else:
        calc = as_int(spec)
        result = num_clauses + calc if calc < 0 else calc
    return min(num_clauses, max(result, 0))


def parse_field_boosts(field_lists: Optional[List[str]]) -> dict:
    """`["title^2", "body"]` -> {"title": 2.0, "body": None} (reference solr.py:62-74)."""
    out = {}
    for spec in field_lists or []:
        parts = spec.split("^")
        out[parts[0]] = None if len(parts) == 1 else float(parts[1])
    return out


def get_field(frame, field) -> SearchArray:
    if field not in frame.columns:
        raise ValueError(f"Field {field} not in dataframe")
    if not isinstance(frame[field].array, SearchArray):
        raise ValueError(f"Field {field} is not a searcharray field")
    return frame[field].array


def parse_query_terms(frame: pd.DataFrame, query: str, query_fields: List[str]):
    """Tokenise the query with every field's own tokenizer (reference solr.py:85-114)."""
    search_terms: Dict[str, List[str]] = {}
    num_search_terms, term_centric = 0, True
    for field in query_fields:
        toks = list(get_field(frame, field).tokenizer(query))
        search_terms[field] = toks
        if num_search_terms == 0:
            num_search_terms = len(toks)
        elif len(toks) != num_search_terms:
            term_centric = False
    return num_search_terms, search_terms, term_centric


def _boost_text(boost):
    return f"{boost}" if boost is not None else "1"


# ------------------------------------------------------------------- device multi handle
class _Multi:
    """An sa_multi over the device indexes of some fields (cached per field tuple)."""

    def __init__(self, arrays: List[SearchArray]):
        self.devs = [a._device() for a in arrays]          # keeps the field handles alive
        handles = (ctypes.c_void_p * len(self.devs))(*[d.handle for d in self.devs])
        self.handle = ctypes.c_void_p()
        _lib.check(_lib.lib().sa_multi_create(handles, len(self.devs), ctypes.byref(self.handle)))
        self.lock = threading.Lock()
        self._finalizer = weakref.finalize(self, _Multi._destroy, self.handle)

    @staticmethod
    def _destroy(handle):
        if handle and _lib._lib is not None:
            _lib._lib.sa_multi_destroy(handle)


# optional per-call wall-clock accounting (tools / bench diagnostics): set to a dict to collect
_TIMING = None


def _timed(name, fn, *args):
    if _TIMING is None:
        return fn(*args)
    import time
    t0 = time.perf_counter()
    rc = fn(*args)
    _TIMING[name] = _TIMING.get(name, 0.0) + time.perf_counter() - t0
    return rc


_multis: Dict[tuple, _Multi] = {}
_multis_lock = threading.Lock()


def _multi_for(arrays: List[SearchArray]) -> _Multi:
    key = tuple(id(a._device()) for a in arrays)
    with _multis_lock:
        m = _multis.pop(key, None)
        if m is None:
            while len(_multis) >= 16:                 # evict the least recently used; a caller still
                _multis.pop(next(iter(_multis)))      # holding it keeps it alive until it is done
            m = _Multi(arrays)
        _multis[key] = m                              # most recently used last
        return m


class _locked:
    """Holds the multi's lock AND every participating array's device lock (in a fixed order) for a whole
    edismax evaluation: the sa_multi_* calls keep intermediate state in the field indexes' scratch
    buffers, which a concurrent .score()/.termfreqs() on the same array would overwrite."""

    def __init__(self, multi: _Multi, arrays: List[SearchArray]):
        uniq = {id(a._shared["lock"]): a._shared["lock"] for a in arrays}
        self.locks = [multi.lock] + [uniq[k] for k in sorted(uniq)]

    def __enter__(self):
        for lk in self.locks:
            lk.acquire()
        return self

    def __exit__(self, *exc):
        for lk in reversed(self.locks):
            lk.release()
        return False


def _u32(values):
    return np.asarray(values, dtype=np.uint32)


def _f32(values):
    return np.asarray(values, dtype=np.float32)


class _Plan:
    """Everything edismax derives from its arguments before any scoring."""

    def __init__(self, frame, q, qf, mm, pf, pf2, pf3, tie, q_op, similarity):
        listify = lambda x: x if isinstance(x, list) else [x]
        self.query_fields = parse_field_boosts(listify(qf))
        self.phrase_fields = parse_field_boosts(listify(pf)) if pf else {}
        self.bigram_fields = parse_field_boosts(pf2) if pf2 else {}
        self.trigram_fields = parse_field_boosts(pf3) if pf3 else {}
        mm = "1" if mm is None else (f"{mm}" if isinstance(mm, int) else mm)
        self.mm = "100%" if q_op == "AND" else mm
        self.tie = tie
        if not isinstance(similarity, dict):
            similarity = {field: similarity for field in self.query_fields}
        for field in self.query_fields:
            similarity.setdefault(field, default_bm25)
        self.similarity = similarity
        self.names = list(self.query_fields)
        self.arrays = [get_field(frame, f) for f in self.names]
        self.num_terms, self.search_terms, self.term_centric = parse_query_terms(frame, q, self.names)

    def device_ok(self):
        from .query import ED_MAX_FIELDS, SA_MAX_PHRASE_TERMS
        return (all(isinstance(self.similarity[f], Bm25Similarity) for f in self.names)
                and all(a.rows is None for a in self.arrays)
                and len({len(a) for a in self.arrays}) == 1 and len(self.names) <= ED_MAX_FIELDS
                and all(len(t) <= SA_MAX_PHRASE_TERMS for t in self.search_terms.values()))

    # explain strings, reference solr.py:133-147, 160-178, 199-200, 219-220, 241-242
    def explain_qf(self):
        if self.term_centric:
            need = parse_min_should_match(self.num_terms, spec=self.mm)
            groups = ["(" + " | ".join(f"{f}:{self.search_terms[f][i]}^{_boost_text(b)}"
                                         for f, b in self.query_fields.items()) + ")"
                      for i in range(self.num_terms)]
            return "(" + " ".join(groups) + f")~{need}"
        parts = []
        for f, b in self.query_fields.items():
            toks = self.search_terms[f]
            need = min(parse_min_should_match(len(toks), spec=self.mm), len(toks))
            parts.append("((" + " ".join(f"{f}:{t}" for t in toks) + f")~{need})^{_boost_text(b)}")
        return " | ".join(parts)

    def phases(self):
        """[(phase name, [(field, boost, [phrase token lists], repeat_last)])] in reference order."""
        def grams(toks, n):
            return [toks[i:i + n] for i in range(len(toks) - n + 1)]
        out = []
        pf = [(f, b, [self.search_terms[f]], False) for f, b in self.phrase_fields.items()
              if len(self.search_terms[f]) >= 2]
        pf2 = [(f, b, grams(self.search_terms[f], 2), True) for f, b in self.bigram_fields.items()
               if len(self.search_terms[f]) >= 2]
        pf3 = [(f, b, grams(self.search_terms[f], 3), False) for f, b in self.trigram_fields.items()
               if len(self.search_terms[f]) >= 3]
        for name, items in (("pf", pf), ("pf2", pf2), ("pf3", pf3)):
            out.append((name, items))
        return out

    def phrase_rows(self):
        """field -> [(phase name, phrase no)]: the rows of the field's one sa_multi_phrases launch, in row order."""
        per_field: Dict[str, List[Tuple[str, int]]] = {}
        for name, items in self.phases():
            for f, _, phrases, _ in items:
                if f not in self.query_fields:
                    raise KeyError(f)                              # like the reference: pf fields must be in qf
                per_field.setdefault(f, []).extend((name, i) for i in range(len(phrases)))
        return per_field

    def phase_entries(self):
        """[(phase name, [(field, row, boost)])]: the entries of each phase's one sa_multi_add_phase call, in the
        reference's summation order (pf2 adds its last bigram twice); row indexes phrase_rows()[field]."""
        row_of = {(f, name, i): r for f, rows in self.phrase_rows().items() for r, (name, i) in enumerate(rows)}
        out = []
        for name, items in self.phases():
            entries = []
            for f, boost, phrases, repeat_last in items:
                order = list(range(len(phrases))) + ([len(phrases) - 1] if repeat_last else [])
                entries.extend((f, row_of[(f, name, i)], boost) for i in order)
            out.append((name, entries))
        return out

    def explain_phases(self):
        text = ""
        for _, items in self.phases():
            for f, b, phrases, _ in items:
                for ph in phrases:
                    text += f" ({f}:\"{' '.join(ph)}\")^{_boost_text(b)}"
        return text


def _run_device(plan: _Plan, multi: _Multi) -> _Multi:
    """qf phase + phrase phases into the multi's HBM-resident combined vector (caller holds `_locked`)."""
    L = _lib.lib()
    for arr in plan.arrays:                    # a sliced view of the same column may have left its row filter installed
        arr._apply_rows(arr._device())
    F = len(plan.names)
    n_terms, tids, idfs, boosts, has_boost, avgdl, k1, b, mms = [], [], [], [], [], [], [], [], []
    for f, arr in zip(plan.names, plan.arrays):
        toks = plan.search_terms[f]
        sim = plan.similarity[f]
        n_terms.append(len(toks))
        tids.extend(arr._term_id(t) for t in toks)
        idfs.extend(compute_idf(arr.corpus_size, np.asarray([arr.docfreq(t)])) for t in toks)
        boost = plan.query_fields[f]
        boosts.append(0.0 if boost is None else boost)
        has_boost.append(0 if boost is None else 1)
        avgdl.append(arr.avg_doc_length)
        k1.append(sim.k1)
        b.append(sim.b)
        if plan.term_centric:
            mms.append(parse_min_should_match(plan.num_terms, spec=plan.mm))
        else:
            mms.append(min(parse_min_should_match(len(toks), spec=plan.mm), len(toks)))
    n_matches = ctypes.c_uint64(0)
    a_nt, a_tid, a_idf = _u32(n_terms), _u32(tids if tids else [0]), _f32(idfs if idfs else [0])
    a_boost, a_hb, a_avgdl, a_k1, a_b, a_mm = _f32(boosts), _u32(has_boost), _f32(avgdl), _f32(k1), _f32(b), _u32(mms)
    _lib.check(_timed("qf", L.sa_multi_qf, multi.handle, 0 if plan.term_centric else 1, _lib.p_u32(a_nt), _lib.p_u32(a_tid),
                             _lib.p_f32(a_idf), _lib.p_f32(a_boost), _lib.p_u32(a_hb), _lib.p_f32(a_avgdl),
                             _lib.p_f32(a_k1), _lib.p_f32(a_b), _lib.p_u32(a_mm), float(plan.tie),
                             ctypes.byref(n_matches)))
    phases = plan.phases()
    comm = plan.arrays[0].comm            # doc-range shards: match counts and filtered dfs are global
    total_matches = n_matches.value if comm is None else int(comm.sum_u64([n_matches.value])[0])
    if total_matches == 0 or not any(items for _, items in phases):
        return multi

    # every phrase of one field runs in one launch on that field's lists filtered to qf > 0
    field_index = {f: i for i, f in enumerate(plan.names)}
    for f, rows in plan.phrase_rows().items():
        fi, arr, sim = field_index[f], plan.arrays[field_index[f]], plan.similarity[f]
        toks = plan.search_terms[f]
        uniq = list(dict.fromkeys(toks))
        slot = {t: i for i, t in enumerate(uniq)}
        u_ids = _u32([arr._term_id(t) for t in uniq])
        dfs = np.zeros(len(uniq), dtype=np.uint64)
        _lib.check(_timed("filter", L.sa_multi_filter, multi.handle, fi, _lib.p_u32(u_ids), len(uniq), _lib.p_u64(dfs)))
        if comm is not None:
            dfs = comm.sum_u64(dfs)
        starts, slots, ids, p_idf = [0], [], [], []
        phrase_lists = {name: phrases for name, items in phases for ff, _, phrases, _ in items if ff == f}
        for name, i in rows:
            ph = phrase_lists[name][i]
            slots.extend(slot[t] for t in ph)
            ids.extend(int(u_ids[slot[t]]) for t in ph)
            starts.append(len(slots))
            p_idf.append(compute_idf(arr.corpus_size, np.asarray([dfs[slot[t]] for t in ph])))
        a_st, a_sl, a_id, a_pi = _u32(starts), _u32(slots), _u32(ids), _f32(p_idf)
        _lib.check(_timed("phrases", L.sa_multi_phrases, multi.handle, fi, len(rows), _lib.p_u32(a_st), _lib.p_u32(a_sl),
                                      _lib.p_u32(a_id), _lib.p_f32(a_pi), arr.avg_doc_length, sim.k1, sim.b))
    for _, entries in plan.phase_entries():
        if entries:
            a_f, a_r = _u32([field_index[f] for f, _, _ in entries]), _u32([r for _, r, _ in entries])
            a_bo = _f32([0.0 if bo is None else bo for _, _, bo in entries])
            a_h = _u32([0 if bo is None else 1 for _, _, bo in entries])
            _lib.check(_timed("add_phase", L.sa_multi_add_phase, multi.handle, len(entries), _lib.p_u32(a_f), _lib.p_u32(a_r),
                                            _lib.p_f32(a_bo), _lib.p_u32(a_h)))
    return multi


def _run_composed(plan: _Plan) -> np.ndarray:
    """Custom similarity callables / sliced frames: every `.score` still runs on the GPU, the
    element-wise combination follows the reference's numpy composition (solr.py:117-355)."""
    arrays = dict(zip(plan.names, plan.arrays))
    n = len(plan.arrays[0])

    def boosted(vec, boost):
        return vec * (1 if boost is None else boost)

    if plan.term_centric:
        term_vecs = []
        for i in range(plan.num_terms):
            hi, tot = np.zeros(n), np.zeros(n)
            for f, boost in plan.query_fields.items():
                s = boosted(arrays[f].score(plan.search_terms[f][i], similarity=plan.similarity[f]), boost)
                tot += s
                hi = np.maximum(hi, s)
            term_vecs.append(hi + (tot - hi) * plan.tie)
        need = parse_min_should_match(plan.num_terms, spec=plan.mm)
        ok = np.sum(np.asarray(term_vecs) > 0, axis=0) >= need
        scores = np.sum(term_vecs, axis=0)
        scores[~ok] = 0
    else:
        field_vecs = []
        for f, boost in plan.query_fields.items():
            toks = plan.search_terms[f]
            ts = np.array([arrays[f].score(t, similarity=plan.similarity[f]) for t in toks])
            need = min(parse_min_should_match(len(toks), spec=plan.mm), len(toks))
            ok = np.sum(ts > 0, axis=0) >= need
            tot = np.sum(ts, axis=0)
            tot[~ok] = 0
            field_vecs.append(boosted(tot, boost))
        stacked = np.asarray(field_vecs)
        tot, hi = np.sum(stacked, axis=0), np.max(stacked, axis=0)
        scores = hi + (tot - hi) * plan.tie
    sliced = {f: arrays[f][scores > 0] for f in plan.names}
    for _, items in plan.phases():
        parts = []
        for f, boost, phrases, repeat_last in items:
            vec = None
            for ph in phrases:
                vec = boosted(sliced[f].score(ph, similarity=plan.similarity[f]), boost)
                parts.append(vec)
            if repeat_last:
                parts.append(vec)
        if parts:
            scores[np.where(scores)[0]] += np.sum(parts, axis=0)
    return scores


# ------------------------------------------------------------------------------ API
def edismax(frame: pd.DataFrame, q: str, qf: List[str], mm: Optional[Union[str, int]] = None,
            pf: Optional[List[str]] = None, pf2: Optional[List[str]] = None, pf3: Optional[List[str]] = None,
            ps2: int = 0, ps3: int = 0, ps: int = 0, tie: float = 0.0, q_op: str = "OR",
            similarity: Union[Similarity, Dict[str, Similarity]] = default_bm25) -> Tuple[np.ndarray, str]:
    """Same signature and result as the reference's `edismax` (solr.py:251-355): the score vector
    over the frame's rows (float64 term-centric, float32 field-centric) and the explain string.
    ps / ps2 / ps3 are accepted and ignored, as in the reference (quirk vii)."""
    plan = _Plan(frame, q, qf, mm, pf, pf2, pf3, tie, q_op, similarity)
    explain = plan.explain_qf() + plan.explain_phases()
    if not plan.device_ok():
        return _run_composed(plan), explain
    n = len(plan.arrays[0])
    multi = _multi_for(plan.arrays)
    with _locked(multi, plan.arrays):
        _run_device(plan, multi)
        out = np.empty(n, dtype=np.float64 if plan.term_centric else np.float32)
        _lib.check(_lib.lib().sa_multi_download(multi.handle, out.ctypes.data_as(ctypes.c_void_p),
                                                0 if plan.term_centric else 1))
    return out, explain


def edismax_topk(frame: pd.DataFrame, q: str, qf: List[str], k: int = 10, mm: Optional[Union[str, int]] = None,
                 pf: Optional[List[str]] = None, pf2: Optional[List[str]] = None, pf3: Optional[List[str]] = None,
                 tie: float = 0.0, q_op: str = "OR",
                 similarity: Union[Similarity, Dict[str, Similarity]] = default_bm25):
    """The k best rows of `edismax(...)` (score desc, row asc) without moving the score vector
    off the GPU.  Returns (rows uint32[k], scores float64[k]); unused slots are 0xFFFFFFFF / 0.  k: 1 <= k <= 1,024
    (query.TOPK_MAX); another k is a ValueError before any device work."""
    from .query import check_k
    k = check_k(k)
    plan = _Plan(frame, q, qf, mm, pf, pf2, pf3, tie, q_op, similarity)
    if not plan.device_ok():
        raise NotImplementedError("edismax_topk needs BM25 similarities on unsliced SearchArray columns")
    docs = np.empty(k, dtype=np.uint32)
    scores = np.empty(k, dtype=np.float64)
    multi = _multi_for(plan.arrays)
    with _locked(multi, plan.arrays):
        _run_device(plan, multi)
        _lib.check(_timed("topk", _lib.lib().sa_multi_topk, multi.handle, k, _lib.p_u32(docs),
                                            scores.ctypes.data_as(ctypes.POINTER(ctypes.c_double))))
    comm = plan.arrays[0].comm
    if comm is not None:                  # one all-gather of the per-shard top-k, merged on every rank
        return comm.merge_topk_f64(docs, scores, k)
    return docs, scores


def _fields_plan(frame, queries, similarity, extra=()):
    """fields_topk's refusals and field slots, before any device work: (the batch flattened for its form, at least
    OCCUR since the multi-field entry takes weights and roles (query.flatten_bool), field name -> slot, per-slot
    arrays, per-slot similarities).  extra: columns the call reads that no clause may name (facet columns), given
    slots after the clauses' fields."""
    from .query import ED_MAX_FIELDS, OCCUR, Field, bool_form, dismax_members, flatten_bool, is_boolean
    queries = list(queries)
    for q in queries:
        if not is_boolean(q):
            raise TypeError(f"fields_topk takes Or / And / Bool / DisMax queries, not {q!r}")
    batch = flatten_bool(queries, max([OCCUR] + [bool_form(q) for q in queries]))
    clauses = [c for c in batch.clauses if c is not None]    # None: a nested clause
    for c in clauses:
        if not isinstance(c, Field):
            raise ValueError(f"every clause of fields_topk names its column: Field(field, {c!r})")
    read = set(c.field for c in clauses)      # the columns a clause scores: their similarities count
    names = list(dict.fromkeys([c.field for c in clauses] + list(extra)))
    if len(names) > ED_MAX_FIELDS:
        raise ValueError(f"fields_topk takes at most {ED_MAX_FIELDS} distinct fields in one call, not {len(names)}")
    arrays = {f: get_field(frame, f) for f in names}
    sims = {}
    for f in names:
        sim = similarity.get(f, default_bm25) if isinstance(similarity, dict) else similarity
        if not isinstance(sim, Bm25Similarity):
            raise TypeError(f"fields_topk supports bm25_similarity only, not {sim!r} on {f!r}")
        sims[f] = sim
    for f, a in arrays.items():
        if a.rows is not None:
            raise NotImplementedError(f"fields_topk on a view (frame[mask]) is not supported yet: {f!r} is sliced; "
                                      "compose .score() on the view")
    if len({len(a) for a in arrays.values()}) > 1:
        raise ValueError("fields_topk needs columns of one length: " + ", ".join(f"{f}: {len(a)}" for f, a in arrays.items()))
    if len({a.device for a in arrays.values()}) > 1:
        raise ValueError("fields_topk needs columns on one device: " + ", ".join(f"{f}: {a.device}" for f, a in arrays.items()))
    # columns that share one device index (a copy of a column) are one slot: the index caches one BM25 norm table
    slot_of, slot_key, slot_arrays, slot_sims, slot_name = {}, {}, [], [], []
    for f in names:
        a, sim = arrays[f], sims[f]
        params = (np.float32(a.avg_doc_length), np.float32(sim.k1), np.float32(sim.b))
        s = slot_key.get(id(a._shared))
        if s is not None:
            if f in read and (np.float32(arrays[slot_name[s]].avg_doc_length), np.float32(slot_sims[s].k1),
                    np.float32(slot_sims[s].b)) != params:
                raise ValueError(f"{f!r} shares its device index with {slot_name[s]!r} but not its similarity: "
                                 "one index caches one set of BM25 parameters")
            slot_of[f] = s
            continue
        slot_of[f] = slot_key[id(a._shared)] = len(slot_arrays)
        slot_arrays.append(a)
        slot_sims.append(sim)
        slot_name.append(f)
    clause_slot = _clause_slots(batch, slot_of)
    if batch.groups is not None:          # DisMax members: sparse-safe k1 / b on their fields
        _check_dismax(dismax_members(queries), batch.clauses, clause_slot, slot_arrays, slot_sims)
    _PreparedBool.columns(batch.clauses, clause_slot, slot_arrays)   # feature / facet names set, In codes in range
    return batch, slot_of, slot_arrays, slot_sims


def _clause_slots(batch, slot_of):
    """uint32 per clause of a fields_topk batch: the slot of its field (_fields_plan), 0 for a nested clause."""
    return _u32([0 if c is None else slot_of[c.field] for c in batch.clauses])


def _facet_pairs(frame, facets):
    """fields_topk's facets= as (column, name) pairs, checked before any device work: a list of at most 4 distinct
    pairs, each column a SearchArray column of the frame (get_field) on whose index the name is set (ValueError)."""
    facets = check_facet_keys(facets, "(column, name) pairs")
    for pair in facets:
        if not (isinstance(pair, tuple) and len(pair) == 2 and isinstance(pair[1], str)):
            raise TypeError(f"a facet of fields_topk is a (column, name) pair, not {pair!r}")
        get_field(frame, pair[0])._facet_slot(pair[1])
    return facets


def _collapse_pair(frame, collapse):
    """fields_topk's collapse= as a (column, name) pair, checked before any device work: a pair (TypeError) whose
    column is a SearchArray column of the frame (get_field) on whose index the group column is set (ValueError)."""
    if not (isinstance(collapse, tuple) and len(collapse) == 2 and isinstance(collapse[1], str)):
        raise TypeError(f"collapse of fields_topk is a (column, name) pair, not {collapse!r}")
    get_field(frame, collapse[0])._group_slot(collapse[1])
    return collapse


def _fields_topk(frame, queries, k, similarity, slop, where=None, facets=None, collapse=None):
    """fields_topk and the number of queries re-run exactly (candidate overflow); with facets (a list of
    (column, name) pairs), (docs, scores, queries re-run, Hits).  collapse: a (column, name) pair, collapsed on."""
    queries = list(queries)
    if where is not None:
        where = pack_where(where, len(frame), len(queries))
    if facets is not None:
        facets = _facet_pairs(frame, facets)
    if collapse is not None:
        collapse = _collapse_pair(frame, collapse)
    extra = ([] if facets is None else [c for c, _ in facets]) + ([] if collapse is None else [collapse[0]])
    batch, slot_of, arrays, sims = _fields_plan(frame, queries, similarity, extra=extra)
    multi = _multi_for(arrays)
    with _locked(multi, arrays):
        return _PreparedBool(arrays, sims, _clause_slots(batch, slot_of), queries, batch, where,
                             None if facets is None else [(p, slot_of[p[0]], p[1]) for p in facets], multi,
                             None if collapse is None else (slot_of[collapse[0]], collapse[1])).run(k, slop)


def fields_score_docs(frame: pd.DataFrame, queries, rows,
                      similarity: Union[Similarity, Dict[str, Similarity]] = default_bm25, slop: int = 0):
    """SearchArray.score_docs over the columns of `frame`: out[q, j] == S_q[rows[q, j]], S_q the composition
    fields_topk ranks query q from (+0 where the row does not rank), so fields_score_docs(frame, queries,
    fields_topk(frame, queries, k)[0]) returns fields_topk's scores bit for bit (sa_multi_score_docs_bool).  queries
    and similarity as in fields_topk, under its refusals and column checks.  rows: an integer array of shape
    (len(queries), K), ids as fields_topk returns them (global doc ids on a shard), NO_DOC giving 0; Feature, Range and
    In clauses are evaluated at each row as fields_topk folds them.  Returns float32
    (len(queries), K).  Another dtype (TypeError), another shape or an id out of range (ValueError) is refused
    before any device work."""
    queries = list(queries)
    batch, slot_of, arrays, sims = _fields_plan(frame, queries, similarity)
    rows = check_docs(rows, len(queries), arrays[0].doc_base, len(frame))
    if rows.size == 0:
        return np.zeros(rows.shape, dtype=np.float32)
    multi = _multi_for(arrays)
    with _locked(multi, arrays):
        return _PreparedBool(arrays, sims, _clause_slots(batch, slot_of), queries, batch,
                             multi=multi).score_docs(rows, slop)


def _fields_topk_rescore(frame, queries, k, similarity, slop, where, facets, rescore):
    """fields_topk with `rescore` (query.Rescore), as SearchArray.search_topk's: pass 1 at k=rescore.window,
    fields_score_docs of the rescore queries at its rows, then query.rescore_window; hits are pass 1's."""
    from .query import Rescore, rescore_window
    if not isinstance(rescore, Rescore):
        raise TypeError(f"rescore is a query.Rescore, not {rescore!r}")
    queries = list(queries)
    rescore.check(len(queries), k)
    _fields_plan(frame, rescore.queries, similarity)        # the rescore queries' refusals, before pass 1
    out = fields_topk(frame, queries, rescore.window, similarity, slop, where, facets)
    s2 = fields_score_docs(frame, rescore.queries, out[0], similarity, rescore.slop)
    docs, scores = rescore_window(out[0], out[1], s2, rescore.query_weight, rescore.rescore_weight, k)
    return (docs, scores) + tuple(out[2:])


def fields_topk(frame: pd.DataFrame, queries, k: int = 10,
                similarity: Union[Similarity, Dict[str, Similarity]] = default_bm25, slop: int = 0, where=None,
                facets=None, rescore=None, collapse=None):
    """Batched Or / And / Bool queries whose clauses are on several columns of `frame` -- Lucene's
    `+title:star overview:war -overview:trek`, or Elasticsearch's most_fields `title:alien^2 overview:alien` -- ranked
    on the device in one batch.  Every clause is a query.Field(field, term or phrase), or a Boost of one; phrases match
    with `slop`.  similarity: one bm25_similarity, or a dict {field: bm25_similarity} (missing fields take the
    default), as in edismax.

    Per query the result is the top k (score desc, doc asc) of the composition search_topk ranks for a Bool, with
    score(Field(f, c)) = frame[f].array.score(c, similarity=similarity[f], slop=slop): each clause with its own
    column's idf, avgdl and doc lengths.  Returns (rows uint32[Q, k], scores float32[Q, k]); empty slots are NO_DOC /
    0; on a shard the rows are global doc ids.  Views, non-BM25 similarities, more than 8 distinct fields, columns of
    different lengths or devices, and two names of one column under different similarities are refused before any
    device work.

    A query.DisMax of Field members is one clause scoring d = max_j v_j + (sum_j v_j - max_j v_j) * tie over
    v_j = w_j * score(member j), each member on its own column: Elasticsearch's
    best_fields as DisMax([Boost(Field("title", "alien"), 2), Field("overview", "alien")], tie=0.3), and edismax's
    term-centric qf as an Or of one such DisMax per term with a Solr mm.  Its members need k1 > 0 and 0 <= b < 1 on
    their fields (ValueError otherwise).

    An Or / And / Bool may be a clause of another, at any depth, as in SearchArray.search_topk: edismax's qf + pf as
    Bool(must=[Or([DisMax(...), DisMax(...)], mm="75%")], should=[Boost(Field("title", ["a", "b"]), 3)]).

    Field(column, Feature(...)), Field(column, Range(...)) and Field(column, In(...)) read the feature or facet
    columns set on that column's index (SearchArray.set_feature / set_facet), as in SearchArray.search_topk:
    Bool(must=[Field("title", "alien")], filter=[Field("title", Range("year", gte=1980))]).

    where: a document filter, as in SearchArray.search_topk -- a boolean array-like (a boolean pd.Series too) of
    shape (len(frame),), one mask for the batch, or (len(queries), len(frame)), one per query.  Per query the
    result is the top k of np.where(mask_q, S_q, 0), S_q the composition above; the mask never changes a score
    (each column's idf, avgdl and doc lengths stay those of the whole column).  A dtype other than bool raises
    TypeError and another shape ValueError, before any device work.

    facets: hit and facet counts, as in SearchArray.search_topk -- a list of at most 4 distinct (column, name) pairs,
    name a facet set on that column (SearchArray.set_facet), possibly empty -- returns (rows, scores, hits), a Hits
    whose facets are keyed by the pairs: hits.total[q] == np.count_nonzero(S_q) and
    hits.facets[(column, name)][q] == np.bincount(codes[(S_q > 0) & (codes >= 0)], minlength=n_buckets), S_q the
    composition above with `where` applied.  The column may be any SearchArray column of the frame, read by a clause
    or not; it takes part in the column checks above.  rows and scores are bit for bit those of the call without
    `facets`.  A pair whose name is not set, a pair given twice or more than 4 pairs is a ValueError before any device
    work.  k: 1 <= k <= query.TOPK_MAX (1,024), as in SearchArray.search_topk; another k is a ValueError before any
    device work.

    rescore: a query.Rescore of queries of this form, as in SearchArray.search_topk -- the top k of the window
    fields_topk ranks at k=rescore.window, by the combined score c; hits are pass 1's.

    collapse: a (column, name) pair naming a group column set on that column (SearchArray.set_group): one row per
    group, as in SearchArray.search_topk -- the k best group leaders of S_q above, hits counting rows.  The column may
    be any SearchArray column of the frame, read by a clause or not; it takes part in the column checks above.  A value
    that is not a pair (TypeError), a name not set (ValueError) and `collapse` with `rescore` (ValueError) are refused
    before any device work.  On a shard the groups are collapsed over the shard's own rows."""
    from .query import check_k
    k = check_k(k)
    if collapse is not None and rescore is not None:
        raise ValueError("collapse cannot be combined with rescore")
    if rescore is not None:
        return _fields_topk_rescore(frame, queries, k, similarity, slop, where, facets, rescore)
    if facets is not None:
        docs, scores, _, hits = _fields_topk(frame, queries, k, similarity, slop, where, facets, collapse)
        return docs, scores, hits
    docs, scores, _ = _fields_topk(frame, queries, k, similarity, slop, where, collapse=collapse)
    return docs, scores
