// sa_bool.cu -- batched boolean queries (OR / AND / min-should-match over term and phrase clauses), ranked on the
// device.
//
// Replaces the reference's own composition of multi-clause queries (test/test_search.py:126-226):
//   scores = arr.score(c0) + arr.score(c1) + ...                              float32, clause order
//   ok     = np.sum(np.array([arr.score(c) for c in clauses]) > 0, axis=0) >= mm
//   top    = np.argpartition(np.where(ok, scores, 0), -k)[-k:]               utils/sort.py:24
//
// Design.  One CTA per (query, 8192-doc tile), the query index fastest (as term_tile_kernel).  Every thread owns
// the 32 docs of the tile that flush_tile_collect hands it (4 g .. 4 g + 3, g = tid + j * 256) and keeps their
// running sums and hit counts in registers; the clauses are folded in order, so each sum is the exact left fold
// above.  A term clause is scanned in place -- its (doc, tf) records, or its posting words with run heads summing
// popcounts -- and scattered as BM25 scores (bm25_from_norm over the cached norms) into a shared tile, which the
// owners read back after a barrier.  A phrase clause reads its count row (materialised beforehand by
// sa_phrase_row) coalesced.  Under parameters that are not sparse-safe a term clause scatters tf and the owners
// evaluate bm25_one over every doc, as the ALL_DOCS term scan does.  Before the fold the CTA counts the clauses that
// have anything in the tile; fewer than mm -> no doc of the tile can rank, and the tile is published empty.
// Then the docs below mm are zeroed and the tile goes through flush_tile_collect, the float32 collector of every
// other path, and topk_select_kernel ranks the candidates.
//
// One entry point per handle (sa_score_batch_topk_bool, sa_multi_score_batch_topk_bool) runs every form, with or
// without counts; the arrays it is given select the form, and the form, the mask and the variant (plain, FEATURE or
// COUNT) select one instance of bool_tile_kernel (bool_kernel).  The flags add, in order:
//
// OCCUR: Lucene's clause roles and per-clause weights, from a separate BoolOccur array: MUST / SHOULD clauses add
// weight * score, only SHOULD clauses count towards mm, and two per-thread masks over the thread's 32 docs record
// where a MUST / FILTER clause misses (`req`) and where a MUST_NOT clause matches (`veto`).  A tile where a MUST /
// FILTER clause has no doc, or with fewer SHOULD clauses than mm, is published empty before the fold.
//
// FIELDS (every multi-field call): clauses on several fields of one document set: a clause carries its field's slot,
// and every step reads that field's lists, norms, doc lengths and BM25 parameters from a small per-call table
// (BoolField) instead of the index in BoolArgs.
//
// DISMAX (a single-index call passes a one-entry field table): disjunction-max groups, a run of consecutive clauses
// that is one clause of its query.  A member's v = weight * score goes into the group's running max m and left-folded
// sum t, kept per owned doc in per-thread strips of dynamic shared memory, and a u32 mask records where any member
// scores > 0; at the group's last member d = m + (t - m) * tie is folded with weight 1 under the group's role, its hit
// being the mask.  A group is present in a tile iff any member is.
//
// NESTED: nested queries, an Or / And / Bool used as a clause of another.  Each nested node is materialised first,
// deepest level first, by the same fold in a store pass: its ranked values (0 where it does not rank) go to its row in
// BoolState::rows and a per-(row, tile) flag records whether anything ranked, a tile that ranks nothing writing only
// its flag.  A parent reads a nested clause's row as the clause's score (no BM25), present in a tile iff the child's
// flag is set; the top-level nodes are collected and selected as in every other instance.
//
// WHERE: a document mask (WhereMask, sa_term.cuh) on any of the five forms: a tile without an allowed doc is published
// empty before any of its lists is read, and a disallowed doc is zeroed with the docs below mm, before the tile's
// bound is taken, so the mask never changes a score, only which docs rank.  In a nested call only the top-level launch
// is masked: a disallowed doc never ranks whatever its nested rows hold.
//
// FEATURE: feature clauses (sa_index_set_feature) on the OCCUR, FIELDS, DISMAX and NESTED forms, in instances of
// their own so that a batch without one runs the instances above unchanged.  A feature clause is present in a tile iff
// its column's tile flag is set; in the fold its owners read their float4s of the column with cached loads (the CTAs
// of a batch's queries on one tile read the same 32 KB) and put v = f(x) into the shared tile, which the term clauses'
// fold then reads as it reads BM25 scores.  An Or / And batch with a feature runs as OCCUR.
//
// Range and In clauses (filters on a feature or a facet column, scored 1.0f where they match) run in the same
// instances, as feature clauses whose BoolFeature::fn is SA_FEATURE_RANGE or SA_FEATURE_IN.  Presence: a range is
// present iff its column's tile flag is set and the tile's [min, max] of values > 0 meets [lo, hi]; an In iff its
// 32-word code set meets the tile's (one word per lane, __any_sync).  A MUST / FILTER range or In absent from a tile
// publishes it empty before any list is read, as a mask does, and the tile is counted in the call's skip counter
// (sa_stats.filter_tiles).  In the fold a range's owners read their float4s of the column, and an In's owners their
// four uint16 codes as one 8-byte load, testing each against the clause's set with cached loads.
//
// COUNT: hit and facet counts (an entry point's out_total non-NULL), in instances of their own (the FEATURE instances
// with COUNT, an Or / And batch running as OCCUR) so that a batch without counts runs the instances above unchanged.
// After the tile's collect, s_tile still holds the ranked values (+0 where a doc does not rank); each thread turns its
// 32 into a mask, a warp adds its popcounts into the query's total with one atomic, and on a tile where anything ranks
// s_tile is reused as a shared histogram of the call's facets (<= 4 x 1,024 u32 = 16 KB): each thread reads the codes
// of its ranked docs (one 8-byte load per float4 group with a ranked doc), one shared atomic per ranked doc with a
// code, and the non-zero bins go to the query's counts with global atomics.  The store passes of a nested call, and a
// query re-run after a candidate overflow, run the instances without COUNT: the first pass has counted every tile of
// every query.
#include "sa_multi.cuh"
#include "sa_term.cuh"
#include "sa_phrase.cuh"

#define SA_BOOL_NO_ROW 0xFFFFFFFFu
#define SA_BOOL_FEATURE_ROW 0xFFFFFFFEu     // BoolClause::row of a feature clause (FEATURE instances)

struct BoolClause {
    u64 word_off, n_words, dir_off, rec_off;   // a term clause's list (TermQuery's fields); n_words == 0: no doc
    float idf;
    u32 row;        // a phrase clause's count row in BoolState::rows (within its group); SA_BOOL_NO_ROW: a term
    u32 sparse;     // Bm25Params::sparse_ok under this clause's idf
    u32 field;      // FIELDS: the clause's slot in the field table; 0 otherwise
};

struct BoolQuery { u32 c0, n, mm, pad; };   // clauses [c0, c0 + n) of the batch

struct BoolArgs {
    const u64 *words;
    const u32 *tile_dir, *recs, *rec_dir;   // see sa_index; recs NULL: no tf table
    const float *norm, *doc_lens;
    const float *rows;                      // phrase clauses' count rows, row_stride floats apart
    u64 row_stride, n_docs, doc_base;
    const BoolClause *clauses;
    const BoolQuery *queries;               // [gridDim.x]
    Bm25Params bm25;                        // idf unused (per clause)
    TopkCtx topk;
};

// A clause's role and weight (clause_weight, clause_occur), read by the OCCUR instances only, so the Or / And
// instance's loads stay those of BoolClause.
struct BoolOccur {
    float weight;   // MUST / SHOULD: s += weight * score (rounded once, then added)
    u32 occur;      // SA_OCCUR_*
};

// One field of sa_multi_score_batch_topk_bool, as the FIELDS instances read it: BoolArgs' per-index members.
struct BoolField {
    const u64 *words;
    const u32 *tile_dir, *recs, *rec_dir;
    const float *norm, *doc_lens;
    Bm25Params bm25;                        // idf unused (per clause)
};

// A clause's disjunction-max group (DISMAX instances only).  A clause outside a DisMax, or the one member of a
// single-member DisMax, is a group of one (member == 0) and folds exactly as in the FIELDS instance.
struct BoolGroup {
    float tie;      // the group's tie (member clauses)
    u32 first;      // the group's first clause, within its query
    u32 member;     // 1: a member of a group of two or more clauses
    u32 last;       // 1: the group's last member
};

// The nested-query part of the NESTED instances' arguments.  A nested node's row is BoolQuery::pad (its slot in
// BoolState::rows, numbered with the phrase rows of its launch group); a nested clause's BoolClause::row is its
// child's row.
struct BoolNest {
    const u32 *nested;  // per clause, as a.clauses: 1: a nested clause, scored by its child's row as stored
    u32 *flags;         // [row * n_tiles + tile]: 1 where the nested node of that row ranks a doc of the tile
    float *store;       // the store pass: a.rows, written at each node's row; NULL: top-level nodes, collected
    u32 n_tiles;
};

// A feature, range or In clause's column and function (FEATURE instances only), per clause as a.clauses; unused at
// other clauses.
struct BoolFeature {
    const float *values;    // feature / range: the column, float [padded n_docs], zero past n_docs
    const u32 *tiles;       // feature / range: its tile flags (1 where some value of the tile is > 0); In: the facet's
                            // tile code sets, SA_FACET_SET_WORDS words per tile
    float param;            // SA_FEATURE_SATURATION: pivot; SA_FEATURE_LOG: scaling factor
    u32 fn;                 // SA_FEATURE_*
    const float2 *bounds;   // range: per tile the (min, max) of the column's values > 0
    float lo, hi;           // range: the clause matches where x > 0 and lo <= x <= hi
    const unsigned short *codes;    // In: the facet column, uint16 [padded n_docs], SA_FACET_NONE for no value
    const u32 *set;         // In: the clause's codes, SA_FACET_SET_WORDS words (in the call's descriptors)
    u32 *skipped;           // the call's count of (node, tile) pairs an absent MUST / FILTER range or In made empty
};

// The counts of a COUNT launch: per query of the launch its total and its facet rows, each facet's column and the
// offset of its first bin in a row.  The kernel indexes the arrays with constants only (a dynamic index would copy the
// struct to local memory).
struct BoolCount {
    u32 *total;                                         // [launch query]
    u32 *counts;                                        // [launch query][n_bins]
    const unsigned short *codes[SA_BOOL_MAX_FACETS];    // uint16 [padded n_docs] (sa_index::d_facets)
    u32 offset[SA_BOOL_MAX_FACETS + 1];                 // offset[n_facets] == n_bins
    u32 n_facets, n_bins;
};

// The group column of a collapse launch (COLLAPSE instances only): per index-local doc its code or SA_GROUP_NONE
// (sa_index::d_groups), and the call's count of walk windows past the first (BoolResult::windows).
struct BoolCollapse {
    const u32 *groups;
    u32 *windows;
};

struct BoolState {
    DevBuf desc;         // the call's descriptor arrays, one section each (BoolDescs)
    DevBuf d_keys;       // the call's result block (BoolResult): one device-to-host copy
    DevBuf rows;
    DevBuf d_flags;      // BoolNest::flags
    DevBuf d_where;      // the WhereMask rows of a masked call
    DevBuf d_docs;       // sa_score_docs_bool: the docs, the scores and the nested-node lists (BoolDocs)
};
void BoolStateDelete::operator()(BoolState *s) const { delete s; }

__device__ __forceinline__ bool bool_uses_recs(const BoolArgs &a, const BoolClause &cl) {
    return a.recs != nullptr && cl.rec_off != SA_NO_DIR && cl.dir_off != SA_NO_DIR;
}

// A term clause's docs of this tile into s_tile: BM25 scores (sparse) or tf.  Slice [lo, hi) of its records or words.
__device__ __forceinline__ void bool_scatter_term(const BoolArgs &a, const BoolClause &cl, u32 lo, u32 hi,
                                                  u32 tile_doc0, u64 tile_doc0_abs, float *s_tile) {
    const float *__restrict__ norm = a.norm + tile_doc0;
    if (bool_uses_recs(a, cl)) {
        const u32 *__restrict__ recs = a.recs + cl.rec_off;
        for (u32 i = lo + threadIdx.x; i < hi; i += SA_TERM_THREADS) {
            const u32 r = __ldg(recs + i), rel = r >> SA_REC_TF_BITS, tf = r & SA_REC_TF_MASK;
            s_tile[rel] = cl.sparse ? bm25_from_norm((float)tf, __ldg(norm + rel), cl.idf) : (float)tf;
        }
        return;
    }
    // words: the thread holding a doc's first word sums the popcounts of the doc's run (a doc never spans tiles)
    const u64 *__restrict__ words = a.words + cl.word_off;
    for (u32 i = lo + threadIdx.x; i < hi; i += SA_TERM_THREADS) {
        const u64 doc = __ldg(words + i) >> SA_KEY_SHIFT;
        if (i > lo && (__ldg(words + i - 1) >> SA_KEY_SHIFT) == doc) continue;
        u32 tf = 0;
        for (u32 j = i; j < hi; j++) {
            const u64 w = __ldg(words + j);
            if ((w >> SA_KEY_SHIFT) != doc) break;
            tf += (u32)__popcll(w & SA_LSB_MASK);
        }
        const u32 rel = (u32)(doc - tile_doc0_abs);
        s_tile[rel] = cl.sparse ? bm25_from_norm((float)tf, __ldg(norm + rel), cl.idf) : (float)tf;
    }
}

// FEATURE: v of a doc whose feature value is x: +0 where x is 0, else x, x / (x + pivot) rounded step by step, or
// log(s + x) in double rounded once (Lucene's FeatureField functions); a range clause's 1.0f where lo <= x <= hi.
__device__ __forceinline__ float bool_feature_value(const BoolFeature &f, float x) {
    if (!(x > 0.0f)) return 0.0f;
    if (f.fn == SA_FEATURE_RANGE) return f.lo <= x && x <= f.hi ? 1.0f : 0.0f;
    if (f.fn == SA_FEATURE_SATURATION) return __fdiv_rn(x, __fadd_rn(x, f.param));
    if (f.fn == SA_FEATURE_LOG) return __double2float_rn(log(__dadd_rn((double)f.param, (double)x)));
    return x;
}

// FEATURE: an In clause's v at a doc whose code is c: 1.0f where c is in the clause's set (never for SA_FACET_NONE).
__device__ __forceinline__ float bool_in_value(const BoolFeature &f, unsigned short c) {
    return c != SA_FACET_NONE && ((__ldg(f.set + (c >> 5)) >> (c & 31)) & 1u) ? 1.0f : 0.0f;
}

// FEATURE: whether a feature, range or In clause is present in the tile (warp-uniform, every lane of the warp calls):
// its column's tile flag, and for a range the tile's bounds meeting [lo, hi]; for an In its set meeting the tile's.
__device__ __forceinline__ u32 bool_feature_present(const BoolFeature &f, u32 tile, unsigned lane) {
    if (f.fn == SA_FEATURE_IN) {
        const u32 w = __ldg(f.tiles + (u64)tile * SA_FACET_SET_WORDS + lane) & __ldg(f.set + lane);
        return __any_sync(0xFFFFFFFFu, w != 0) ? 1u : 0u;
    }
    if (!__ldg(f.tiles + tile)) return 0;
    if (f.fn != SA_FEATURE_RANGE) return 1;
    const float2 b = __ldg(f.bounds + tile);
    return b.x <= f.hi && b.y >= f.lo ? 1u : 0u;
}

// FEATURE: a feature, range or In clause's v at the thread's own docs into s_tile (each thread its own float4s, which
// it reads back in the fold; an In clause's four codes in one 8-byte load).  Not unrolled: the fold's registers stay
// live across it.
__device__ __forceinline__ void bool_feature_tile(const BoolFeature &f, u32 tile_doc0, float4 *s_tile4) {
    if (f.fn == SA_FEATURE_IN) {
        const ushort4 *__restrict__ c4 = reinterpret_cast<const ushort4 *>(f.codes + tile_doc0);
#pragma unroll 1
        for (int j = 0; j < SA_TILE_DOCS / SA_TERM_THREADS / 4; j++) {
            const unsigned g = threadIdx.x + j * SA_TERM_THREADS;
            const ushort4 c = __ldg(c4 + g);
            s_tile4[g] = make_float4(bool_in_value(f, c.x), bool_in_value(f, c.y), bool_in_value(f, c.z),
                                     bool_in_value(f, c.w));
        }
        return;
    }
    const float4 *__restrict__ v4 = reinterpret_cast<const float4 *>(f.values + tile_doc0);
#pragma unroll 1
    for (int j = 0; j < SA_TILE_DOCS / SA_TERM_THREADS / 4; j++) {
        const unsigned g = threadIdx.x + j * SA_TERM_THREADS;
        const float4 x = __ldg(v4 + g);
        s_tile4[g] = make_float4(bool_feature_value(f, x.x), bool_feature_value(f, x.y), bool_feature_value(f, x.z),
                                 bool_feature_value(f, x.w));
    }
}

// OCCUR: doc i = 4 j + e of the thread's 32 gets the clause's exact score v.  MUST / SHOULD add
// weight * v, each product rounded before the add as numpy rounds it (no FMA contraction); only SHOULD counts a hit,
// on the unweighted v, so a zero weight still matches; MUST / FILTER clear the doc's `req` bit where v is not > 0;
// MUST_NOT sets its `veto` bit where v > 0.  The occur tests are clause-uniform branches, which skip the work of the
// other roles (a branch-free select form measured slower).
__device__ __forceinline__ void bool_fold_occur(float &acc, u32 &hits, u32 &req, u32 &veto, int i, float v,
                                                const BoolOccur &oc) {
    if (oc.occur == SA_OCCUR_SHOULD || oc.occur == SA_OCCUR_MUST) acc = __fadd_rn(acc, __fmul_rn(oc.weight, v));
    if (oc.occur == SA_OCCUR_SHOULD) hits += (v > 0.0f ? 1u : 0u) << (8 * (i & 3));
    if ((oc.occur == SA_OCCUR_MUST || oc.occur == SA_OCCUR_FILTER) && !(v > 0.0f)) req &= ~(1u << i);
    if (oc.occur == SA_OCCUR_MUST_NOT && v > 0.0f) veto |= 1u << i;
}

// DISMAX: bool_fold_occur of a DisMax group's d, with the group's hit (any member > 0) in place of
// d > 0 and weight 1.
__device__ __forceinline__ void bool_fold_group(float &acc, u32 &hits, u32 &req, u32 &veto, int i, float d, bool hit,
                                                u32 occur) {
    if (occur == SA_OCCUR_SHOULD || occur == SA_OCCUR_MUST) acc = __fadd_rn(acc, d);
    if (occur == SA_OCCUR_SHOULD) hits += (hit ? 1u : 0u) << (8 * (i & 3));
    if ((occur == SA_OCCUR_MUST || occur == SA_OCCUR_FILTER) && !hit) req &= ~(1u << i);
    if (occur == SA_OCCUR_MUST_NOT && hit) veto |= 1u << i;
}

// DISMAX: member v of a group at owned doc i (sparse-safe, so v >= +0): the running max and left-folded sum of the
// weighted scores where the group scores (MUST / SHOULD), the hit mask in every role.  s_m / s_t: the thread's strips,
// doc i at [i * SA_TERM_THREADS].
__device__ __forceinline__ void bool_dismax_member(float &m, float &t, u32 &any, int i, float v, const BoolOccur &oc) {
    if (oc.occur == SA_OCCUR_SHOULD || oc.occur == SA_OCCUR_MUST) {
        const float w = __fmul_rn(oc.weight, v);
        m = fmaxf(m, w);
        t = __fadd_rn(t, w);
    }
    any |= (v > 0.0f ? 1u : 0u) << i;
}

// DISMAX, at a group's last member, for owned doc i with running max m and sum t: d = m + (t - m) * tie, rounded step
// by step as numpy (no FMA), folded under the group's role with the hit mask; m and t are reset for the next group.
__device__ __forceinline__ void bool_dismax_doc_end(float &acc, u32 &hits, u32 &req, u32 &veto, int i, u32 any,
                                                    float &m, float &t, float tie, u32 occur) {
    float d = 0.0f;
    if (occur == SA_OCCUR_SHOULD || occur == SA_OCCUR_MUST) {
        d = __fadd_rn(m, __fmul_rn(__fsub_rn(t, m), tie));
        m = t = 0.0f;
    }
    bool_fold_group(acc, hits, req, veto, i, d, ((any >> i) & 1u) != 0, occur);
}

// DISMAX, at a group's last member: bool_dismax_doc_end at each owned doc, then the hit mask is reset.
template <int N>
__device__ __forceinline__ void bool_dismax_group_end(float (&acc)[N * 4], u32 (&hits)[N], u32 &req, u32 &veto,
                                                      u32 &any, float *s_m, float *s_t, float tie, u32 occur) {
#pragma unroll
    for (int i = 0; i < N * 4; i++)
        bool_dismax_doc_end(acc[i], hits[i >> 2], req, veto, i, any, s_m[i * SA_TERM_THREADS], s_t[i * SA_TERM_THREADS],
                            tie, occur);
    any = 0;
}

// FIELDS: point the view `v` (a copy of the kernel's BoolArgs) at field slot f of the table: its lists, norms, doc
// lengths and BM25 parameters.  The entry's address is CTA-uniform, so its loads are broadcasts that stay cached.
template <bool FIELDS>
__device__ __forceinline__ void bool_set_field(BoolArgs &v, const BoolField *__restrict__ fld, u32 f) {
    if (!FIELDS) return;
    const BoolField &e = fld[f];
    v.words = e.words;
    v.tile_dir = e.tile_dir;
    v.recs = e.recs;
    v.rec_dir = e.rec_dir;
    v.norm = e.norm;
    v.doc_lens = e.doc_lens;
    v.bm25 = e.bm25;
}

// The thread index read afresh (asm volatile, never merged with other reads), so that a rare `tid == 0` test in the
// masked instances does not hold a predicate live through the fold (at the fields instance's 80-register cap it spilled).
__device__ __forceinline__ unsigned bool_fresh_tid() {
    unsigned t;
    asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t));
    return t;
}

// COUNT: the counting pass of one (query, tile), after flush_tile_collect (whose last barrier follows its last read
// of s_tile): s_tile holds the tile's ranked values, +0 where a doc does not rank.  All threads must call.
__device__ __forceinline__ void bool_count_tile(const BoolCount &cn, float *s_tile) {
    constexpr int PER = SA_TILE_DOCS / SA_TERM_THREADS / 4;
    const unsigned tid = bool_fresh_tid();
    const u32 q = blockIdx.x, tile = blockIdx.y;
    const float4 *s_tile4 = reinterpret_cast<const float4 *>(s_tile);
    u32 ranked = 0;                        // bit 4 j + e: doc 4 g + e ranks
#pragma unroll
    for (int j = 0; j < PER; j++) {
        const float4 x = s_tile4[tid + j * SA_TERM_THREADS];
        ranked |= ((x.x > 0.0f ? 1u : 0u) | (x.y > 0.0f ? 2u : 0u) | (x.z > 0.0f ? 4u : 0u) | (x.w > 0.0f ? 8u : 0u))
                  << (4 * j);
    }
    // the barrier also orders every read above before s_tile becomes the histogram
    if (!__syncthreads_or(ranked != 0)) return;
    const u32 n = __reduce_add_sync(0xFFFFFFFFu, (u32)__popc(ranked));
    if ((tid & 31) == 0 && n) atomicAdd(cn.total + q, n);
    if (cn.n_facets == 0) return;                                   // CTA-uniform
    u32 *s_hist = reinterpret_cast<u32 *>(s_tile);
    const u32 n_bins = cn.n_bins;
    for (u32 i = tid; i < n_bins; i += SA_TERM_THREADS) s_hist[i] = 0;
    __syncthreads();
    const u32 tile_doc0 = tile * SA_TILE_DOCS;
#pragma unroll
    for (int f = 0; f < SA_BOOL_MAX_FACETS; f++) {
        if (f >= (int)cn.n_facets) break;
        const ushort4 *__restrict__ c4 = reinterpret_cast<const ushort4 *>(cn.codes[f] + tile_doc0);
        u32 *h = s_hist + cn.offset[f];
#pragma unroll
        for (int j = 0; j < PER; j++) {
            const u32 m = (ranked >> (4 * j)) & 0xFu;
            if (!m) continue;
            const ushort4 c = __ldg(c4 + tid + j * SA_TERM_THREADS);
            if ((m & 1u) && c.x != SA_FACET_NONE) atomicAdd(h + c.x, 1u);
            if ((m & 2u) && c.y != SA_FACET_NONE) atomicAdd(h + c.y, 1u);
            if ((m & 4u) && c.z != SA_FACET_NONE) atomicAdd(h + c.z, 1u);
            if ((m & 8u) && c.w != SA_FACET_NONE) atomicAdd(h + c.w, 1u);
        }
    }
    __syncthreads();
    u32 *dst = cn.counts + (u64)q * n_bins;
    for (u32 i = tid; i < n_bins; i += SA_TERM_THREADS) {
        const u32 v = s_hist[i];
        if (v) atomicAdd(dst + i, v);
    }
}

// The tile fold of one (query, tile).  OCCUR = false: Or / And (every clause SHOULD, weight 1).  OCCUR = true:
// per-clause roles and weights in occ[], indexed as a.clauses; a query's mm counts its SHOULD clauses.  FIELDS: each
// clause reads the field fld[clause.field] (bool_set_field) in place of the index in `a`; n_docs, doc_base, the
// phrase rows and the top-k context stay common.  DISMAX (with OCCUR and FIELDS): clauses form groups (grp[], indexed
// as a.clauses); mm counts SHOULD groups; s_dyn holds the groups' running max and sum, 2 * 32 floats per thread, and
// s_g[3] (shared) the groups' presence masks.  NESTED (with DISMAX): nested clauses and the store pass (BoolNest).
// WHERE: only docs whose bit of the mask row of query blockIdx.x is set rank (never in a store pass).  FEATURE (with
// OCCUR): clauses whose row is SA_BOOL_FEATURE_ROW score their column feat[clause] (BoolFeature).  COUNT (with
// FEATURE): the collected tile is counted into `cn` (bool_count_tile).  DEEP: k > SA_TOPK_MAX, the tile's candidates
// from deep_tile_collect.  COLLAPSE: the tile's k best group leaders (collapse_tile_collect over the group column
// co.groups, its hash in s_dyn, free once the fold is done), then, when the launch counts (cn.total non-NULL, a
// CTA-uniform test), the tile's hits and facets as COUNT counts them.
template <bool OCCUR, bool FIELDS, bool DISMAX, bool NESTED, bool WHERE, bool FEATURE, bool COUNT, bool DEEP,
          bool COLLAPSE = false>
__device__ __forceinline__ void bool_tile(const BoolArgs &a, const BoolOccur *__restrict__ occ,
                                          const BoolField *__restrict__ fld, const BoolGroup *__restrict__ grp,
                                          float *s_dyn, unsigned long long *s_g, const BoolNest nb, const WhereMask wh,
                                          const BoolFeature *__restrict__ feat, const BoolCount cn,
                                          const BoolCollapse co) {
    constexpr int PER = SA_TILE_DOCS / SA_TERM_THREADS / 4;        // float4 groups per thread
    __shared__ __align__(16) float s_tile[SA_TILE_DOCS];
    __shared__ u32 s_lo[SA_BOOL_MAX_CLAUSES], s_hi[SA_BOOL_MAX_CLAUSES];
    __shared__ u32 s_top[(SA_TERM_THREADS / 32) * 8];
    __shared__ u32 s_ncand, s_tile_max, s_present;
    // DISMAX: bit g of s_g[0] / [1] / [2]: the group whose first clause is the query's clause g has a member in the
    // tile / is SHOULD / is MUST or FILTER
    unsigned long long &s_g_present = s_g[0], &s_g_should = s_g[1], &s_g_req = s_g[2];
    const u32 q = blockIdx.x, tile = blockIdx.y;
    const BoolQuery bq = a.queries[q];
    const unsigned tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const u32 tile_doc0 = tile * SA_TILE_DOCS;
    const u64 tile_doc0_abs = a.doc_base + tile_doc0;              // as stored in the words
    float4 *s_tile4 = reinterpret_cast<float4 *>(s_tile);
    BoolArgs view = a;                                              // FIELDS: the clause's field (bool_set_field)

    // 1. zero the tile; every clause's slice of the tile, and how many clauses have anything in it
#pragma unroll
    for (int j = 0; j < PER; j++) s_tile4[tid + j * SA_TERM_THREADS] = make_float4(0.f, 0.f, 0.f, 0.f);
    const bool tid0 = WHERE ? bool_fresh_tid() == 0 : tid == 0;
    if (tid0) s_present = 0;
    if (DISMAX && tid0) s_g_present = s_g_should = s_g_req = 0;
    u32 allow = ~0u;                       // WHERE: bit 4 j + e: the mask allows doc 4 g + e
    if (WHERE) {
        // no allowed doc in the tile: nothing ranks, and no list is read (contiguous filters skip whole tiles)
        allow = where_word(wh, q, tile);
        if (!__syncthreads_or(allow != 0)) {
            publish_empty_tile(a.topk, q, tile, bool_fresh_tid());
            return;
        }
    } else {
        __syncthreads();
    }
    for (u32 c = warp; c < bq.n; c += SA_TERM_THREADS / 32) {      // warp-uniform
        const BoolClause cl = a.clauses[bq.c0 + c];
        bool_set_field<FIELDS>(view, fld, cl.field);
        const BoolArgs &ca = FIELDS ? view : a;
        u32 lo = 0, hi = 0;
        bool filt = false;                  // FEATURE: a range or In clause
        if (NESTED && nb.nested[bq.c0 + c]) {
            hi = nb.flags[(u64)cl.row * nb.n_tiles + tile] != 0;   // the child ranks a doc of the tile
        } else if (FEATURE && cl.row == SA_BOOL_FEATURE_ROW) {
            const BoolFeature &f = feat[bq.c0 + c];
            hi = bool_feature_present(f, tile, lane);               // some doc of the tile can match
            filt = f.fn >= SA_FEATURE_RANGE;
        } else if (cl.row != SA_BOOL_NO_ROW) {
            hi = 1;                                                 // a phrase row counts as present
        } else if (cl.n_words == 0) {
        } else if (cl.dir_off != SA_NO_DIR) {
            const u32 *dir = (bool_uses_recs(ca, cl) ? ca.rec_dir : ca.tile_dir) + cl.dir_off + tile;
            lo = __ldg(dir);
            hi = __ldg(dir + 1);
        } else {
            const u64 *w = ca.words + cl.word_off;
            lo = (u32)warp_lower_bound_shifted(w, 0, cl.n_words, tile_doc0_abs, SA_KEY_SHIFT);
            hi = (u32)warp_lower_bound_shifted(w, lo, cl.n_words, tile_doc0_abs + SA_TILE_DOCS, SA_KEY_SHIFT);
        }
        if (lane == 0) {
            s_lo[c] = lo;
            s_hi[c] = hi;
            if (DISMAX) {
                const u32 o = occ[bq.c0 + c].occur;
                const unsigned long long bit = 1ull << grp[bq.c0 + c].first;
                if (hi > lo) atomicOr(&s_g_present, bit);
                if (o == SA_OCCUR_SHOULD) atomicOr(&s_g_should, bit);
                if (o == SA_OCCUR_MUST || o == SA_OCCUR_FILTER) atomicOr(&s_g_req, bit);
            } else if (OCCUR) {
                // low 16 bits: SHOULD clauses present; high bits: MUST / FILTER clauses absent (<= 64 clauses)
                const u32 o = occ[bq.c0 + c].occur;
                const u32 add = o == SA_OCCUR_SHOULD ? (hi > lo ? 1u : 0u)
                              : (o == SA_OCCUR_MUST || o == SA_OCCUR_FILTER) && hi <= lo ? 1u << 16 : 0u;
                if (add) atomicAdd(&s_present, add);
            } else if (hi > lo) {
                atomicAdd(&s_present, 1u);
            }
            // bit 24: an absent MUST / FILTER range or In (above the OCCUR counts, <= 64 << 16)
            if (FEATURE && filt && hi <= lo) {
                const u32 o = occ[bq.c0 + c].occur;
                if (o == SA_OCCUR_MUST || o == SA_OCCUR_FILTER) atomicOr(&s_present, 1u << 24);
            }
        }
    }
    __syncthreads();
    // 2. a clause with nothing in the tile scores > 0 at no doc of it: fewer such clauses than mm, nothing ranks;
    //    nor does anything where a MUST / FILTER clause is absent
    //    (DISMAX: fewer SHOULD groups with a member in the tile than mm, or a MUST / FILTER group without one)
    if (DISMAX ? ((u32)__popcll(s_g_present & s_g_should) < bq.mm || (s_g_req & ~s_g_present) != 0)
               : OCCUR ? ((s_present & 0xFFFFu) < bq.mm || (s_present >> 16) != 0) : s_present < bq.mm) {   // CTA-uniform
        if (FEATURE && (s_present >> 24) && bool_fresh_tid() == 0) atomicAdd(feat[bq.c0].skipped, 1u);
        if (NESTED && nb.store != nullptr) {                        // a nested node: its flag only
            if (tid == 0) nb.flags[(u64)bq.pad * nb.n_tiles + tile] = 0;
            return;
        }
        publish_empty_tile(a.topk, q, tile, threadIdx.x);
        return;
    }

    // 3. the fold, clause by clause in order
    float acc[PER * 4];
    u32 hits[PER];                         // byte e of hits[j]: clauses scoring > 0 at doc 4 g + e (<= 64 clauses)
#pragma unroll
    for (int i = 0; i < PER * 4; i++) acc[i] = 0.0f;
#pragma unroll
    for (int j = 0; j < PER; j++) hits[j] = 0;
    // OCCUR: bit 4 j + e of the thread's docs (PER * 4 == 32).  WHERE: a doc the mask leaves out starts as a missed
    // requirement, so step 4 drops it with the others without another register held through the fold
    u32 req = allow, veto = 0;
    static_assert(PER * 4 == 32, "one u32 mask bit per owned doc");
    u32 any = 0;                           // DISMAX: bit 4 j + e: a member of the current group scores > 0 there
    float *s_m = s_dyn + tid, *s_t = s_dyn + PER * 4 * SA_TERM_THREADS + tid;
    if (DISMAX) {
#pragma unroll
        for (int i = 0; i < PER * 4; i++) s_m[i * SA_TERM_THREADS] = s_t[i * SA_TERM_THREADS] = 0.0f;
    }
    Bm25Params p = a.bm25;
    for (u32 c = 0; c < bq.n; c++) {
        const BoolClause cl = a.clauses[bq.c0 + c];
        const u32 lo = s_lo[c], hi = s_hi[c];
        BoolGroup gr{0.0f, 0u, 0u, 0u};
        if (DISMAX) gr = grp[bq.c0 + c];
        // CTA-uniform: +0 at every doc of the tile, which changes neither a group's max nor its sum (v >= +0); a
        // group's last member still folds the group
        const bool absent = cl.sparse && hi <= lo;
        if (absent && !(DISMAX && gr.last)) continue;
        BoolOccur oc{1.0f, SA_OCCUR_SHOULD};
        if (OCCUR) oc = occ[bq.c0 + c];
        if (DISMAX && absent) {
            bool_dismax_group_end(acc, hits, req, veto, any, s_m, s_t, gr.tie, oc.occur);
            continue;
        }
        bool_set_field<FIELDS>(view, fld, cl.field);
        const BoolArgs &ca = FIELDS ? view : a;
        if (FIELDS) p = ca.bm25;
        p.idf = cl.idf;
        const bool feature = FEATURE && cl.row == SA_BOOL_FEATURE_ROW;
        if (cl.row != SA_BOOL_NO_ROW && !feature) {
            // phrase clause (sparse-safe parameters only): BM25 of its counts, zero counts score +0.  NESTED: a nested
            // clause's row holds its child's ranked scores (>= +0), read as they are
            const bool nested = NESTED && nb.nested[bq.c0 + c];
            const float4 *__restrict__ r4 = reinterpret_cast<const float4 *>(a.rows + (u64)cl.row * a.row_stride + tile_doc0);
#pragma unroll
            for (int j = 0; j < PER; j++) {
                const unsigned g = tid + j * SA_TERM_THREADS;
                const float4 x = __ldcs(r4 + g);
                const float xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    const u64 d = (u64)tile_doc0 + g * 4 + e;
                    float v = 0.0f;
                    if (NESTED && nested) v = xs[e];
                    else if (xs[e] > 0.0f && d < a.n_docs) v = bm25_from_norm(xs[e], __ldg(ca.norm + d), cl.idf);
                    if (DISMAX && gr.member) {
                        bool_dismax_member(s_m[(j * 4 + e) * SA_TERM_THREADS], s_t[(j * 4 + e) * SA_TERM_THREADS], any,
                                           j * 4 + e, v, oc);
                    } else if (OCCUR) {
                        bool_fold_occur(acc[j * 4 + e], hits[j], req, veto, j * 4 + e, v, oc);
                    } else {
                        acc[j * 4 + e] = __fadd_rn(acc[j * 4 + e], v);
                        hits[j] += (v > 0.0f ? 1u : 0u) << (8 * e);
                    }
                }
            }
        } else {
            // a feature clause (sparse, so v is read as it is) or a term clause
            if (feature) bool_feature_tile(feat[bq.c0 + c], tile_doc0, s_tile4);
            else bool_scatter_term(ca, cl, lo, hi, tile_doc0, tile_doc0_abs, s_tile);
            __syncthreads();
#pragma unroll
            for (int j = 0; j < PER; j++) {
                const unsigned g = tid + j * SA_TERM_THREADS;
                const float4 x = s_tile4[g];
                s_tile4[g] = make_float4(0.f, 0.f, 0.f, 0.f);
                const float xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    const u64 d = (u64)tile_doc0 + g * 4 + e;
                    float v = xs[e];
                    // bm25.pyx:20-25 over every doc (NaN / inf / -0.0 of exotic parameters)
                    if (!cl.sparse) v = d < a.n_docs ? bm25_one(xs[e], __ldg(ca.doc_lens + d), p) : 0.0f;
                    if (DISMAX && gr.member) {
                        bool_dismax_member(s_m[(j * 4 + e) * SA_TERM_THREADS], s_t[(j * 4 + e) * SA_TERM_THREADS], any,
                                           j * 4 + e, v, oc);
                    } else if (OCCUR) {
                        bool_fold_occur(acc[j * 4 + e], hits[j], req, veto, j * 4 + e, v, oc);
                    } else {
                        acc[j * 4 + e] = __fadd_rn(acc[j * 4 + e], v);
                        hits[j] += (v > 0.0f ? 1u : 0u) << (8 * e);
                    }
                }
            }
            __syncthreads();
        }
        if (DISMAX && gr.last) bool_dismax_group_end(acc, hits, req, veto, any, s_m, s_t, gr.tie, oc.occur);
    }

    // 4. docs with fewer than mm hits (or a sum <= 0 / NaN), and under OCCUR docs a MUST / FILTER clause misses or a
    //    MUST_NOT clause matches, do not rank, nor under WHERE docs the mask leaves out (in `req`; zeroed here,
    //    before my_max: a bound taken over disallowed scores could push allowed docs out of the candidates); collect
    //    the tile's top-k candidates
    const u32 keep = req & ~veto;
    u32 my_max = 0;
#pragma unroll
    for (int j = 0; j < PER; j++) {
        float o[4];
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const float s = acc[j * 4 + e];
            const bool ok = (OCCUR || WHERE) ? ((keep >> (j * 4 + e)) & 1u) != 0 : true;
            o[e] = (ok && ((hits[j] >> (8 * e)) & 0xFFu) >= bq.mm && s > 0.0f) ? s : 0.0f;
            my_max = max(my_max, __float_as_uint(o[e]));
        }
        s_tile4[tid + j * SA_TERM_THREADS] = make_float4(o[0], o[1], o[2], o[3]);
    }
    if (NESTED && nb.store != nullptr) {
        // a nested node: its ranked values to its row where anything ranks (each thread its own float4s), and the
        // tile's flag
        const int ranked = __syncthreads_or(my_max != 0);
        if (ranked) {
            float4 *dst = reinterpret_cast<float4 *>(nb.store + (u64)bq.pad * a.row_stride + tile_doc0);
#pragma unroll
            for (int j = 0; j < PER; j++) dst[tid + j * SA_TERM_THREADS] = s_tile4[tid + j * SA_TERM_THREADS];
        }
        if (tid == 0) nb.flags[(u64)bq.pad * nb.n_tiles + tile] = ranked ? 1u : 0u;
        return;
    }
    if constexpr (COLLAPSE) {
        collapse_tile_collect(s_tile, a.topk, q, tile, co.groups, reinterpret_cast<u32 *>(s_dyn), co.windows);
        if (cn.total != nullptr) bool_count_tile(cn, s_tile);
        return;
    }
    flush_tile_collect<false, DEEP>(s_tile, nullptr, a.topk, q, tile, my_max, SA_TILE_DOCS, 0, s_top, &s_ncand,
                                    &s_tile_max);
    if (COUNT) bool_count_tile(cn, s_tile);
}

// Every instance of the fold: bool_tile with every argument, of which it reads those its flags name (the others are
// NULL and never read).  MIN_CTAS holds an instance to the CTAs per SM it was tuned for (0: no minimum); bool_kernel
// lists the instances.  DISMAX: the groups' running max and sum live in SA_BOOL_DISMAX_SMEM bytes of dynamic shared
// memory (a thread's strips, owner-only, so no extra barriers).  COLLAPSE: the collector's hash in the same dynamic
// memory (bool_smem).
#define SA_BOOL_DISMAX_SMEM (2 * SA_TILE_DOCS * sizeof(float))

// bool_tile's s_g placed ahead of the fold's own shared arrays.  Where the compiler places a __shared__ array follows
// where it is declared: the unmasked DisMax instances without FEATURE were tuned with s_g first (a local of this
// helper, one instance per kernel), the others with it last (a local of the kernel), and each keeps its layout.
template <bool NESTED, bool DEEP>
__device__ __forceinline__ unsigned long long *bool_s_g_first() {
    __shared__ unsigned long long s_g[3];
    return s_g;
}

template <bool OCCUR, bool FIELDS, bool DISMAX, bool NESTED, bool WHERE, bool FEATURE, bool COUNT, bool DEEP,
          int MIN_CTAS, bool COLLAPSE = false>
__global__ void __launch_bounds__(SA_TERM_THREADS, MIN_CTAS)
bool_tile_kernel(const BoolArgs a, const BoolOccur *__restrict__ occ, const BoolField *__restrict__ fld,
                 const BoolGroup *__restrict__ grp, const BoolNest nb, const WhereMask wh,
                 const BoolFeature *__restrict__ feat, const BoolCount cn, const BoolCollapse co) {
    extern __shared__ __align__(16) float s_dyn[];
    if constexpr (DISMAX && !WHERE && !FEATURE) {
        bool_tile<OCCUR, FIELDS, DISMAX, NESTED, WHERE, FEATURE, COUNT, DEEP, COLLAPSE>(
            a, occ, fld, grp, s_dyn, bool_s_g_first<NESTED, DEEP>(), nb, wh, feat, cn, co);
    } else {
        __shared__ unsigned long long s_g[3];
        bool_tile<OCCUR, FIELDS, DISMAX, NESTED, WHERE, FEATURE, COUNT, DEEP, COLLAPSE>(a, occ, fld, grp, s_dyn, s_g, nb,
                                                                                  wh, feat, cn, co);
    }
}

// ----------------------------------------------------------------------------------- scoring at given documents
// sa_score_docs_bool evaluates the tile fold at a list of documents: one thread per (query, doc), one CTA per 256 docs
// of one query, every clause looked up at the doc and folded with the tile fold's own device functions, so each value
// is bit for bit the one bool_tile ranks from (its step 4 at one doc).  A clause absent from a tile, which the tile
// fold skips, is folded here with its value +0 at the doc: the same result wherever a doc ranks.

// What bool_docs_kernel reads besides BoolArgs.  The per-clause arrays are those of the call's form, NULL above it, as
// bool_run_group passes them.
struct BoolDocs {
    const BoolOccur *occ;
    const BoolField *fld;
    const BoolGroup *grp;
    const BoolFeature *feat;
    const u32 *nest;         // per clause: 1 for a nested clause (BoolNest::nested); NULL: no nested node
    const u32 *child;        // per clause: a nested clause's child, as its slot in its query's node list
    const u32 *node_start;   // per top-level query q: its nested nodes are node_list[node_start[q] .. node_start[q + 1])
    const u32 *node_list;    // each query's nested nodes, deepest first, as indices of their BoolArgs::queries entries
    const u32 *docs;         // [n_queries][n_per]: global doc ids in the index's range, or SA_NO_DOC
    float *out;              // [n_queries][n_per]
    u32 n_per, chunks;       // docs per query; CTAs per query, ceil(n_per / SA_TERM_THREADS)
};

// A term clause's tf at local doc dl, read as bool_scatter_term reads it: the doc's record in its tile's slice of the
// tf table, or the popcounts of the doc's run of posting words; the first of either found by binary search, the words
// within the tile's slice where the term has a tile directory and within the whole list otherwise.  Returns
// SA_DOCS_FOUND | tf where the doc is in the list, 0 where it is not.  `ca`: the clause's field (bool_set_field).
#define SA_DOCS_FOUND (1ull << 32)
__device__ __forceinline__ u64 bool_docs_tf(const BoolArgs &ca, const BoolClause &cl, u32 dl) {
    if (cl.n_words == 0) return 0;
    const u32 tile = dl / SA_TILE_DOCS, rel = dl % SA_TILE_DOCS;
    if (bool_uses_recs(ca, cl)) {
        const u32 *__restrict__ dir = ca.rec_dir + cl.dir_off + tile;
        const u32 *__restrict__ recs = ca.recs + cl.rec_off;
        u32 lo = __ldg(dir), end = __ldg(dir + 1), hi = end;
        while (lo < hi) {
            const u32 mid = (lo + hi) >> 1;
            if ((__ldg(recs + mid) >> SA_REC_TF_BITS) < rel) lo = mid + 1;
            else hi = mid;
        }
        if (lo == end) return 0;
        const u32 r = __ldg(recs + lo);
        return (r >> SA_REC_TF_BITS) == rel ? SA_DOCS_FOUND | (r & SA_REC_TF_MASK) : 0;
    }
    const u64 *__restrict__ words = ca.words + cl.word_off;
    u64 lo = 0, end = cl.n_words;
    if (cl.dir_off != SA_NO_DIR) {
        const u32 *__restrict__ dir = ca.tile_dir + cl.dir_off + tile;
        lo = __ldg(dir);
        end = __ldg(dir + 1);
    }
    const u64 doc = ca.doc_base + dl;                              // as stored in the words
    u64 hi = end;
    while (lo < hi) {
        const u64 mid = (lo + hi) >> 1;
        if ((__ldg(words + mid) >> SA_KEY_SHIFT) < doc) lo = mid + 1;
        else hi = mid;
    }
    u32 tf = 0;
    bool found = false;
    for (u64 j = lo; j < end; j++) {
        const u64 w = __ldg(words + j);
        if ((w >> SA_KEY_SHIFT) != doc) break;
        tf += (u32)__popcll(w & SA_LSB_MASK);
        found = true;
    }
    return found ? SA_DOCS_FOUND | tf : 0;
}

// Clause c's value v at local doc dl, as bool_tile's step 3 gives it: a nested clause its child's ranked value (in the
// thread's strip `mine`, slot x.child[c]), a feature, range or In clause its v, a phrase clause BM25 of its count row, a term clause
// BM25 of its tf -- from the cached norm where the clause is sparse-safe (+0 off its list), else bm25_one at every doc.
__device__ __forceinline__ float bool_docs_value(const BoolArgs &a, const BoolDocs &x, u32 c, const BoolClause &cl,
                                                 u32 dl, const float *mine) {
    if (x.nest && x.nest[c]) return mine[x.child[c] * SA_TERM_THREADS];
    if (x.feat && cl.row == SA_BOOL_FEATURE_ROW) {
        const BoolFeature &f = x.feat[c];
        if (f.fn == SA_FEATURE_IN) return bool_in_value(f, __ldg(f.codes + dl));
        return bool_feature_value(f, __ldg(f.values + dl));
    }
    BoolArgs view = a;
    if (x.fld) bool_set_field<true>(view, x.fld, cl.field);
    if (cl.row != SA_BOOL_NO_ROW) {
        const float r = __ldg(a.rows + (u64)cl.row * a.row_stride + dl);
        return r > 0.0f ? bm25_from_norm(r, __ldg(view.norm + dl), cl.idf) : 0.0f;
    }
    const u64 found_tf = bool_docs_tf(view, cl, dl);
    const u32 tf = (u32)found_tf;
    if (cl.sparse) return found_tf ? bm25_from_norm((float)tf, __ldg(view.norm + dl), cl.idf) : 0.0f;
    Bm25Params p = view.bm25;
    p.idf = cl.idf;
    return bm25_one((float)tf, __ldg(view.doc_lens + dl), p);     // bm25.pyx:20-25 over every doc
}

// The value node bq ranks local doc dl with: its clauses folded in order (bool_fold_occur, or a DisMax group's
// bool_dismax_member and bool_dismax_doc_end, at the one doc i = 0), +0 where it does not rank.
__device__ __forceinline__ float bool_docs_node(const BoolArgs &a, const BoolDocs &x, const BoolQuery bq, u32 dl,
                                                const float *mine) {
    float acc = 0.0f, m = 0.0f, t = 0.0f;   // the sum; the current DisMax group's running max and sum
    u32 hits = 0, req = 1u, veto = 0, any = 0;
    for (u32 c = bq.c0; c < bq.c0 + bq.n; c++) {
        const BoolClause cl = a.clauses[c];
        const float v = bool_docs_value(a, x, c, cl, dl, mine);
        const BoolOccur oc = x.occ ? x.occ[c] : BoolOccur{1.0f, SA_OCCUR_SHOULD};
        const BoolGroup gr = x.grp ? x.grp[c] : BoolGroup{0.0f, 0u, 0u, 0u};
        if (gr.member) {
            bool_dismax_member(m, t, any, 0, v, oc);
            if (gr.last) {
                bool_dismax_doc_end(acc, hits, req, veto, 0, any, m, t, gr.tie, oc.occur);
                any = 0;
            }
        } else {
            bool_fold_occur(acc, hits, req, veto, 0, v, oc);
        }
    }
    return ((req & ~veto) & 1u) && (hits & 0xFFu) >= bq.mm && acc > 0.0f ? acc : 0.0f;
}

// The thread's pair (q, j): its index q * x.n_per + j in docs and out, and its query q, from the CTA and thread
// indices read afresh (asm volatile): values computed once at the start stayed live across the fold's division
// calls (the slow path of __fdiv_rn is a subroutine) and spilled.
__device__ __forceinline__ u64 bool_docs_at(const BoolDocs &x, u32 q0, u32 *q) {
    unsigned b, t;
    asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(b));
    asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t));
    *q = q0 + b / x.chunks;
    return (u64)*q * x.n_per + (b % x.chunks) * SA_TERM_THREADS + t;
}

// Pairs (q, j) of queries [q0, q0 + gridDim.x / x.chunks), j < x.n_per: out = the value query q ranks doc docs[q][j]
// with, its nested nodes evaluated first, deepest first, each into the thread's strip of s_nest (slot i at
// [i * SA_TERM_THREADS]); SA_NO_DOC gives +0.
__global__ void __launch_bounds__(SA_TERM_THREADS)
bool_docs_kernel(const BoolArgs a, const BoolDocs x, u32 q0) {
    extern __shared__ float s_nest[];
    if ((blockIdx.x % x.chunks) * SA_TERM_THREADS + threadIdx.x >= x.n_per) return;   // no barrier follows
    u32 q;
    const u32 doc = __ldg(x.docs + bool_docs_at(x, q0, &q));
    float v = 0.0f;
    if (doc != SA_NO_DOC) {
        const u32 dl = doc - (u32)a.doc_base;                      // ids are u32: doc_base + n_docs <= 2^32
        if (x.nest) {
            const u32 n0 = x.node_start[q], n1 = x.node_start[q + 1];
            for (u32 i = n0; i < n1; i++)
                s_nest[(i - n0) * SA_TERM_THREADS + threadIdx.x] =
                    bool_docs_node(a, x, a.queries[x.node_list[i]], dl, s_nest + threadIdx.x);
        }
        v = bool_docs_node(a, x, a.queries[q], dl, s_nest + threadIdx.x);
    }
    x.out[bool_docs_at(x, q0, &q)] = v;
}

// ------------------------------------------------------------------------------------------------------------ host
namespace {

// The form of a call, which picks its instance: Or / And; roles and weights (OCCUR); every multi-field call (FIELDS);
// DisMax groups (on a field table, a single-index call passing one field); nested nodes.
enum BoolForm { BOOL_OR_AND, BOOL_OCCUR, BOOL_FIELDS, BOOL_DISMAX, BOOL_NESTED };

// The instances of a form: plain; FEATURE, for a batch with feature clauses; COUNT (with FEATURE), for the first pass
// of a counting call; COLLAPSE (with FEATURE from BOOL_OCCUR up, counting at run time), for the top-level launch of a
// collapsed call.  FEATURE and COUNT exist from BOOL_OCCUR up.
enum BoolVariant { BOOL_PLAIN, BOOL_FEATURE, BOOL_COUNT, BOOL_COLLAPSE };

typedef void (*BoolKernel)(BoolArgs, const BoolOccur *, const BoolField *, const BoolGroup *, BoolNest, WhereMask,
                           const BoolFeature *, BoolCount, BoolCollapse);

// The instance a launch of `form` runs, with or without a document mask.  The fields instance is held to three CTAs per
// SM, as the single-field roles instance runs (80 registers, no spills; at two, 90 registers, it ran 23-24% slower);
// the DisMax and nested ones to two (DESIGN.md sections 3.10.3, 3.10.4); each masked instance to its unmasked
// instance's CTAs per SM (section 3.11); the FEATURE and COUNT instances to their form's (three for the roles form).
// The COLLAPSE instances (one depth: DEEP is unused) run at two CTAs per SM, which their shared memory allows (the
// tile, the window's run and a 32 KB hash: ~74 KB); at three the roles and fields ones spilled 336 bytes.  A nested
// call's store passes run the unmasked nested instance.
template <bool DEEP>
BoolKernel bool_instance(BoolForm form, bool masked, BoolVariant variant) {
    static const BoolKernel instances[4][5][2] = {
        {
            {bool_tile_kernel<false, false, false, false, false, false, false, DEEP, 0>,
             bool_tile_kernel<false, false, false, false, true, false, false, DEEP, 2>},
            {bool_tile_kernel<true, false, false, false, false, false, false, DEEP, 0>,
             bool_tile_kernel<true, false, false, false, true, false, false, DEEP, 3>},
            {bool_tile_kernel<true, true, false, false, false, false, false, DEEP, 3>,
             bool_tile_kernel<true, true, false, false, true, false, false, DEEP, 3>},
            {bool_tile_kernel<true, true, true, false, false, false, false, DEEP, 2>,
             bool_tile_kernel<true, true, true, false, true, false, false, DEEP, 2>},
            {bool_tile_kernel<true, true, true, true, false, false, false, DEEP, 2>,
             bool_tile_kernel<true, true, true, true, true, false, false, DEEP, 2>},
        },
        {
            {nullptr, nullptr},
            {bool_tile_kernel<true, false, false, false, false, true, false, DEEP, 3>,
             bool_tile_kernel<true, false, false, false, true, true, false, DEEP, 3>},
            {bool_tile_kernel<true, true, false, false, false, true, false, DEEP, 3>,
             bool_tile_kernel<true, true, false, false, true, true, false, DEEP, 3>},
            {bool_tile_kernel<true, true, true, false, false, true, false, DEEP, 2>,
             bool_tile_kernel<true, true, true, false, true, true, false, DEEP, 2>},
            {bool_tile_kernel<true, true, true, true, false, true, false, DEEP, 2>,
             bool_tile_kernel<true, true, true, true, true, true, false, DEEP, 2>},
        },
        {
            {nullptr, nullptr},
            {bool_tile_kernel<true, false, false, false, false, true, true, DEEP, 3>,
             bool_tile_kernel<true, false, false, false, true, true, true, DEEP, 3>},
            {bool_tile_kernel<true, true, false, false, false, true, true, DEEP, 3>,
             bool_tile_kernel<true, true, false, false, true, true, true, DEEP, 3>},
            {bool_tile_kernel<true, true, true, false, false, true, true, DEEP, 2>,
             bool_tile_kernel<true, true, true, false, true, true, true, DEEP, 2>},
            {bool_tile_kernel<true, true, true, true, false, true, true, DEEP, 2>,
             bool_tile_kernel<true, true, true, true, true, true, true, DEEP, 2>},
        },
        {
            {bool_tile_kernel<false, false, false, false, false, false, false, false, 2, true>,
             bool_tile_kernel<false, false, false, false, true, false, false, false, 2, true>},
            {bool_tile_kernel<true, false, false, false, false, true, false, false, 2, true>,
             bool_tile_kernel<true, false, false, false, true, true, false, false, 2, true>},
            {bool_tile_kernel<true, true, false, false, false, true, false, false, 2, true>,
             bool_tile_kernel<true, true, false, false, true, true, false, false, 2, true>},
            {bool_tile_kernel<true, true, true, false, false, true, false, false, 2, true>,
             bool_tile_kernel<true, true, true, false, true, true, false, false, 2, true>},
            {bool_tile_kernel<true, true, true, true, false, true, false, false, 2, true>,
             bool_tile_kernel<true, true, true, true, true, true, false, false, 2, true>},
        },
    };
    return instances[variant][form][masked];
}

// deep: k > SA_TOPK_MAX, the instance whose tiles collect with deep_tile_collect
BoolKernel bool_kernel(BoolForm form, bool masked, BoolVariant variant, bool deep) {
    return deep ? bool_instance<true>(form, masked, variant) : bool_instance<false>(form, masked, variant);
}

// The dynamic shared memory of an instance: the DisMax groups' strips from BOOL_DISMAX up, and a COLLAPSE instance's
// hash (collapse_tile_collect), which reuses the strips once the fold is done.
size_t bool_smem(BoolForm form, bool collapse) {
    const size_t fold = form >= BOOL_DISMAX ? SA_BOOL_DISMAX_SMEM : 0;
    return collapse ? std::max<size_t>(fold, SA_COLLAPSE_TILE_SMEM) : fold;
}

// The fields of one call and where the call keeps its state.  The single-index entry point passes one field and the
// index's own buffers (ix->boolq, ix->cand, ix->h_pinned); sa_multi_score_batch_topk_bool passes the multi's fields,
// its BoolState and candidate buffer, and field 0's pinned staging.  Every field's stream is `lead`'s (FieldGuard).
struct BoolCall {
    std::vector<sa_index *> ix;         // per field slot
    std::vector<float> avgdl, k1, b;    // per field slot
    bool fields_kernel;                 // a multi-field call: BOOL_FIELDS at least (clauses carry their field slot)
    BoolState *S;
    DevBuf *cand;
    PinnedBuf *h_pinned;
    sa_index *lead() const { return ix[0]; }
};

bool bool_is_feature_term(u32 t) { return t >= SA_FEATURE_TERM_BASE && t != SA_NO_TERM; }

// What a leaf clause is, decided from its entries in one place (BoolInput::kind): a term (one id), a phrase (several
// ids, or one feature id among several entries, which bool_check refuses), a feature (one reserved id), a range (a
// reserved id of SA_FEATURE_RANGE, then its bounds' bits) or an In (a reserved id of SA_FEATURE_IN, then its codes).
enum BoolKind { KIND_TERM, KIND_PHRASE, KIND_FEATURE, KIND_RANGE, KIND_IN };

// A call's arrays and scalars as its entry point was given them, in the entry points' argument order.
// clause_weight / clause_occur NULL: Or / And, every clause SHOULD with weight 1, mm over all.  clause_field NULL:
// every clause on field 0.  clause_group / clause_tie non-NULL (with clause_occur): DisMax groups, on a field table.
// clause_node non-NULL (with the DisMax arrays): n_nodes nodes, the first n_queries top-level, clause c being nested
// node clause_node[c] unless SA_NO_NODE; otherwise n_nodes == n_queries.  where_bits non-NULL: the document mask.
// out_total non-NULL: hit counts, and counts over the n_facets facets.  groups non-NULL: a collapsed call on that group
// column (index-local ids), set by the collapse entry points.
struct BoolInput {
    u32 n_nodes;
    const u32 *node_clause_starts, *clause_node, *clause_field, *clause_terms, *clause_term_starts;
    const float *clause_idf, *clause_weight;
    const uint8_t *clause_occur;
    const u32 *clause_group;
    const float *clause_tie;
    const u32 *mm;
    u32 n_queries, slop, k;
    const u32 *where_bits;
    uint64_t where_n, where_stride;
    u32 *out_docs;
    float *out_scores;
    u32 *n_redone;
    u32 n_facets;
    const u32 *facet_field, *facet_slot;
    u32 *out_total, *out_facet_counts;
    const u32 *groups;

    bool nested(u32 c) const { return clause_node && clause_node[c] != SA_NO_NODE; }
    u32 field(u32 c) const { return clause_field ? clause_field[c] : 0; }
    const u32 *terms(u32 c) const { return clause_terms + clause_term_starts[c]; }
    u32 n_terms(u32 c) const { return clause_term_starts[c + 1] - clause_term_starts[c]; }
    // clause c's kind (a leaf with at least one entry)
    BoolKind kind(u32 c) const {
        const u32 t = terms(c)[0], n = n_terms(c);
        if (bool_is_feature_term(t)) {
            const u32 fn = (t >> 8) & 0xFFFFu;
            if (fn == SA_FEATURE_RANGE) return KIND_RANGE;
            if (fn == SA_FEATURE_IN) return KIND_IN;
            if (n == 1) return KIND_FEATURE;
        }
        return n == 1 ? KIND_TERM : KIND_PHRASE;
    }
    // a feature, range or In clause: a column of its field's index, scored without BM25
    bool column(u32 c) const { return kind(c) >= KIND_FEATURE; }
    // clause c of a node with clauses [c0, c1) is a member of a DisMax group of two or more clauses
    bool member(u32 c, u32 c0, u32 c1) const {
        return clause_group && ((c > c0 && clause_group[c] == clause_group[c - 1]) ||
                                (c + 1 < c1 && clause_group[c + 1] == clause_group[c]));
    }
};

// What bool_check learns of a call for the steps after it.
struct BoolChecked {
    bool features = false;  // some clause is a feature, range or In
    bool empty = false;     // nothing can rank: no query, no doc, or every field's avgdl 0 and no feature
    BoolCount count{};      // counting: the facets' columns and bins (the rows are placed per launch)
};

// Where each descriptor array of a call starts, in bytes, in BoolState::desc and in the host block it is uploaded
// from in one copy: one section per array, each 256-byte aligned.
struct BoolDescs { size_t clauses, queries, occur, groups, nest, fields, features, sets, bytes; };

// The result block of a call, in BoolState::d_keys and downloaded whole into the pinned staging: the keys
// [n_queries][k], then the overflow flags [n_queries] and, counting, the totals [n_queries] and the facet rows
// [n_queries][n_bins], then the tiles absent range and In filters made empty (BoolFeature::skipped) and the collapse
// walk's windows past the first (BoolCollapse::windows).  `base` is either copy.
struct BoolResult {
    size_t n_keys, n_queries, n_bins;
    bool counting;
    u64 *keys(void *base) const { return (u64 *)base; }
    u32 *ovf(void *base) const { return (u32 *)(keys(base) + n_keys); }
    u32 *total(void *base) const { return ovf(base) + n_queries; }
    u32 *counts(void *base) const { return total(base) + n_queries; }
    u32 *skipped(void *base) const { return ovf(base) + n_queries * (counting ? 2 + n_bins : 1); }
    u32 *windows(void *base) const { return skipped(base) + 1; }
    size_t bytes() const { return n_keys * sizeof(u64) + (n_queries * (counting ? 2 + n_bins : 1) + 2) * sizeof(u32); }
};

struct BoolPlan {
    BoolForm form = BOOL_OR_AND;
    u32 slots = 0;                      // candidate slots per tile of a first pass (k when collapsing)
    std::vector<BoolClause> clauses;
    std::vector<BoolQuery> queries;
    std::vector<u32> group_start;       // queries [group_start[i], group_start[i + 1]) share one launch and its rows
    std::vector<BoolOccur> occur;       // per clause, as clauses (from BOOL_OCCUR up)
    std::vector<BoolGroup> groups;      // per clause, as clauses (from BOOL_DISMAX up)
    u32 max_rows = 0;
    // nested calls: nodes 0 .. n_queries - 1 are the top-level queries (queries[0 .. n_queries)), the others nested
    std::vector<u32> root, depth;       // per node: its top-level query, and its depth below it
    std::vector<u32> nested;            // nested nodes by (launch group, depth desc, top-level query);
                                        // queries[n_queries + i] is nested[i]'s descriptor
    std::vector<u32> nest;              // per clause, as clauses: 1 for a nested clause (BOOL_NESTED)
    std::vector<BoolFeature> features;  // per clause, as clauses, when a clause is a feature, range or In (the FEATURE
                                        // instances); an In's `set` and every `skipped` are placed by bool_upload
    std::vector<u32> sets;              // the In clauses' code sets in clause order, SA_FACET_SET_WORDS words each
    std::vector<char> field_sparse;     // per field slot: 1 with a sparse-safe clause (its norms are cached)
    BoolCount count{};                  // the facet table of bool_check
    BoolDescs descs{};
    BoolResult result{};
};

// The variant a launch runs: COUNT for the first pass of a counting call (count), otherwise FEATURE when the batch has
// a feature clause.
BoolVariant bool_variant(const BoolPlan &P, bool count) {
    return count ? BOOL_COUNT : P.features.empty() ? BOOL_PLAIN : BOOL_FEATURE;
}

// The count rows of the phrase clauses of queries [q0, q1) and of their nested nodes (rows are numbered within the
// group), each on its clause's field, synchronously.
int bool_build_rows(const BoolCall &X, const BoolPlan &P, const BoolInput &in, u32 q0, u32 q1) {
    const u64 stride = sa_padded_docs(X.lead()->n_docs);
    int rc;
    std::vector<u32> nodes;
    for (u32 q = q0; q < q1; q++) nodes.push_back(q);
    for (u32 n : P.nested)
        if (P.root[n] >= q0 && P.root[n] < q1) nodes.push_back(n);
    for (u32 n : nodes) {
        for (u32 c = in.node_clause_starts[n]; c < in.node_clause_starts[n + 1]; c++) {
            const BoolClause &cl = P.clauses[c];
            if (cl.row == SA_BOOL_NO_ROW || cl.row == SA_BOOL_FEATURE_ROW || in.nested(c)) continue;
            sa_index *ix = X.ix[cl.field];
            bool scored;
            if ((rc = sa_phrase_row(ix, in.terms(c), in.n_terms(c), in.slop, nullptr, nullptr, nullptr, &scored)))
                return rc;
            SA_CUDA(cudaMemcpyAsync(X.S->rows.as<float>() + (u64)cl.row * stride, ix->dense.p, ix->n_docs * sizeof(float),
                                    cudaMemcpyDeviceToDevice, ix->stream));
        }
    }
    return SA_OK;
}

// The kernels' BoolArgs of an uploaded call, without a top-k context: the lead index's lists, norms and BM25
// parameters below BOOL_FIELDS (the field-table forms read them per clause), the rows, and every query's descriptor
// from queries[0] on.
BoolArgs bool_args(const BoolCall &X, const BoolPlan &P) {
    sa_index *ix = X.lead();
    BoolArgs a;
    memset(&a, 0, sizeof(a));
    if (P.form < BOOL_FIELDS) {
        a.words = ix->d_words.as<u64>();
        a.tile_dir = ix->d_tile_dir.as<u32>();
        a.recs = ix->d_recs.as<u32>();
        a.rec_dir = ix->d_rec_dir.as<u32>();
        a.norm = ix->d_norm.as<float>();
        a.doc_lens = ix->d_doc_lens.as<float>();
        a.bm25 = make_bm25(1.0f, X.avgdl[0], X.k1[0], X.b[0], ix->doc_lens_nonneg);
    }
    const char *d = X.S->desc.as<const char>();
    a.rows = X.S->rows.as<float>();
    a.row_stride = sa_padded_docs(ix->n_docs);
    a.n_docs = ix->n_docs;
    a.doc_base = ix->doc_base;
    a.clauses = (const BoolClause *)(d + P.descs.clauses);
    a.queries = (const BoolQuery *)(d + P.descs.queries);
    return a;
}

// Queries [q0, q1) with `slots` candidate slots per tile: their rows, the tile kernel and the selection, enqueued.
// count: the first pass of a counting call, the top-level launch counting into the call's rows.
int bool_run_group(const BoolCall &X, const BoolPlan &P, const BoolInput &in, const WhereMask &where, u32 slots,
                   u32 q0, u32 q1, bool count) {
    sa_index *ix = X.lead();
    BoolState &S = *X.S;
    const u32 n_tiles = sa_n_tiles(ix->n_docs), nq = q1 - q0;
    int rc;
    if ((rc = bool_build_rows(X, P, in, q0, q1))) return rc;
    if ((rc = X.cand->reserve(cand_bytes(n_tiles, nq, slots)))) return rc;
    TopkCtx t = make_topk_ctx(X.cand->p, n_tiles, nq, slots, in.k, P.result.ovf(S.d_keys.p) + q0);
    BoolArgs a = bool_args(X, P);
    const char *d = S.desc.as<const char>();
    const BoolQuery *queries = a.queries;
    a.queries = queries + q0;
    a.topk = t;
    WhereMask wh = where;                   // row 0 of the launch is query q0's
    if (wh.bits) wh.bits += (u64)q0 * wh.stride;
    // the arrays P.form reads, NULL above it
    const BoolOccur *occ = P.form >= BOOL_OCCUR ? (const BoolOccur *)(d + P.descs.occur) : nullptr;
    const BoolField *fld = P.form >= BOOL_FIELDS ? (const BoolField *)(d + P.descs.fields) : nullptr;
    const BoolGroup *grp = P.form >= BOOL_DISMAX ? (const BoolGroup *)(d + P.descs.groups) : nullptr;
    BoolNest nb{nullptr, nullptr, nullptr, 0};
    const BoolFeature *feat = P.features.empty() ? nullptr : (const BoolFeature *)(d + P.descs.features);
    BoolCount cn = P.count;                 // counting: the call's rows, from query q0's in the counting launch
    if (in.out_total) {
        const u32 row0 = count ? q0 : 0;
        cn.total = P.result.total(S.d_keys.p) + row0;
        cn.counts = P.result.counts(S.d_keys.p) + (u64)row0 * cn.n_bins;
    }
    const BoolCollapse co{in.groups, P.result.windows(S.d_keys.p)};
    auto launch = [&](bool c, bool masked, u32 n_q, const BoolArgs &args, const BoolNest &n, const WhereMask &w) -> int {
        // a collapsed call's top-level launch collapses (and counts where cn.total is set: a collapse is never re-run)
        const bool collapse = in.groups && !n.store;
        const BoolVariant variant = collapse ? BOOL_COLLAPSE : bool_variant(P, c);
        bool_kernel(P.form, masked, variant, in.k > SA_TOPK_MAX)<<<dim3(n_q, n_tiles), SA_TERM_THREADS,
                                                                    bool_smem(P.form, collapse), ix->stream>>>(
            args, occ, fld, grp, n, w, feat, cn, co);
        SA_CUDA(cudaGetLastError());
        if (collapse) ix->stats.collapse_tiles += (u64)n_q * n_tiles;
        else if (in.k > SA_TOPK_MAX && !n.store) ix->stats.deep_tiles += (u64)n_q * n_tiles;
        ix->stats.total_launches++;
        ix->stats.bool_instances |= 1ull << (variant * 10 + P.form * 2 + (masked ? 1 : 0));
        return SA_OK;
    };
    if (P.form == BOOL_NESTED) {
        // the nested nodes of these queries, deepest level first (one launch per level: a level's nodes of the run
        // are consecutive in P.nested), each into its row and flags, unmasked; then the top-level nodes, collected
        nb = BoolNest{(const u32 *)(d + P.descs.nest), S.d_flags.as<u32>(), S.rows.as<float>(), n_tiles};
        for (size_t i = 0; i < P.nested.size();) {
            auto in_run = [&](size_t x) { return P.root[P.nested[x]] >= q0 && P.root[P.nested[x]] < q1; };
            if (!in_run(i)) { i++; continue; }
            size_t j = i + 1;
            while (j < P.nested.size() && in_run(j) && P.depth[P.nested[j]] == P.depth[P.nested[i]]) j++;
            BoolArgs an = a;
            an.queries = queries + in.n_queries + i;
            if ((rc = launch(false, false, (u32)(j - i), an, nb, WhereMask{nullptr, 0}))) return rc;
            i = j;
        }
        nb.store = nullptr;
    }
    if ((rc = launch(count, wh.bits != nullptr, nq, a, nb, wh))) return rc;
    u64 *keys = P.result.keys(S.d_keys.p) + (size_t)q0 * in.k;
    if (in.groups) return launch_topk_collapse(ix, t, nq, ix->doc_base, in.groups, keys, co.windows);
    return launch_topk_select(ix, t, nq, ix->doc_base, keys, nullptr);
}

// An instance's dynamic shared memory (`bytes`, above what fits the default 48 KB with its static arrays), and the
// carveout that fits its CTAs per SM (two DisMax CTAs: ~2 x 98 KB), on the current device (function attributes are
// per device).
int bool_set_smem(BoolKernel kernel, size_t bytes) {
    SA_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    SA_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout,
                                 (int)cudaSharedmemCarveoutMaxShared));
    return SA_OK;
}

// A feature clause's reserved term id and parameter (include/searcharray_b200.h), on index ix: SA_ERR_ARG unless
// its function is known, its slot set on ix and its parameter in range.
int bool_check_feature(const sa_index *ix, u32 c, u32 term, float param) {
    const u32 fn = (term >> 8) & 0xFFFFu, slot = term & 0xFFu;
    SA_CHECK(fn <= SA_FEATURE_LOG, "clause %u: term id 0x%08x names no feature function", c, term);
    SA_CHECK(slot < SA_MAX_FEATURES && (ix->feature_set >> slot & 1u), "clause %u: feature slot %u is not set", c,
             slot);
    SA_CHECK(fn != SA_FEATURE_LINEAR || param == 0.0f, "clause %u: a linear feature takes no parameter (0)", c);
    SA_CHECK(fn != SA_FEATURE_SATURATION || (std::isfinite(param) && param > 0.0f),
             "clause %u: a saturation pivot is finite and > 0", c);
    SA_CHECK(fn != SA_FEATURE_LOG || (std::isfinite(param) && param >= 1.0f),
             "clause %u: a log scaling factor is finite and >= 1", c);
    return SA_OK;
}

// A range clause's entries (its reserved id, then the bits of lo and hi) and parameter, on index ix: SA_ERR_ARG unless
// its slot is a feature set on ix, it has three entries, neither bound is NaN and the parameter is 0.
int bool_check_range(const sa_index *ix, u32 c, const u32 *e, u32 n, float param) {
    const u32 slot = e[0] & 0xFFu;
    SA_CHECK(slot < SA_MAX_FEATURES && (ix->feature_set >> slot & 1u), "clause %u: feature slot %u is not set", c,
             slot);
    SA_CHECK(n == 3, "clause %u: a range clause has 3 entries (id, lo, hi), not %u", c, n);
    float lo, hi;
    memcpy(&lo, e + 1, sizeof(float));
    memcpy(&hi, e + 2, sizeof(float));
    SA_CHECK(!std::isnan(lo) && !std::isnan(hi), "clause %u: a range bound is NaN", c);
    SA_CHECK(param == 0.0f, "clause %u: a range clause takes no parameter (0)", c);
    return SA_OK;
}

// An In clause's entries (its reserved id, then its codes) and parameter, on index ix: SA_ERR_ARG unless its slot is a
// facet set on ix, it has a code, every code is below the facet's n_buckets and the parameter is 0.
int bool_check_in(const sa_index *ix, u32 c, const u32 *e, u32 n, float param) {
    const u32 slot = e[0] & 0xFFu;
    SA_CHECK(slot < SA_MAX_FACETS && (ix->facet_set >> slot & 1u), "clause %u: facet slot %u is not set", c, slot);
    SA_CHECK(n >= 2, "clause %u: an In clause has at least one code", c);
    for (u32 i = 1; i < n; i++)
        SA_CHECK(e[i] < ix->facet_buckets[slot], "clause %u: code %u is not below the facet's %u buckets", c, e[i],
                 ix->facet_buckets[slot]);
    SA_CHECK(param == 0.0f, "clause %u: an In clause takes no parameter (0)", c);
    return SA_OK;
}

// Bm25Params::sparse_ok of a clause with idf `idf` on field f.
bool bool_sparse(const BoolCall &X, u32 f, float idf) {
    return make_bm25(idf, X.avgdl[f], X.k1[f], X.b[f], X.ix[f]->doc_lens_nonneg).sparse_ok != 0;
}

// Every refusal of a call (SA_ERR_ARG), with no CUDA API call.  The BM25-parameter refusals come last, and only where
// something can rank, on fields with avgdl > 0: a call or a clause that scores nothing takes any parameters.
int bool_check(const BoolCall &X, const BoolInput &in, BoolChecked *out) {
    const u32 n_fields = (u32)X.ix.size(), n_nodes = in.n_nodes, n_queries = in.n_queries;
    const u32 *starts = in.node_clause_starts;
    const bool occur = in.clause_occur != nullptr, dismax = in.clause_group != nullptr;
    int rc;
    SA_CHECK(n_nodes >= n_queries, "n_nodes (%u) is below n_queries (%u)", n_nodes, n_queries);
    SA_CHECK(n_nodes == 0 || starts[0] == 0, "query_clause_starts[0] must be 0");
    for (u32 q = 0; q < n_nodes; q++) {
        SA_CHECK(starts[q + 1] > starts[q] && starts[q + 1] - starts[q] <= SA_BOOL_MAX_CLAUSES,
                 "query %u: a boolean query has 1 to %d clauses", q, SA_BOOL_MAX_CLAUSES);
        u32 n_should = starts[q + 1] - starts[q];
        if (occur) {
            n_should = 0;
            for (u32 c = starts[q]; c < starts[q + 1]; c++) {
                SA_CHECK(in.clause_occur[c] <= SA_OCCUR_MUST_NOT, "clause %u: occur %u is not an SA_OCCUR_* value", c,
                         (unsigned)in.clause_occur[c]);
                SA_CHECK(std::isfinite(in.clause_weight[c]) && in.clause_weight[c] >= 0.0f,
                         "clause %u: a weight is finite and >= 0", c);
                if (dismax) {
                    // a group: consecutive clauses of one query, one occur; its tie at its first clause
                    const u32 g = in.clause_group[c];
                    SA_CHECK(g >= starts[q] && g <= c && (g == c || in.clause_group[c - 1] == g),
                             "clause %u: group %u is not a run of consecutive clauses of query %u", c, g, q);
                    SA_CHECK(in.clause_occur[c] == in.clause_occur[g],
                             "clause %u: the members of group %u differ in occur", c, g);
                    if (g == c) {
                        SA_CHECK(std::isfinite(in.clause_tie[c]) && in.clause_tie[c] >= 0.0f && in.clause_tie[c] <= 1.0f,
                                 "clause %u: a tie is finite and in [0, 1]", c);
                    } else {
                        continue;   // mm counts groups
                    }
                }
                n_should += in.clause_occur[c] == SA_OCCUR_SHOULD;
            }
        }
        SA_CHECK(in.mm[q] <= n_should, "query %u: mm exceeds its %s", q,
                 dismax ? "SHOULD groups" : occur ? "SHOULD clauses" : "clauses");
    }
    // nested nodes: each referenced by exactly one clause of an earlier node, as a clause of its own (no terms, not a
    // DisMax member); the top-level nodes by none
    std::vector<u32> refs(in.clause_node ? n_nodes : 0, 0);
    for (u32 n = 0; in.clause_node && n < n_nodes; n++) {
        for (u32 c = starts[n]; c < starts[n + 1]; c++) {
            if (!in.nested(c)) continue;
            const u32 ch = in.clause_node[c];
            SA_CHECK(ch < n_nodes && ch >= n_queries && ch > n,
                     "clause %u: node %u is not a nested node after its holder %u (%u nodes, %u top-level)", c, ch, n,
                     n_nodes, n_queries);
            SA_CHECK(refs[ch]++ == 0, "node %u is referenced by more than one clause", ch);
            SA_CHECK(in.n_terms(c) == 0, "clause %u: a nested clause has no terms", c);
            SA_CHECK(in.clause_group[c] == c && (c + 1 == starts[n + 1] || in.clause_group[c + 1] != c),
                     "clause %u: a nested clause is not a DisMax member", c);
        }
    }
    for (u32 n = n_queries; in.clause_node && n < n_nodes; n++)
        SA_CHECK(refs[n] == 1, "node %u is referenced by no clause", n);
    if ((rc = sa_where_check(in.where_bits, in.where_n, in.where_stride, X.lead()->n_docs))) return rc;
    // hit and facet counts: each facet a set slot of its field's index
    BoolCount &count = out->count;
    if (in.out_total) {
        SA_CHECK(in.n_facets <= SA_BOOL_MAX_FACETS, "at most %d facets in one call, not %u", SA_BOOL_MAX_FACETS,
                 in.n_facets);
        SA_CHECK(in.n_facets == 0 || (in.facet_field && in.facet_slot && in.out_facet_counts), "NULL argument");
        for (u32 i = 0; i < in.n_facets; i++) {
            const u32 f = in.facet_field[i], slot = in.facet_slot[i];
            SA_CHECK(f < n_fields, "facet %u: field %u out of range (%u fields)", i, f, n_fields);
            SA_CHECK(slot < SA_MAX_FACETS && (X.ix[f]->facet_set >> slot & 1u), "facet %u: facet slot %u is not set",
                     i, slot);
            count.codes[i] = X.ix[f]->d_facets[slot].as<const unsigned short>();
            count.offset[i + 1] = count.offset[i] + X.ix[f]->facet_buckets[slot];
        }
        count.n_facets = in.n_facets;
        count.n_bins = count.offset[in.n_facets];
    }
    const u32 c_begin = n_nodes ? starts[0] : 0, c_end = n_nodes ? starts[n_nodes] : 0;
    for (u32 c = c_begin; c < c_end; c++) {
        if (in.nested(c)) continue;
        const u32 nt = in.n_terms(c);
        SA_CHECK(in.clause_term_starts[c + 1] > in.clause_term_starts[c], "clause %u: bad number of terms", c);
        const BoolKind kind = in.kind(c);
        SA_CHECK(kind == KIND_IN || nt <= SA_MAX_PHRASE_TERMS, "clause %u: bad number of terms", c);
        const u32 f = in.field(c);
        SA_CHECK(f < n_fields, "clause %u: field %u out of range (%u fields)", c, f, n_fields);
        const u32 *tids = in.terms(c);
        if (kind >= KIND_FEATURE) {
            if (kind == KIND_FEATURE) rc = bool_check_feature(X.ix[f], c, tids[0], in.clause_idf[c]);
            else if (kind == KIND_RANGE) rc = bool_check_range(X.ix[f], c, tids, nt, in.clause_idf[c]);
            else rc = bool_check_in(X.ix[f], c, tids, nt, in.clause_idf[c]);
            if (rc) return rc;
            SA_CHECK(!dismax || ((c == c_begin || in.clause_group[c - 1] != in.clause_group[c]) &&
                                 (c + 1 == c_end || in.clause_group[c + 1] != in.clause_group[c])),
                     "clause %u: a feature clause is not a DisMax member", c);
            out->features = true;
            continue;
        }
        for (u32 i = 0; i < nt; i++)
            SA_CHECK(!bool_is_feature_term(tids[i]), "clause %u: a feature term id inside a phrase", c);
        if ((rc = sa_check_term_ids(X.ix[f], tids, nt))) return rc;
    }
    // .score is all zeros on a field whose avgdl is 0: its clauses are empty (bool_plan), and without any other field
    // nothing ranks
    bool any_avgdl = false;
    for (u32 f = 0; f < n_fields; f++) any_avgdl = any_avgdl || X.avgdl[f] != 0.0f;
    out->empty = n_queries == 0 || X.lead()->n_docs == 0 || (!any_avgdl && !out->features);
    if (out->empty) return SA_OK;
    for (u32 n = 0; n < n_nodes; n++) {
        for (u32 c = starts[n]; c < starts[n + 1]; c++) {
            const u32 f = in.field(c);
            if (in.nested(c) || in.column(c) || X.avgdl[f] == 0.0f) continue;
            const bool sparse = bool_sparse(X, f, in.clause_idf[c]);
            SA_CHECK(in.n_terms(c) == 1 || sparse, "phrase queries in a batch need ordinary BM25 parameters (k1 > 0, 0 <= b < 1, finite idf)");
            SA_CHECK(!in.member(c, starts[n], starts[n + 1]) || sparse, "clause %u: DisMax members need ordinary BM25 "
                     "parameters (k1 > 0, 0 <= b < 1, finite idf >= 0)", c);
        }
    }
    return SA_OK;
}

// Where the descriptor arrays of P go in BoolState::desc.
BoolDescs bool_descs(const BoolPlan &P, size_t n_fields) {
    size_t end = 0;
    auto section = [&](size_t bytes) {
        const size_t at = end;
        end = (at + bytes + 255) & ~(size_t)255;
        return at;
    };
    BoolDescs L;
    L.clauses = section(P.clauses.size() * sizeof(BoolClause));
    L.queries = section(P.queries.size() * sizeof(BoolQuery));
    L.occur = section(P.occur.size() * sizeof(BoolOccur));
    L.groups = section(P.groups.size() * sizeof(BoolGroup));
    L.nest = section(P.nest.size() * sizeof(u32));
    L.fields = section((P.form >= BOOL_FIELDS ? n_fields : 0) * sizeof(BoolField));
    L.features = section(P.features.size() * sizeof(BoolFeature));
    L.sets = section(P.sets.size() * sizeof(u32));
    L.bytes = end;
    return L;
}

// The launches of a checked call and its descriptors, on the host: the form, the launch groups (at most ~1 GB of
// candidate slots and ~4 GB of phrase rows each), the row numbering and the per-clause arrays.  It makes no CUDA API
// call and takes no d_norm pointer: bool_upload's sa_ensure_norm may move d_norm.
BoolPlan bool_plan(const BoolCall &X, const BoolInput &in, const BoolChecked &chk) {
    const u32 n_nodes = in.n_nodes, n_queries = in.n_queries, n_fields = (u32)X.ix.size();
    const u32 *starts = in.node_clause_starts;
    const bool occur = in.clause_occur != nullptr, dismax = in.clause_group != nullptr;
    // an Or / And batch with a feature clause, or counts without collapsing (whose Or / And instance counts), runs as
    // roles and weights, every clause SHOULD with weight 1
    const bool roles = occur || chk.features || (in.out_total != nullptr && !in.groups);
    auto role = [&](u32 c) {
        return occur ? BoolOccur{in.clause_weight[c], in.clause_occur[c]} : BoolOccur{1.0f, SA_OCCUR_SHOULD};
    };
    BoolPlan P;
    const u32 n_tiles = sa_n_tiles(X.lead()->n_docs);
    P.slots = in.groups ? in.k : sa_topk_slots(in.k);     // a collapse tile keeps its k best leaders
    const u64 stride = sa_padded_docs(X.lead()->n_docs);
    const u32 group_q = (u32)std::min<u64>(65535, std::max<u64>(1, (1ull << 30) / ((u64)n_tiles * (P.slots * sizeof(u64) + 8))));
    const u32 group_rows = (u32)std::max<u64>(1, (4ull << 30) / (stride * sizeof(float)));
    P.form = in.clause_node ? BOOL_NESTED : dismax ? BOOL_DISMAX : X.fields_kernel ? BOOL_FIELDS : roles ? BOOL_OCCUR : BOOL_OR_AND;
    P.root.resize(n_nodes);
    P.depth.assign(n_nodes, 0);
    // every node's top-level query and depth (references point forward, so a holder is seen before its children), and
    // the rows each top-level query needs: its phrase leaves and its nested nodes
    std::vector<u32> q_rows(n_queries, 0);
    for (u32 n = 0; n < n_nodes; n++) {
        if (n < n_queries) P.root[n] = n;
        else q_rows[P.root[n]]++;
        for (u32 c = starts[n]; c < starts[n + 1]; c++) {
            if (in.nested(c)) {
                P.root[in.clause_node[c]] = P.root[n];
                P.depth[in.clause_node[c]] = P.depth[n] + 1;
                continue;
            }
            q_rows[P.root[n]] += in.kind(c) == KIND_PHRASE && X.avgdl[in.field(c)] != 0.0f;
        }
    }
    P.group_start.push_back(0);
    std::vector<u32> group_of(n_queries), g_rows;       // per launch group: its rows so far
    u32 rows = 0;
    for (u32 q = 0; q < n_queries; q++) {
        if (q > P.group_start.back() && (q - P.group_start.back() == group_q || rows + q_rows[q] > group_rows)) {
            P.group_start.push_back(q);
            rows = 0;
        }
        rows += q_rows[q];
        group_of[q] = (u32)P.group_start.size() - 1;
        P.max_rows = std::max(P.max_rows, rows);
    }
    P.group_start.push_back(n_queries);
    g_rows.assign(P.group_start.size() - 1, 0);
    // the nested nodes' rows first (a parent's clause names its child's row), then the phrase rows
    std::vector<u32> node_row(n_nodes, 0);
    for (u32 n = n_queries; n < n_nodes; n++) {
        P.nested.push_back(n);
        node_row[n] = g_rows[group_of[P.root[n]]]++;
    }
    std::stable_sort(P.nested.begin(), P.nested.end(), [&](u32 x, u32 y) {
        const u32 gx = group_of[P.root[x]], gy = group_of[P.root[y]];
        if (gx != gy) return gx < gy;
        if (P.depth[x] != P.depth[y]) return P.depth[x] > P.depth[y];
        return P.root[x] < P.root[y];
    });
    P.queries.resize(n_queries);                      // then the nested nodes' descriptors, in P.nested's order
    P.field_sparse.assign(n_fields, 0);
    const u32 c_end = n_nodes ? starts[n_nodes] : 0;
    for (u32 q = 0; q < n_nodes; q++) {
        const u32 c0 = starts[q], c1 = starts[q + 1];
        u32 &next_row = g_rows[group_of[P.root[q]]];
        if (q < n_queries) P.queries[q] = BoolQuery{(u32)P.clauses.size(), c1 - c0, in.mm[q], 0};
        for (u32 c = c0; c < c1; c++) {
            if (in.clause_node) P.nest.push_back(in.nested(c) ? 1u : 0u);
            if (in.nested(c)) {             // scored by its child's row, present where the child ranks
                P.occur.push_back(role(c));
                P.groups.push_back(BoolGroup{0.0f, c - c0, 0u, 0u});
                P.clauses.push_back(BoolClause{0, 0, SA_NO_DIR, SA_NO_DIR, 0.0f, node_row[in.clause_node[c]], 1u, 0u});
                continue;
            }
            const u32 f = in.field(c);
            sa_index *ix = X.ix[f];
            const u32 *tids = in.terms(c);
            const u32 nt = in.n_terms(c);
            if (roles) P.occur.push_back(role(c));
            // a member of a group of two or more: scores >= +0 everywhere (sparse-safe), which its max relies on
            const bool member = in.member(c, c0, c1);
            if (dismax)
                P.groups.push_back(BoolGroup{in.clause_tie[in.clause_group[c]], in.clause_group[c] - c0, member ? 1u : 0u,
                                             member && (c + 1 == c1 || in.clause_group[c + 1] != in.clause_group[c]) ? 1u : 0u});
            if (in.column(c)) {             // its column on its field's index
                const u32 slot = tids[0] & 0xFFu, fn = (tids[0] >> 8) & 0xFFFFu;
                P.features.resize(c_end);
                BoolFeature &bf = P.features[P.clauses.size()];
                bf.fn = fn;
                if (fn == SA_FEATURE_IN) {
                    bf.codes = ix->d_facets[slot].as<const unsigned short>();
                    bf.tiles = ix->d_facet_tiles[slot].as<u32>();
                    const size_t at = P.sets.size();
                    P.sets.resize(at + SA_FACET_SET_WORDS, 0u);
                    for (u32 i = 1; i < nt; i++) P.sets[at + (tids[i] >> 5)] |= 1u << (tids[i] & 31);
                } else {
                    bf.values = ix->d_features[slot].as<float>();
                    bf.tiles = ix->d_feature_tiles.as<u32>() + (size_t)slot * n_tiles;
                    bf.param = in.clause_idf[c];
                    if (fn == SA_FEATURE_RANGE) {
                        bf.bounds = ix->d_feature_bounds.as<float2>() + (size_t)slot * n_tiles;
                        memcpy(&bf.lo, tids + 1, sizeof(float));
                        memcpy(&bf.hi, tids + 2, sizeof(float));
                    }
                }
                P.clauses.push_back(BoolClause{0, 0, SA_NO_DIR, SA_NO_DIR, 0.0f, SA_BOOL_FEATURE_ROW, 1u, f});
                continue;
            }
            if (X.avgdl[f] == 0.0f) {       // scores +0 at every doc: no list, no row
                P.clauses.push_back(BoolClause{0, 0, SA_NO_DIR, SA_NO_DIR, in.clause_idf[c], SA_BOOL_NO_ROW, 1u, f});
                continue;
            }
            const bool sparse = bool_sparse(X, f, in.clause_idf[c]);   // phrases and members are (bool_check)
            const TermQuery tq = make_term_query(ix, nt == 1 ? tids[0] : SA_NO_TERM, in.clause_idf[c]);
            P.clauses.push_back(BoolClause{tq.word_off, tq.n_words, tq.dir_off, tq.rec_off, in.clause_idf[c],
                                           nt == 1 ? SA_BOOL_NO_ROW : next_row++, sparse ? 1u : 0u, f});
            P.field_sparse[f] = P.field_sparse[f] || sparse;
        }
    }
    for (u32 n : P.nested)
        P.queries.push_back(BoolQuery{starts[n], starts[n + 1] - starts[n], in.mm[n], node_row[n]});
    P.count = chk.count;
    P.descs = bool_descs(P, n_fields);
    P.result = BoolResult{(size_t)n_queries * in.k, n_queries, chk.count.n_bins, in.out_total != nullptr};
    return P;
}

// The call's buffers, the norms of its sparse-safe fields, the descriptors in one copy (the field table after the
// norms: sa_ensure_norm may move d_norm), the mask (*where), the DisMax shared memory, and zeroed flags and counts.
int bool_upload(const BoolCall &X, const BoolInput &in, const BoolPlan &P, WhereMask *where) {
    sa_index *lead = X.lead();
    BoolState &S = *X.S;
    const u32 n_fields = (u32)X.ix.size(), n_tiles = sa_n_tiles(lead->n_docs);
    const u64 stride = sa_padded_docs(lead->n_docs);
    int rc;
    if ((rc = S.desc.reserve(P.descs.bytes)) || (rc = S.d_keys.reserve(P.result.bytes())) ||
        (rc = S.rows.reserve(std::max<size_t>((size_t)P.max_rows * stride * sizeof(float), 64))) ||
        (rc = S.d_flags.reserve(P.form == BOOL_NESTED ? (size_t)P.max_rows * n_tiles * sizeof(u32) : 0)) ||
        (rc = X.h_pinned->reserve(P.result.bytes())))
        return rc;
    for (u32 f = 0; f < n_fields; f++)
        if (P.field_sparse[f] && (rc = sa_ensure_norm(X.ix[f], X.k1[f], X.b[f], X.avgdl[f]))) return rc;
    std::vector<char> staged(P.descs.bytes, 0);
    auto put = [&](size_t at, const auto &v) {
        if (!v.empty()) memcpy(staged.data() + at, v.data(), v.size() * sizeof(v[0]));
    };
    put(P.descs.clauses, P.clauses);
    put(P.descs.queries, P.queries);
    put(P.descs.occur, P.occur);
    put(P.descs.groups, P.groups);
    put(P.descs.nest, P.nest);
    // each In clause's set in the descriptors, and the call's skip counter in its result block
    std::vector<BoolFeature> feats(P.features);
    size_t n_sets = 0;
    for (BoolFeature &f : feats) {
        f.skipped = P.result.skipped(S.d_keys.p);
        if (f.codes) f.set = (const u32 *)(S.desc.as<const char>() + P.descs.sets) + SA_FACET_SET_WORDS * n_sets++;
    }
    put(P.descs.features, feats);
    put(P.descs.sets, P.sets);
    if (P.form >= BOOL_FIELDS) {
        std::vector<BoolField> fields;
        for (u32 f = 0; f < n_fields; f++) {
            sa_index *ix = X.ix[f];
            fields.push_back(BoolField{ix->d_words.as<u64>(), ix->d_tile_dir.as<u32>(), ix->d_recs.as<u32>(),
                                       ix->d_rec_dir.as<u32>(), ix->d_norm.as<float>(), ix->d_doc_lens.as<float>(),
                                       make_bm25(1.0f, X.avgdl[f], X.k1[f], X.b[f], ix->doc_lens_nonneg)});
        }
        put(P.descs.fields, fields);
    }
    SA_CUDA(cudaMemcpyAsync(S.desc.p, staged.data(), staged.size(), cudaMemcpyHostToDevice, lead->stream));
    if ((rc = sa_where_upload(lead, S.d_where, in.where_bits, lead->n_docs, in.where_stride, in.n_queries, where)))
        return rc;
    if (P.form >= BOOL_DISMAX) {
        // the first pass's variant and that of the store passes and re-runs, each masked only when the call is
        const BoolVariant first = bool_variant(P, in.out_total != nullptr), rest = bool_variant(P, false);
        for (int masked = 0; masked <= (where->bits != nullptr); masked++)
            if ((rc = bool_set_smem(bool_kernel(P.form, masked, first, in.k > SA_TOPK_MAX), SA_BOOL_DISMAX_SMEM)) ||
                (rest != first &&
                 (rc = bool_set_smem(bool_kernel(P.form, masked, rest, in.k > SA_TOPK_MAX), SA_BOOL_DISMAX_SMEM))))
                return rc;
    }
    for (int masked = 0; in.groups && masked <= (where->bits != nullptr); masked++)
        if ((rc = bool_set_smem(bool_kernel(P.form, masked, BOOL_COLLAPSE, false), bool_smem(P.form, true)))) return rc;
    SA_CUDA(cudaMemsetAsync(P.result.ovf(S.d_keys.p), 0, P.result.bytes() - P.result.n_keys * sizeof(u64),
                            lead->stream));
    return SA_OK;
}

// The result block in one device-to-host copy and one synchronise: the keys into out_docs / out_scores and the counts
// into out_total / out_facet_counts.  Then a query whose tile overflowed is re-run alone with a slot per doc of the
// tile, which cannot overflow, and without counting: its first pass has counted it.
int bool_collect(const BoolCall &X, const BoolPlan &P, const BoolInput &in, const WhereMask &where) {
    sa_index *lead = X.lead();
    const BoolResult &R = P.result;
    void *d = X.S->d_keys.p, *h = X.h_pinned->p;
    const u32 nq = in.n_queries, k = in.k;
    int rc;
    SA_CUDA(cudaMemcpyAsync(h, d, R.bytes(), cudaMemcpyDeviceToHost, lead->stream));
    SA_CUDA(cudaStreamSynchronize(lead->stream));
    const std::vector<u32> ovf(R.ovf(h), R.ovf(h) + nq);
    sa_unpack_keys(R.keys(h), R.n_keys, in.out_docs, in.out_scores);
    lead->stats.filter_tiles += *R.skipped(h);
    lead->stats.collapse_windows += *R.windows(h);
    if (R.counting) {
        memcpy(in.out_total, R.total(h), (size_t)nq * sizeof(u32));
        if (R.n_bins) memcpy(in.out_facet_counts, R.counts(h), (size_t)nq * R.n_bins * sizeof(u32));
    }
    u32 redone = 0;
    for (u32 q = 0; q < nq; q++) {
        if (!ovf[q]) continue;
        SA_CUDA(cudaMemsetAsync(R.ovf(d) + q, 0, sizeof(u32), lead->stream));
        if ((rc = bool_run_group(X, P, in, where, SA_TILE_DOCS, q, q + 1, false))) return rc;
        SA_CUDA(cudaMemcpyAsync(h, R.keys(d) + (size_t)q * k, k * sizeof(u64), cudaMemcpyDeviceToHost, lead->stream));
        SA_CUDA(cudaStreamSynchronize(lead->stream));
        sa_unpack_keys(R.keys(h), k, in.out_docs + (size_t)q * k, in.out_scores + (size_t)q * k);
        redone++;
    }
    if (in.n_redone) *in.n_redone = redone;
    return SA_OK;
}

// Both entry points, with the call's indexes locked and their device current: the refusals, the outputs filled as
// for no match, then the plan, its upload, the launch groups and the results.
int bool_topk(const BoolCall &X, const BoolInput &in) {
    BoolChecked chk;
    int rc;
    if ((rc = bool_check(X, in, &chk))) return rc;
    const size_t nk = (size_t)in.n_queries * in.k;
    for (size_t i = 0; i < nk; i++) { in.out_docs[i] = SA_NO_DOC; in.out_scores[i] = 0.0f; }
    if (in.out_total) {
        memset(in.out_total, 0, (size_t)in.n_queries * sizeof(u32));
        if (chk.count.n_bins) memset(in.out_facet_counts, 0, (size_t)in.n_queries * chk.count.n_bins * sizeof(u32));
    }
    if (chk.empty) return SA_OK;
    const BoolPlan P = bool_plan(X, in, chk);
    WhereMask where;
    if ((rc = bool_upload(X, in, P, &where))) return rc;
    for (size_t i = 0; i + 1 < P.group_start.size(); i++)
        if ((rc = bool_run_group(X, P, in, where, P.slots, P.group_start[i], P.group_start[i + 1],
                                 in.out_total != nullptr))) return rc;
    return bool_collect(X, P, in, where);
}

// The most nested nodes one top-level query of sa_score_docs_bool may hold (query.SA_BOOL_MAX_NESTED): the kernel keeps
// their values per thread in dynamic shared memory, 64 x 256 floats at most.
#define SA_BOOL_DOCS_MAX_NESTED 64

// sa_score_docs_bool reads the phrase clauses' count rows and no nested node's: the phrase rows alone, numbered within
// launch groups of at most ~4 GB of rows, replace the plan's rows and groups (whose group size also bounds top-k
// candidate memory, which scoring at docs has none of).
void bool_docs_rows(const BoolCall &X, const BoolInput &in, BoolPlan &P) {
    const u32 n_queries = in.n_queries;
    const u64 stride = sa_padded_docs(X.lead()->n_docs);
    const u64 group_rows = std::max<u64>(1, (4ull << 30) / (stride * sizeof(float)));
    std::vector<std::vector<u32>> nodes(n_queries);                  // each top-level query's nodes
    for (u32 q = 0; q < n_queries; q++) nodes[q].push_back(q);
    for (u32 n : P.nested) nodes[P.root[n]].push_back(n);
    auto phrase = [&](u32 c) {
        const u32 row = P.clauses[c].row;
        return row != SA_BOOL_NO_ROW && row != SA_BOOL_FEATURE_ROW && !in.nested(c);
    };
    P.group_start.assign(1, 0);
    P.max_rows = 0;
    u64 rows = 0;
    for (u32 q = 0; q < n_queries; q++) {
        u64 need = 0;
        for (u32 n : nodes[q])
            for (u32 c = in.node_clause_starts[n]; c < in.node_clause_starts[n + 1]; c++) need += phrase(c);
        if (q > P.group_start.back() && rows + need > group_rows) {
            P.group_start.push_back(q);
            rows = 0;
        }
        for (u32 n : nodes[q])
            for (u32 c = in.node_clause_starts[n]; c < in.node_clause_starts[n + 1]; c++)
                if (phrase(c)) P.clauses[c].row = (u32)rows++;
        P.max_rows = std::max(P.max_rows, (u32)rows);
    }
    P.group_start.push_back(n_queries);
}

// Both score-docs entry points, with the call's indexes locked and their device current: the refusals, the outputs
// zeroed, then the plan with phrase rows alone, its upload, the nested nodes' lists and the docs in two copies, per
// launch group its phrase rows and one bool_docs_kernel launch, and the scores in one copy.
int bool_score_docs(const BoolCall &X, const BoolInput &in, const u32 *docs, u32 n_per, float *out) {
    sa_index *lead = X.lead();
    BoolState &S = *X.S;
    const u32 nq = in.n_queries;
    const u64 n = (u64)nq * n_per;
    BoolChecked chk;
    int rc;
    if ((rc = bool_check(X, in, &chk))) return rc;
    SA_CHECK(n < (1ull << 31), "n_queries * n_per_query (%llu) must be below 2^31", (unsigned long long)n);
    for (u64 i = 0; i < n; i++)
        SA_CHECK(docs[i] == SA_NO_DOC || (docs[i] >= lead->doc_base && docs[i] - lead->doc_base < lead->n_docs),
                 "docs[%llu] = %u is neither SA_NO_DOC nor a doc of the index ([%llu, %llu))", (unsigned long long)i,
                 docs[i], (unsigned long long)lead->doc_base, (unsigned long long)(lead->doc_base + lead->n_docs));
    const u32 n_nodes = in.n_nodes;
    if (in.clause_node) {                  // each top-level query's nested nodes (references point forward)
        std::vector<u32> root(n_nodes), count(nq, 0);
        for (u32 node = 0; node < n_nodes; node++) {
            if (node < nq) root[node] = node;
            else count[root[node]]++;
            for (u32 c = in.node_clause_starts[node]; c < in.node_clause_starts[node + 1]; c++)
                if (in.nested(c)) root[in.clause_node[c]] = root[node];
        }
        for (u32 q = 0; q < nq; q++)
            SA_CHECK(count[q] <= SA_BOOL_DOCS_MAX_NESTED, "query %u: at most %d nested nodes, not %u", q,
                     SA_BOOL_DOCS_MAX_NESTED, count[q]);
    }
    std::fill(out, out + n, 0.0f);
    if (chk.empty || n == 0) return SA_OK;
    BoolPlan P = bool_plan(X, in, chk);
    bool_docs_rows(X, in, P);
    WhereMask where;
    if ((rc = bool_upload(X, in, P, &where))) return rc;
    // node lists in P.nested's order (deepest first per query), slots by position, each nested clause's child slot
    std::vector<u32> node_start(nq + 1, 0), node_list, child;
    size_t max_nested = 0;
    if (in.clause_node) {
        std::vector<std::vector<u32>> per_q(nq);
        for (size_t i = 0; i < P.nested.size(); i++) per_q[P.root[P.nested[i]]].push_back((u32)i);
        std::vector<u32> slot(n_nodes, 0);
        for (u32 q = 0; q < nq; q++) {
            node_start[q] = (u32)node_list.size();
            for (u32 i : per_q[q]) {
                slot[P.nested[i]] = (u32)(node_list.size() - node_start[q]);
                node_list.push_back(nq + i);
            }
            max_nested = std::max(max_nested, per_q[q].size());
        }
        node_start[nq] = (u32)node_list.size();
        const u32 c_end = in.node_clause_starts[n_nodes];
        child.assign(c_end, 0);
        for (u32 c = 0; c < c_end; c++)
            if (in.nested(c)) child[c] = slot[in.clause_node[c]];
    }
    // d_docs: the docs, the scores, then node_start, node_list and child
    const size_t docs_at = 0, out_at = (n * 4 + 255) & ~(size_t)255, lists_at = out_at + ((n * 4 + 255) & ~(size_t)255);
    std::vector<u32> lists_h(node_start);
    lists_h.insert(lists_h.end(), node_list.begin(), node_list.end());
    lists_h.insert(lists_h.end(), child.begin(), child.end());
    if ((rc = S.d_docs.reserve(lists_at + lists_h.size() * sizeof(u32))) || (rc = X.h_pinned->reserve(n * 4)))
        return rc;
    char *dd = S.d_docs.as<char>();
    memcpy(X.h_pinned->p, docs, n * sizeof(u32));
    SA_CUDA(cudaMemcpyAsync(dd + docs_at, X.h_pinned->p, n * sizeof(u32), cudaMemcpyHostToDevice, lead->stream));
    if (in.clause_node)
        SA_CUDA(cudaMemcpyAsync(dd + lists_at, lists_h.data(), lists_h.size() * sizeof(u32), cudaMemcpyHostToDevice,
                                lead->stream));
    const char *d = S.desc.as<const char>();
    const u32 *lists_d = (const u32 *)(dd + lists_at);
    BoolDocs x;
    x.occ = P.form >= BOOL_OCCUR ? (const BoolOccur *)(d + P.descs.occur) : nullptr;
    x.fld = P.form >= BOOL_FIELDS ? (const BoolField *)(d + P.descs.fields) : nullptr;
    x.grp = P.form >= BOOL_DISMAX ? (const BoolGroup *)(d + P.descs.groups) : nullptr;
    x.feat = P.features.empty() ? nullptr : (const BoolFeature *)(d + P.descs.features);
    x.nest = in.clause_node ? (const u32 *)(d + P.descs.nest) : nullptr;
    x.node_start = lists_d;
    x.node_list = lists_d + nq + 1;
    x.child = x.node_list + node_list.size();
    x.docs = (const u32 *)(dd + docs_at);
    x.out = (float *)(dd + out_at);
    x.n_per = n_per;
    x.chunks = (n_per + SA_TERM_THREADS - 1) / SA_TERM_THREADS;
    const size_t smem = max_nested * SA_TERM_THREADS * sizeof(float);
    if (smem > 48 * 1024)
        SA_CUDA(cudaFuncSetAttribute(bool_docs_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const BoolArgs a = bool_args(X, P);
    for (size_t g = 0; g + 1 < P.group_start.size(); g++) {
        const u32 q0 = P.group_start[g], q1 = P.group_start[g + 1];
        if ((rc = bool_build_rows(X, P, in, q0, q1))) return rc;
        bool_docs_kernel<<<(q1 - q0) * x.chunks, SA_TERM_THREADS, smem, lead->stream>>>(a, x, q0);
        SA_CUDA(cudaGetLastError());
        lead->stats.total_launches++;
    }
    SA_CUDA(cudaMemcpyAsync(X.h_pinned->p, x.out, n * sizeof(float), cudaMemcpyDeviceToHost, lead->stream));
    SA_CUDA(cudaStreamSynchronize(lead->stream));
    memcpy(out, X.h_pinned->p, n * sizeof(float));
    return SA_OK;
}

// f(X) under the multi's lock, with its state and candidate buffer, and field 0's pinned staging.  Fields that share
// an index share its norm cache, which holds one parameter set; each index is locked once, in address order, and its
// stream swapped to the multi's for the whole call.
template <typename F>
int bool_multi_call(sa_multi *m, const float *avg_doc_len, const float *k1, const float *b, F f) {
    std::lock_guard<std::mutex> g(m->mu);
    SA_CUDA(cudaSetDevice(m->device));
    const u32 n_fields = (u32)m->fields.size();
    std::vector<sa_index *> distinct;
    for (u32 i = 0; i < n_fields; i++) {
        for (u32 e = 0; e < i; e++)
            SA_CHECK(m->fields[e] != m->fields[i] ||
                     (avg_doc_len[e] == avg_doc_len[i] && k1[e] == k1[i] && b[e] == b[i]),
                     "fields %u and %u share an index but not their BM25 parameters", e, i);
        if (std::find(distinct.begin(), distinct.end(), m->fields[i]) == distinct.end()) distinct.push_back(m->fields[i]);
    }
    std::sort(distinct.begin(), distinct.end());
    std::vector<std::unique_ptr<FieldGuard>> guards;
    for (sa_index *ix : distinct) guards.emplace_back(new FieldGuard(ix, m->stream));
    if (!m->boolq) m->boolq.reset(new BoolState());
    const BoolCall X{m->fields, std::vector<float>(avg_doc_len, avg_doc_len + n_fields),
                     std::vector<float>(k1, k1 + n_fields), std::vector<float>(b, b + n_fields), true, m->boolq.get(),
                     &m->cand, &m->fields[0]->h_pinned};
    return f(X);
}

}  // namespace

// bool_topk under the index's own lock, with its state and buffers; collapsed on the index's group column
// *group_slot where group_slot is not NULL.
static int bool_topk_index(sa_index *ix, const uint32_t *group_slot, uint32_t n_nodes,
                           const uint32_t *node_clause_starts, const uint32_t *clause_node, const uint32_t *clause_terms,
                           const uint32_t *clause_term_starts, const float *clause_idf, const float *clause_weight,
                           const uint8_t *clause_occur, const uint32_t *clause_group, const float *clause_tie,
                           const uint32_t *mm, uint32_t n_queries, uint32_t slop, float avg_doc_len, float k1, float b,
                           uint32_t k, const uint32_t *where_bits, uint64_t where_n, uint64_t where_stride,
                           uint32_t *out_docs, float *out_scores, uint32_t *n_redone, uint32_t n_facets,
                           const uint32_t *facet_field, const uint32_t *facet_slot, uint32_t *out_total,
                           uint32_t *out_facet_counts) {
    SA_CHECK(!clause_weight == !clause_occur, "clause_weight and clause_occur are both given or both NULL");
    SA_CHECK(!clause_group == !clause_tie && (!clause_group || clause_occur),
             "clause_group and clause_tie are both given (with clause_occur) or both NULL");
    SA_CHECK(clause_node ? clause_group != nullptr : n_nodes == n_queries,
             "clause_node needs the DisMax arrays; without it n_nodes == n_queries");
    SA_CHECK(ix && out_docs && out_scores, "NULL argument");
    SA_CHECK(n_nodes == 0 || (node_clause_starts && clause_terms && clause_term_starts && clause_idf && mm),
             "NULL argument");
    SA_CHECK(k >= 1 && k <= SA_TOPK_DEEP_MAX, "k must be in [1, %d]", SA_TOPK_DEEP_MAX);
    if (n_redone) *n_redone = 0;
    std::lock_guard<std::mutex> g(ix->mu);
    SA_CUDA(cudaSetDevice(ix->device));
    if (!ix->boolq) ix->boolq.reset(new BoolState());
    const BoolCall X{{ix}, {avg_doc_len}, {k1}, {b}, false, ix->boolq.get(), &ix->cand, &ix->h_pinned};
    BoolInput in{n_nodes, node_clause_starts, clause_node, nullptr, clause_terms, clause_term_starts, clause_idf,
                 clause_weight, clause_occur, clause_group, clause_tie, mm, n_queries, slop, k, where_bits,
                 where_n, where_stride, out_docs, out_scores, n_redone, n_facets, facet_field, facet_slot,
                 out_total, out_facet_counts, nullptr};
    if (group_slot) {
        SA_CHECK(*group_slot < SA_MAX_GROUPS && (ix->group_set >> *group_slot & 1u), "group slot %u is not set",
                 *group_slot);
        in.groups = ix->d_groups[*group_slot].as<const u32>();
    }
    return bool_topk(X, in);
}

extern "C" int sa_score_batch_topk_bool(sa_index *ix, uint32_t n_nodes, const uint32_t *node_clause_starts,
                                        const uint32_t *clause_node, const uint32_t *clause_terms,
                                        const uint32_t *clause_term_starts, const float *clause_idf,
                                        const float *clause_weight, const uint8_t *clause_occur,
                                        const uint32_t *clause_group, const float *clause_tie, const uint32_t *mm,
                                        uint32_t n_queries, uint32_t slop, float avg_doc_len, float k1, float b,
                                        uint32_t k, const uint32_t *where_bits, uint64_t where_n,
                                        uint64_t where_stride, uint32_t *out_docs, float *out_scores,
                                        uint32_t *n_redone, uint32_t n_facets, const uint32_t *facet_field,
                                        const uint32_t *facet_slot, uint32_t *out_total, uint32_t *out_facet_counts) {
    return bool_topk_index(ix, nullptr, n_nodes, node_clause_starts, clause_node, clause_terms, clause_term_starts,
                           clause_idf, clause_weight, clause_occur, clause_group, clause_tie, mm, n_queries, slop,
                           avg_doc_len, k1, b, k, where_bits, where_n, where_stride, out_docs, out_scores, n_redone,
                           n_facets, facet_field, facet_slot, out_total, out_facet_counts);
}

extern "C" int sa_score_batch_topk_bool_collapse(sa_index *ix, uint32_t group_slot, uint32_t n_nodes,
                                                 const uint32_t *node_clause_starts, const uint32_t *clause_node,
                                                 const uint32_t *clause_terms, const uint32_t *clause_term_starts,
                                                 const float *clause_idf, const float *clause_weight,
                                                 const uint8_t *clause_occur, const uint32_t *clause_group,
                                                 const float *clause_tie, const uint32_t *mm, uint32_t n_queries,
                                                 uint32_t slop, float avg_doc_len, float k1, float b, uint32_t k,
                                                 const uint32_t *where_bits, uint64_t where_n, uint64_t where_stride,
                                                 uint32_t *out_docs, float *out_scores, uint32_t *n_redone,
                                                 uint32_t n_facets, const uint32_t *facet_field,
                                                 const uint32_t *facet_slot, uint32_t *out_total,
                                                 uint32_t *out_facet_counts) {
    return bool_topk_index(ix, &group_slot, n_nodes, node_clause_starts, clause_node, clause_terms, clause_term_starts,
                           clause_idf, clause_weight, clause_occur, clause_group, clause_tie, mm, n_queries, slop,
                           avg_doc_len, k1, b, k, where_bits, where_n, where_stride, out_docs, out_scores, n_redone,
                           n_facets, facet_field, facet_slot, out_total, out_facet_counts);
}

// bool_topk under the multi's lock, with its state and candidate buffer; collapsed on group column group[1] of field
// group[0]'s index where group is not NULL.
static int bool_topk_multi(sa_multi *m, const uint32_t *group, uint32_t n_nodes, const uint32_t *node_clause_starts,
                           const uint32_t *clause_node, const uint32_t *clause_field, const uint32_t *clause_terms,
                           const uint32_t *clause_term_starts, const float *clause_idf, const float *clause_weight,
                           const uint8_t *clause_occur, const uint32_t *clause_group, const float *clause_tie,
                           const uint32_t *mm, uint32_t n_queries, uint32_t slop, const float *avg_doc_len,
                           const float *k1, const float *b, uint32_t k, const uint32_t *where_bits, uint64_t where_n,
                           uint64_t where_stride, uint32_t *out_docs, float *out_scores, uint32_t *n_redone,
                           uint32_t n_facets, const uint32_t *facet_field, const uint32_t *facet_slot,
                           uint32_t *out_total, uint32_t *out_facet_counts) {
    SA_CHECK(!clause_group == !clause_tie, "clause_group and clause_tie are both given or both NULL");
    SA_CHECK(clause_node ? clause_group != nullptr : n_nodes == n_queries,
             "clause_node needs the DisMax arrays; without it n_nodes == n_queries");
    SA_CHECK(m && out_docs && out_scores && avg_doc_len && k1 && b, "NULL argument");
    SA_CHECK(n_nodes == 0 || (node_clause_starts && clause_field && clause_terms && clause_term_starts &&
                                clause_idf && clause_weight && clause_occur && mm), "NULL argument");
    SA_CHECK(k >= 1 && k <= SA_TOPK_DEEP_MAX, "k must be in [1, %d]", SA_TOPK_DEEP_MAX);
    if (n_redone) *n_redone = 0;
    return bool_multi_call(m, avg_doc_len, k1, b, [&](const BoolCall &X) {
        BoolInput in{n_nodes, node_clause_starts, clause_node, clause_field, clause_terms, clause_term_starts,
                     clause_idf, clause_weight, clause_occur, clause_group, clause_tie, mm, n_queries, slop, k,
                     where_bits, where_n, where_stride, out_docs, out_scores, n_redone, n_facets, facet_field,
                     facet_slot, out_total, out_facet_counts, nullptr};
        if (group) {
            SA_CHECK(group[0] < X.ix.size(), "group field %u out of range (%u fields)", group[0], (u32)X.ix.size());
            SA_CHECK(group[1] < SA_MAX_GROUPS && (X.ix[group[0]]->group_set >> group[1] & 1u),
                     "group slot %u is not set on field %u", group[1], group[0]);
            in.groups = X.ix[group[0]]->d_groups[group[1]].as<const u32>();
        }
        return bool_topk(X, in);
    });
}

extern "C" int sa_multi_score_batch_topk_bool(sa_multi *m, uint32_t n_nodes, const uint32_t *node_clause_starts,
                                              const uint32_t *clause_node, const uint32_t *clause_field,
                                              const uint32_t *clause_terms, const uint32_t *clause_term_starts,
                                              const float *clause_idf, const float *clause_weight,
                                              const uint8_t *clause_occur, const uint32_t *clause_group,
                                              const float *clause_tie, const uint32_t *mm, uint32_t n_queries,
                                              uint32_t slop, const float *avg_doc_len, const float *k1, const float *b,
                                              uint32_t k, const uint32_t *where_bits, uint64_t where_n,
                                              uint64_t where_stride, uint32_t *out_docs, float *out_scores,
                                              uint32_t *n_redone, uint32_t n_facets, const uint32_t *facet_field,
                                              const uint32_t *facet_slot, uint32_t *out_total,
                                              uint32_t *out_facet_counts) {
    return bool_topk_multi(m, nullptr, n_nodes, node_clause_starts, clause_node, clause_field, clause_terms,
                           clause_term_starts, clause_idf, clause_weight, clause_occur, clause_group, clause_tie, mm,
                           n_queries, slop, avg_doc_len, k1, b, k, where_bits, where_n, where_stride, out_docs,
                           out_scores, n_redone, n_facets, facet_field, facet_slot, out_total, out_facet_counts);
}

extern "C" int sa_multi_score_batch_topk_bool_collapse(
    sa_multi *m, uint32_t group_field, uint32_t group_slot, uint32_t n_nodes, const uint32_t *node_clause_starts,
    const uint32_t *clause_node, const uint32_t *clause_field, const uint32_t *clause_terms,
    const uint32_t *clause_term_starts, const float *clause_idf, const float *clause_weight,
    const uint8_t *clause_occur, const uint32_t *clause_group, const float *clause_tie, const uint32_t *mm,
    uint32_t n_queries, uint32_t slop, const float *avg_doc_len, const float *k1, const float *b, uint32_t k,
    const uint32_t *where_bits, uint64_t where_n, uint64_t where_stride, uint32_t *out_docs, float *out_scores,
    uint32_t *n_redone, uint32_t n_facets, const uint32_t *facet_field, const uint32_t *facet_slot,
    uint32_t *out_total, uint32_t *out_facet_counts) {
    const uint32_t group[2] = {group_field, group_slot};
    return bool_topk_multi(m, group, n_nodes, node_clause_starts, clause_node, clause_field, clause_terms,
                           clause_term_starts, clause_idf, clause_weight, clause_occur, clause_group, clause_tie, mm,
                           n_queries, slop, avg_doc_len, k1, b, k, where_bits, where_n, where_stride, out_docs,
                           out_scores, n_redone, n_facets, facet_field, facet_slot, out_total, out_facet_counts);
}

// The value query q ranks doc docs[q * n_per_query + j] with, for each pair: bool_score_docs under the index's lock.
// Reference: postings.py:652 `score`, indexed at the candidates (arr.score(q)[docs[q]]).
extern "C" int sa_score_docs_bool(sa_index *ix, uint32_t n_nodes, const uint32_t *node_clause_starts,
                                  const uint32_t *clause_node, const uint32_t *clause_terms,
                                  const uint32_t *clause_term_starts, const float *clause_idf,
                                  const float *clause_weight, const uint8_t *clause_occur,
                                  const uint32_t *clause_group, const float *clause_tie, const uint32_t *mm,
                                  uint32_t n_queries, uint32_t slop, float avg_doc_len, float k1, float b,
                                  const uint32_t *docs, uint32_t n_per_query, float *out_scores) {
    SA_CHECK(!clause_weight == !clause_occur, "clause_weight and clause_occur are both given or both NULL");
    SA_CHECK(!clause_group == !clause_tie && (!clause_group || clause_occur),
             "clause_group and clause_tie are both given (with clause_occur) or both NULL");
    SA_CHECK(clause_node ? clause_group != nullptr : n_nodes == n_queries,
             "clause_node needs the DisMax arrays; without it n_nodes == n_queries");
    SA_CHECK(ix && ((u64)n_queries * n_per_query == 0 || (docs && out_scores)), "NULL argument");
    SA_CHECK(n_nodes == 0 || (node_clause_starts && clause_terms && clause_term_starts && clause_idf && mm),
             "NULL argument");
    std::lock_guard<std::mutex> g(ix->mu);
    SA_CUDA(cudaSetDevice(ix->device));
    if (!ix->boolq) ix->boolq.reset(new BoolState());
    const BoolCall X{{ix}, {avg_doc_len}, {k1}, {b}, false, ix->boolq.get(), &ix->cand, &ix->h_pinned};
    const BoolInput in{n_nodes, node_clause_starts, clause_node, nullptr, clause_terms, clause_term_starts, clause_idf,
                       clause_weight, clause_occur, clause_group, clause_tie, mm, n_queries, slop, 1, nullptr, 0, 0,
                       nullptr, nullptr, nullptr, 0, nullptr, nullptr, nullptr, nullptr};
    return bool_score_docs(X, in, docs, n_per_query, out_scores);
}

// sa_score_docs_bool over the fields of a multi, under its lock, as sa_multi_score_batch_topk_bool.
extern "C" int sa_multi_score_docs_bool(sa_multi *m, uint32_t n_nodes, const uint32_t *node_clause_starts,
                                        const uint32_t *clause_node, const uint32_t *clause_field,
                                        const uint32_t *clause_terms, const uint32_t *clause_term_starts,
                                        const float *clause_idf, const float *clause_weight,
                                        const uint8_t *clause_occur, const uint32_t *clause_group,
                                        const float *clause_tie, const uint32_t *mm, uint32_t n_queries,
                                        uint32_t slop, const float *avg_doc_len, const float *k1, const float *b,
                                        const uint32_t *docs, uint32_t n_per_query, float *out_scores) {
    SA_CHECK(!clause_group == !clause_tie, "clause_group and clause_tie are both given or both NULL");
    SA_CHECK(clause_node ? clause_group != nullptr : n_nodes == n_queries,
             "clause_node needs the DisMax arrays; without it n_nodes == n_queries");
    SA_CHECK(m && avg_doc_len && k1 && b && ((u64)n_queries * n_per_query == 0 || (docs && out_scores)),
             "NULL argument");
    SA_CHECK(n_nodes == 0 || (node_clause_starts && clause_field && clause_terms && clause_term_starts &&
                                clause_idf && clause_weight && clause_occur && mm), "NULL argument");
    return bool_multi_call(m, avg_doc_len, k1, b, [&](const BoolCall &X) {
        const BoolInput in{n_nodes, node_clause_starts, clause_node, clause_field, clause_terms, clause_term_starts,
                           clause_idf, clause_weight, clause_occur, clause_group, clause_tie, mm, n_queries, slop, 1,
                           nullptr, 0, 0, nullptr, nullptr, nullptr, 0, nullptr, nullptr, nullptr, nullptr};
        return bool_score_docs(X, in, docs, n_per_query, out_scores);
    });
}
