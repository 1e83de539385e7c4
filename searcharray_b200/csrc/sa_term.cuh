// sa_term.cuh -- kernel-side declarations shared by the term-path translation units, and the per-tile top-k
// collectors every scoring kernel ends with: flush_tile_collect for float32 scores, collect_tile_f64 for float64
// scores ranked by a float32 proxy (classic similarity, edismax).
#pragma once
#include <cmath>
#include <type_traits>

#include "sa_common.cuh"
#include "sa_scan.cuh"

#define SA_TILE_DOCS 8192          // docs per CTA tile (32 KB of float32 scores)
#define SA_TERM_UNROLL 4           // 30-word windows loaded per warp before processing
#define SA_TERM_THREADS 256
// The three tf-table knobs below were swept on H100 (DESIGN.md §3.1); these values were the fastest on the bench mix.
#define SA_STAGED_NORM_MIN_WORDS 1024   // tiles with at least this many posting words stage the tile's norms (sa_term.cu)
#define SA_STAGED_NORM_MIN_RECS 48      // ... or this many (doc, tf) records on the tf-table path
#define SA_TERM_CTAS_PER_SM 6           // resident term CTAs per SM (the launch bound); sets the L2 prefetch distance (sa_term.cu)
#define SA_TERM_DEEP_CTAS_PER_SM 5      // the same for the deep instances: 32 KB tile + 9.3 KB run and histogram each
#define SA_TERM_QUAD_MIN_RECS 512       // four records per thread from this many records per tile on (and >= 16 * k, sa_term.cu)
#define SA_TOPK_MAX 32             // warp-level threshold estimation handles k <= 32
// k in (SA_TOPK_MAX, SA_TOPK_DEEP_MAX] (searcharray_b200.h): each tile keeps its exact top k (deep_tile_collect)

enum TermMode { TERM_MODE_TF = 0, TERM_MODE_SCORE = 1 };

// Per-query top-k collection state in HBM (see sa_topk.cu).  No global atomics: every
// (query, tile) CTA owns `slots` candidate slots.
struct TopkCtx {
    u32 *tile_cnt;     // [Q][n_tiles] candidates written by the tile's CTA (<= slots)
    u32 *tile_max;     // [Q][n_tiles] score bits of the tile's best candidate (0 = none)
    u64 *tile_cand;    // [Q][n_tiles][slots] key = score_bits << 32 | (0xFFFFFFFF - local_doc)
    u32 *overflow;     // [Q] set when some tile had more than `slots` candidates
    u32 n_tiles;
    u32 slots;         // k on the deep path: a tile's candidates are then one run sorted by key, descending
    u32 k;             // 0 => no top-k collection
};

// A document mask of the batched top-k (the entry points' where_bits): one row of packed bits for the batch, or one per
// query.  The tile kernels that take it (bool_tile, sim_tile) have thread tid own docs 4 g .. 4 g + 3 of a tile,
// g = tid + j * SA_TERM_THREADS (flush_tile_collect's layout), so a row stores its bits in that owner order, not in
// doc order: word tile * SA_TERM_THREADS + tid holds, at bit 4 j + e, doc tile * SA_TILE_DOCS + 4 g + e.  A thread
// then reads its 32 bits as one u32 and a warp one 128-byte line; in doc order each thread would gather a nibble
// from each of 8 words.  Bits past the last doc are 0.
struct WhereMask {
    const u32 *bits;   // row 0 of the mask on the device; NULL: no mask
    u64 stride;        // words from one query's row to the next; 0: one row for every query
};

// The calling thread's 32 mask bits of `tile` in mask row `row`.  The thread index is read afresh (asm volatile):
// merged with the kernel's other reads, its 64-bit widening stayed live through the tile fold and spilled.
__device__ __forceinline__ u32 where_word(const WhereMask &w, u64 row, u32 tile) {
    unsigned tid;
    asm volatile("mov.u32 %0, %%tid.x;" : "=r"(tid));
    return __ldg(w.bits + row * w.stride + (u64)tile * SA_TERM_THREADS + tid);
}

struct TermBatchArgs {
    const u64 *words;
    const float *doc_lens;
    const float *norm;          // per-doc BM25 length norm (padded to a tile multiple), SCORE mode
    const u32 *tile_dir;        // tile directories (see sa_index::d_tile_dir)
    const u32 *recs;            // per-term (doc, tf) records (sa_index::d_recs) or NULL
    const u32 *rec_dir;         // record directories, same offsets as tile_dir
    u64 n_docs;
    u64 doc_base;
    const TermQuery *queries;   // [Q]
    float *out;                 // [Q][out_stride]
    u64 out_stride;             // multiple of SA_TILE_DOCS
    Bm25Params bm25;            // idf field unused (per query)
    u64 min_payload, max_payload;
    int filter;                 // apply the payload_slice filter
    int mode;
    u32 staged_norm_min_words;  // set by launch_term_batch
    u32 staged_norm_min_recs, quad_min_recs;   // set by launch_term_batch
    u32 prefetch_tiles;         // L2 prefetch distance in tiles on the tf-table path (0 = off); set by launch_term_batch
    // CTA order (set by launch_term_batch): CTA b of the 1-D grid of n_queries * n_tiles walks the rows in groups of
    // `group` consecutive queries, the queries of a group fastest, then the tiles, then the groups (sa_term.cu)
    u32 n_queries, n_tiles, group, group_ctas;   // group_ctas = group * n_tiles
    TopkCtx topk;
};

// group: the CTA order's query-group width G (0 = every query, the (queries, tiles) order).  G = 1 walks each row's
// tiles back to back; SA_TERM_QUERY_MAJOR=1 forces it for every launch.
int launch_term_batch(sa_index *ix, const TermBatchArgs &a, u32 n_queries, u32 group = 0);
int sa_ensure_norm(sa_index *ix, float k1, float b, float avg_doc_len);
int launch_topk_select(sa_index *ix, const TopkCtx &t, u32 n_queries, u64 doc_base, u64 *d_out_keys,
                       const u32 *d_out_index);
u32 sa_topk_slots(u32 k);
// The collapsed top k of each query from the runs of collapse_tile_collect (tile slots == k): the k best distinct
// groups' leaders, keys as topk_select_kernel writes them to d_out_keys[q * k ..]; groups: the group column
// (index-local ids); *d_windows counts the walk's windows past the first (see sa_topk.cu).
int launch_topk_collapse(sa_index *ix, const TopkCtx &t, u32 n_queries, u64 doc_base, const u32 *groups,
                         u64 *d_out_keys, u32 *d_windows);
// Slots of a tile of collect_tile_f64: `shallow` for k <= SA_TOPK_MAX, max(k, 256) above (the deep bound keeps the k
// best keys plus their ties)
inline u32 sa_topk_slots_f64(u32 k, u32 shallow) { return k > SA_TOPK_MAX ? std::max(k, 256u) : shallow; }
// topk_select_kernel for candidates whose key carries a float32 proxy of a float64 score (d_tile_d: the score bits,
// slot for slot); exact in float64, see sa_topk.cu.  d_out_scores[out_index[q] * k + i] = the float64 scores.
int launch_topk_select_f64(sa_index *ix, const TopkCtx &t, const u64 *d_tile_d, u32 n_queries, u64 doc_base,
                           u64 *d_out_keys, double *d_out_scores, const u32 *d_out_index);
// sim_tile_kernel<kind> (sa_view.cu) over n doc-space count rows of ix->dense's stride: counts + j * stride is row j,
// d_idf[j] its idf, row row0 + j of t takes its candidates.  Position i < n_pos reads its count at doc rows[i] (rows ==
// NULL: doc i) and its doc length from doc_lens as sim_tile_kernel describes.  bm25 / sim: the parameters of the
// kind; tile_d: the float64 candidate scores (SA_SIM_CLASSIC only).
struct SimParams;
// wh (sim_where_tile_kernel): position i ranks only where its mask bit is set, in the mask row of query
// d_row_query[j] for row j.
int launch_sim_tiles(sa_index *ix, int kind, const float *counts, const u64 *rows, const float *doc_lens, u64 n_pos,
                     const Bm25Params &bm25, const SimParams &sim, const double *d_idf, u32 n, u32 row0,
                     const TopkCtx &t, u64 *tile_d, const WhereMask &wh = WhereMask{nullptr, 0},
                     const u32 *d_row_query = nullptr);
int launch_topk_merge(sa_index *ix, const u64 *d_in, u64 rank_stride, u32 world, u32 n_queries, u32 k, u64 *d_out);
// A batch's result block in HBM: nq * k keys followed by SA_BATCH_TAIL summary words written by the batch's last
// kernel -- [0] queries that need the exact host-side re-run (candidate overflow, wrong same-term guess, scratch
// exhausted), [1] continuation words and [2] matched docs of the phrase queries (roofline accounting).  The tail
// travels with the keys (one D2H; one all-gather when sharded), so a clean batch costs ONE stream synchronise.
#define SA_BATCH_TAIL 4
int sa_batch_download_locked(sa_index *ix, uint32_t *out_docs, float *out_scores, uint32_t *n_overflow);
// batch plumbing shared by sa_index.cu / sa_comm.cu (callers hold ix->mu)
int sa_batch_upload_locked(sa_index *ix, const uint32_t *terms, const uint32_t *term_starts,
                           const float *idf, uint32_t n_queries, uint32_t slop,
                           float avg_doc_len, float k1, float b, uint32_t k);
int sa_batch_execute_locked(sa_index *ix);
int sa_batch_fix_overflow_locked(sa_index *ix, u32 *n_redone);
void sa_batch_dims(sa_index *ix, u32 *nq, u32 *k);
void sa_unpack_keys(const u64 *keys, u64 n, uint32_t *out_docs, float *out_scores);
int sa_filter_terms(sa_index *ix, const uint32_t *term_ids, uint32_t n_terms, bool use_rows,
                    u64 pay_lo, u64 pay_hi, bool use_payload, std::vector<u64> &offs, std::vector<u64> &lens);
int sa_filter_terms_mask(sa_index *ix, const uint32_t *term_ids, uint32_t n_terms, const unsigned char *d_mask,
                         u64 pay_lo, u64 pay_hi, bool use_payload, std::vector<u64> &offs, std::vector<u64> &lens,
                         std::vector<u64> *df_out);
// Dense row 0 of ix->dense to the host (the selected rows only, when a row filter is installed), synchronously.
int sa_copy_out_dense(sa_index *ix, float *out_host);

// ---- host-side query set-up shared by every entry point
// Dense rows are padded to whole tiles.
inline u32 sa_n_tiles(u64 n_docs) { return (u32)((n_docs + SA_TILE_DOCS - 1) / SA_TILE_DOCS); }
inline u64 sa_padded_docs(u64 n_docs) { return (u64)sa_n_tiles(n_docs) * SA_TILE_DOCS; }
static_assert(SA_WHERE_WORDS(1) == SA_TERM_THREADS && SA_WHERE_WORDS(SA_TILE_DOCS + 1) == 2 * SA_TERM_THREADS,
              "a WhereMask row is SA_TERM_THREADS words per tile");
// The entry points' mask arguments against the n docs (positions) the call ranks, on the host: where_bits
// NULL (no mask), or where_n == n and where_stride 0 or SA_WHERE_WORDS(n).
int sa_where_check(const uint32_t *where_bits, uint64_t where_n, uint64_t where_stride, u64 n);
// A checked mask's rows over n docs (one, or n_queries when where_stride != 0) into buf on ix->stream; *out addresses
// them (bits NULL without a mask).
int sa_where_upload(sa_index *ix, DevBuf &buf, const uint32_t *where_bits, u64 n, uint64_t where_stride, u32 n_queries,
                    WhereMask *out);

inline Bm25Params make_bm25(float idf, float avg_doc_len, float k1, float b, bool doc_lens_nonneg) {
    Bm25Params p;
    p.idf = idf;
    p.avg_doc_len = avg_doc_len;
    p.k1 = k1;
    p.b = b;
    p.one_minus_b = 1 - b;       // float arithmetic, as `cdef float one_minus_b = 1 - b` (bm25.pyx:19)
    p.sparse_ok = (doc_lens_nonneg && k1 > 0.0f && std::isfinite(k1) && b >= 0.0f && b < 1.0f &&
                   avg_doc_len > 0.0f && std::isfinite(avg_doc_len) && std::isfinite(idf) &&
                   idf >= 0.0f && !std::signbit(idf)) ? 1 : 0;
    return p;
}

// Every id is SA_NO_TERM or a term of the index.
inline int sa_check_term_ids(const sa_index *ix, const u32 *term_ids, u32 n) {
    for (u32 i = 0; i < n; i++)
        SA_CHECK(term_ids[i] == SA_NO_TERM || term_ids[i] < ix->n_terms, "term id %u out of range", term_ids[i]);
    return SA_OK;
}

// The index's lists of a query's terms (offsets, lengths, tile directories).  *missing: some term is SA_NO_TERM or has
// an empty list, so the query matches nothing; every list is then reported empty.  *literal: every list starts with a
// word at (doc 0, block 0), the span search's replayed corner (SpanQuery::literal).
inline int sa_resolve_terms(const sa_index *ix, const u32 *term_ids, u32 n, u64 *offs, u64 *lens, u64 *dirs,
                            bool *missing, bool *literal) {
    int rc = sa_check_term_ids(ix, term_ids, n);
    if (rc) return rc;
    *missing = false;
    for (u32 i = 0; i < n; i++)
        if (term_ids[i] == SA_NO_TERM || ix->h_len[term_ids[i]] == 0) *missing = true;
    *literal = !*missing;
    for (u32 i = 0; i < n; i++) {
        offs[i] = *missing ? 0 : ix->h_off[term_ids[i]];
        lens[i] = *missing ? 0 : ix->h_len[term_ids[i]];
        dirs[i] = *missing ? SA_NO_DIR : ix->h_dir_off[term_ids[i]];
        *literal = *literal && ix->h_first0[term_ids[i]];
    }
    return SA_OK;
}

// The dense rows of a batch of queries.  The queries are cut, in order, into chunks of `chunk` queries: one chunk's
// doc-space rows stay within about 4 GB of HBM (compressible term rows may add up to 1/8 of padding,
// sa_batch_upload_locked), and its queries fit the span kernels' second grid dimension (65,535).  Inside a chunk the
// term queries take the first rows, then the multi-term queries, each group in query order.
struct RowChunk { u32 row0, n_term, n_phrase; };
struct RowPlan {
    u32 chunk;
    std::vector<RowChunk> chunks;
    std::vector<u32> row_query;      // row -> query
};

inline RowPlan sa_plan_rows(u64 n_docs, const u32 *term_starts, u32 n_queries) {
    RowPlan P;
    const u64 row_bytes = sa_padded_docs(std::max<u64>(n_docs, 1)) * sizeof(float);
    P.chunk = (u32)std::min<u64>(65535, std::max<u64>(1, std::min<u64>(n_queries, (4ull << 30) / row_bytes)));
    P.row_query.reserve(n_queries);
    for (u32 q0 = 0; q0 < n_queries; q0 += P.chunk) {
        const u32 q1 = std::min(n_queries, q0 + P.chunk);
        RowChunk C{(u32)P.row_query.size(), 0, 0};
        for (int pass = 0; pass < 2; pass++)
            for (u32 q = q0; q < q1; q++) {
                const bool term = term_starts[q + 1] - term_starts[q] == 1;
                if (term != (pass == 0)) continue;
                P.row_query.push_back(q);
                (term ? C.n_term : C.n_phrase)++;
            }
        P.chunks.push_back(C);
    }
    return P;
}

inline TermQuery make_term_query(const sa_index *ix, u32 t, float idf) {
    TermQuery tq;
    memset(&tq, 0, sizeof(tq));
    tq.word_off = t == SA_NO_TERM ? 0 : ix->h_off[t];
    tq.n_words = t == SA_NO_TERM ? 0 : ix->h_len[t];
    tq.dir_off = t == SA_NO_TERM ? SA_NO_DIR : ix->h_dir_off[t];
    tq.rec_off = (t == SA_NO_TERM || ix->h_rec_off.empty()) ? SA_NO_DIR : ix->h_rec_off[t];
    tq.idf = idf;
    return tq;
}

// Top-k candidate buffer of Q queries: keys [Q][n_tiles][slots], then counts and maxima [Q][n_tiles] each.
inline size_t cand_bytes(u32 n_tiles, u32 Q, u32 slots) {
    return (size_t)Q * n_tiles * ((size_t)slots * sizeof(u64) + 2 * sizeof(u32)) + 64;
}

inline TopkCtx make_topk_ctx(void *cand, u32 n_tiles, u32 Q, u32 slots, u32 k, u32 *d_overflow) {
    TopkCtx t;
    t.tile_cand = (u64 *)cand;
    t.tile_cnt = (u32 *)(t.tile_cand + (u64)Q * n_tiles * slots);
    t.tile_max = t.tile_cnt + (u64)Q * n_tiles;
    t.overflow = d_overflow;
    t.n_tiles = n_tiles;
    t.slots = slots;
    t.k = k;
    return t;
}

// BM25 scores of the index's own lists into ix->dense, one row per query
inline TermBatchArgs make_term_args(sa_index *ix, const TermQuery *d_queries, const Bm25Params &p, const TopkCtx &t) {
    TermBatchArgs a;
    memset(&a, 0, sizeof(a));
    a.words = ix->d_words.as<u64>();
    a.doc_lens = ix->d_doc_lens.as<float>();
    a.n_docs = ix->n_docs;
    a.doc_base = ix->doc_base;
    a.queries = d_queries;
    a.out = ix->dense.as<float>();
    a.out_stride = sa_padded_docs(ix->n_docs);
    a.bm25 = p;
    a.min_payload = 0;
    a.max_payload = SA_ALL_BITS;
    a.filter = 0;
    a.mode = TERM_MODE_SCORE;
    a.topk = t;
    return a;
}

#ifdef __CUDACC__
// n_pow2 keys in shared memory sorted descending; all threads call
__device__ inline void bitonic_sort_desc_smem(u64 *s, u32 n_pow2) {
    for (u32 k = 2; k <= n_pow2; k <<= 1) {
        for (u32 j = k >> 1; j > 0; j >>= 1) {
            for (u32 i = threadIdx.x; i < n_pow2; i += blockDim.x) {
                u32 ixj = i ^ j;
                if (ixj > i) {
                    u64 a = s[i], b = s[ixj];
                    bool desc = ((i & k) == 0);
                    if ((a < b) == desc) { s[i] = b; s[ixj] = a; }
                }
            }
            __syncthreads();
        }
    }
}

// thread 0: walk the 256-bin histogram from the top until `rem` keys are covered
__device__ __forceinline__ void radix_pick(const u32 *hist, u32 &rem, int &bin) {
    u32 acc = 0;
    int b = 255;
    for (; b > 0; b--) {
        if (acc + hist[b] >= rem) break;
        acc += hist[b];
    }
    rem -= acc;
    bin = b;
}

// k-th largest, with multiplicity, of the BITS-bit keys `visit` yields (0 when it yields fewer than k): an 8-bit
// radix select from the most significant digit, as in topk_select_kernel.  All threads call; all get the result.
template <typename K, int BITS, typename V>
__device__ K radix_kth_largest(u32 k, u32 *s_hist, K *s_prefix, u32 *s_krem, V visit) {
    if (threadIdx.x == 0) { *s_prefix = 0; *s_krem = k; }
    __syncthreads();
    for (int shift = BITS - 8; shift >= 0; shift -= 8) {
        for (u32 i = threadIdx.x; i < 256; i += blockDim.x) s_hist[i] = 0;
        __syncthreads();
        const K prefix = *s_prefix;
        visit([&](K key) {
            if (shift == BITS - 8 || (key >> (shift + 8)) == (prefix >> (shift + 8)))
                atomicAdd(&s_hist[(u32)(key >> shift) & 255u], 1u);
        });
        __syncthreads();
        if (threadIdx.x == 0) {
            u32 rem = *s_krem;
            int b;
            radix_pick(s_hist, rem, b);
            *s_krem = rem;
            *s_prefix = prefix | ((K)(u32)b << shift);
        }
        __syncthreads();
    }
    return *s_prefix;
}

// Thread 0's publication of one (row, tile) for topk_select_kernel: cnt candidates in the tile's slots, max_bits the
// best one's score bits (0: none).  overflow: the tile had more candidates than slots, so its row takes the exact
// host-side re-run.
__device__ __forceinline__ void publish_tile(const TopkCtx &t, u32 row, u32 tile, u32 cnt, u32 max_bits,
                                             bool overflow = false) {
    const u64 t_idx = (u64)row * t.n_tiles + tile;
    t.tile_cnt[t_idx] = cnt;
    t.tile_max[t_idx] = max_bits;
    if (overflow) t.overflow[row] = 1u;
}

// A (row, tile) where nothing ranks: no candidates, bound 0.  tid: the calling thread's index (the boolean kernels
// read it afresh, bool_fresh_tid, so that the test holds no register live through their fold).
__device__ __forceinline__ void publish_empty_tile(const TopkCtx &t, u32 row, u32 tile, unsigned tid) {
    if (tid == 0) publish_tile(t, row, tile, 0, 0);
}

// A (row, tile) without a match: the caller's THREADS threads store its dense tile as zeros straight from registers
// (no shared tile, no barrier), and it is published empty when the launch collects a top k.
template <u32 THREADS>
__device__ __forceinline__ void store_empty_tile(float *__restrict__ out_tile, const TopkCtx &t, u32 row, u32 tile) {
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < SA_TILE_DOCS / THREADS / 4; i++)
        __stcs(reinterpret_cast<float4 *>(out_tile) + threadIdx.x + i * THREADS, z);
    if (t.k) publish_empty_tile(t, row, tile, threadIdx.x);
}

// The deep tile collector (k > SA_TOPK_MAX): the tile's EXACT top k by key score_bits << 32 | ~doc, written as one run
// sorted by key, descending, so that topk_select_kernel<true> reads only the prefix of each run above its threshold.
// s_tile holds the tile's final float32 scores (a doc ranks iff its score is > 0; NaN never does).  With n ranked
// docs, n <= k keeps them all; otherwise a radix select over the 48-bit keys score_bits << 16 | (0xFFFF - local) -- the
// same order, ties to the lower doc -- finds the k-th, and exactly k keys reach it (they are distinct).  The run is
// sorted in shared memory (<= 8 KB) and stored; tile_cnt = its length, tile_max = its first score.  Never overflows.
// All SA_TERM_THREADS threads call; returns after a barrier, so the caller may reuse s_tile.
__device__ __forceinline__ void deep_tile_collect(const float *s_tile, const TopkCtx &t, u32 row, u32 tile) {
    __shared__ u64 s_run[SA_TOPK_DEEP_MAX];
    __shared__ u32 s_hist[256];
    __shared__ u64 s_prefix;
    __shared__ u32 s_krem, s_n, s_m;
    const unsigned tid = threadIdx.x;
    const u32 k = t.k;
    auto visit = [&](auto f) {
#pragma unroll
        for (int jj = 0; jj < SA_TILE_DOCS / SA_TERM_THREADS / 4; jj++) {
            const unsigned g = tid + jj * SA_TERM_THREADS;
            const float4 v = reinterpret_cast<const float4 *>(s_tile)[g];
            const float vs[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int e = 0; e < 4; e++)
                if (vs[e] > 0.0f) f(((u64)__float_as_uint(vs[e]) << 16) | (u64)(0xFFFFu - (g * 4 + e)));
        }
    };
    if (tid == 0) { s_n = 0; s_m = 0; }
    __syncthreads();
    u32 mine = 0;
    visit([&](u64) { mine++; });
    mine = __reduce_add_sync(0xffffffffu, mine);
    if ((tid & 31) == 0 && mine) atomicAdd(&s_n, mine);
    __syncthreads();
    const u32 n = s_n;                                               // CTA-uniform
    const u64 kth = n > k ? radix_kth_largest<u64, 48>(k, s_hist, &s_prefix, &s_krem, visit) : 0ull;
    const u32 tile_doc0 = tile * SA_TILE_DOCS;
    visit([&](u64 key) {
        if (key >= kth) {
            const u32 slot = atomicAdd(&s_m, 1u);
            const u32 local = 0xFFFFu - (u32)(key & 0xFFFFu);
            if (slot < k) s_run[slot] = ((key >> 16) << 32) | (u64)(0xFFFFFFFFu - (tile_doc0 + local));
        }
    });
    const u32 m = min(n, k);
    if (m > 1) {                                                     // CTA-uniform
        u32 n2 = 2;
        while (n2 < m) n2 <<= 1;
        __syncthreads();
        for (u32 i = m + tid; i < n2; i += blockDim.x) s_run[i] = 0ull;
        __syncthreads();
        bitonic_sort_desc_smem(s_run, n2);
    } else {
        __syncthreads();
    }
    const u64 t_idx = (u64)row * t.n_tiles + tile;
    u64 *__restrict__ run = t.tile_cand + t_idx * t.slots;
    for (u32 i = tid; i < m; i += blockDim.x) run[i] = s_run[i];
    if (tid == 0) publish_tile(t, row, tile, m, m ? (u32)(s_run[0] >> 32) : 0u);
    __syncthreads();
}

// ---- collapse (sa_score_batch_topk_bool_collapse): one leader per group, taken by a walk over ranked keys in
// descending order, window by window.  The groups taken so far and those of the current window live in a
// shared-memory hash of 2^bits (code, position) pairs: s_hash[0 .. 2^bits) the codes (SA_COLLAPSE_EMPTY: a free
// slot; group codes are below 2^31 - 1) and s_hash[2^bits .. 2^(bits+1)) per code 0 once taken, otherwise 1 + the
// least window position holding it.
#define SA_COLLAPSE_EMPTY 0xFFFFFFFFu
#define SA_COLLAPSE_TILE_HASH_BITS 12      // a tile: <= k taken + SA_TOPK_DEEP_MAX in a window = 2,048 codes
#define SA_COLLAPSE_TILE_SMEM ((2u << SA_COLLAPSE_TILE_HASH_BITS) * sizeof(u32))   // 32 KB of dynamic memory

// Every thread of the CTA calls: every slot free.
__device__ __forceinline__ void collapse_hash_clear(u32 *s_hash, u32 bits) {
    for (u32 i = threadIdx.x; i < (2u << bits); i += blockDim.x) s_hash[i] = SA_COLLAPSE_EMPTY;
}

// The slot of code g (not SA_GROUP_NONE), inserted if absent: open addressing with linear probes.
__device__ __forceinline__ u32 collapse_slot(u32 *s_hash, u32 bits, u32 g) {
    const u32 mask = (1u << bits) - 1;
    u32 h = (g * 0x9E3779B1u) >> (32 - bits);
    for (;;) {
        const u32 prev = atomicCAS(s_hash + h, SA_COLLAPSE_EMPTY, g);
        if (prev == SA_COLLAPSE_EMPTY || prev == g) return h;
        h = (h + 1) & mask;
    }
}

// One window of the walk: s_win[0, m) ranked run keys (score_bits << 32 | ~doc, doc index-local) sorted descending,
// m <= NT * PER, thread t owning positions PER t .. PER t + PER - 1.  A key is a leader iff its doc's code (groups[doc])
// is SA_GROUP_NONE, or is not taken and no earlier position of the window holds it.  The leaders go, in order, to
// ranks taken, taken + 1, ... below k through emit(rank, key); every code of the window is then taken.  Returns the
// new number of leaders (<= k).  Every thread of the NT-thread CTA calls; returns after a barrier.
template <int NT, int PER, typename E>
__device__ __forceinline__ u32 collapse_window(const u64 *s_win, u32 m, const u32 *__restrict__ groups, u32 *s_hash,
                                               u32 bits, u32 taken, u32 k, E emit) {
    __shared__ u32 s_warp[NT / 32];
    u32 *s_pos = s_hash + (1u << bits);
    const u32 p0 = threadIdx.x * PER;
    u32 slot[PER];
#pragma unroll
    for (int j = 0; j < PER; j++) {
        slot[j] = SA_COLLAPSE_EMPTY;
        if (p0 + j >= m) continue;
        const u32 g = __ldg(groups + (0xFFFFFFFFu - (u32)s_win[p0 + j]));
        if (g == SA_GROUP_NONE) continue;
        slot[j] = collapse_slot(s_hash, bits, g);
        atomicMin(s_pos + slot[j], p0 + j + 1);
    }
    __syncthreads();
    u32 keep = 0;
#pragma unroll
    for (int j = 0; j < PER; j++)
        if (p0 + j < m && (slot[j] == SA_COLLAPSE_EMPTY || s_pos[slot[j]] == p0 + j + 1)) keep |= 1u << j;
    u32 total;
    u32 r = taken + block_exclusive_sum<NT>((u32)__popc(keep), s_warp, total);
#pragma unroll
    for (int j = 0; j < PER; j++)
        if ((keep >> j) & 1u) {
            if (r < k) emit(r, s_win[p0 + j]);
            r++;
        }
    __syncthreads();                                                 // every test above read s_pos
#pragma unroll
    for (int j = 0; j < PER; j++)
        if (slot[j] != SA_COLLAPSE_EMPTY) s_pos[slot[j]] = 0;
    __syncthreads();
    return min(taken + total, k);
}

// The collapse tile collector: the tile's EXACT k best leaders (collapse_window) as one run sorted by key, descending,
// with tile_cnt = its length and tile_max = its first score, as deep_tile_collect publishes its run.  A group whose
// global leader d lies in this tile has fewer than k groups above it in the tile (each of them ranks above it
// globally), so it is among the tile's k best leaders: topk_collapse_kernel's select over the runs is exact.  The
// ranked keys are walked in windows of SA_TOPK_DEEP_MAX, each the next keys below the last window's least (a radix
// select over the 48-bit keys of deep_tile_collect, sorted in s_run), until k leaders are taken or the ranked docs
// run out.  groups: the group column (index-local ids); s_hash: SA_COLLAPSE_TILE_SMEM bytes; *windows counts the
// windows past the first.  s_tile holds the tile's final scores, as deep_tile_collect takes them, and is not written.
// All SA_TERM_THREADS threads call; returns after a barrier.
__device__ __forceinline__ void collapse_tile_collect(const float *s_tile, const TopkCtx &t, u32 row, u32 tile,
                                                      const u32 *__restrict__ groups, u32 *s_hash, u32 *windows) {
    __shared__ u64 s_run[SA_TOPK_DEEP_MAX];
    __shared__ u32 s_hist[256];
    __shared__ u64 s_prefix;
    __shared__ u32 s_krem, s_n, s_m, s_max;
    const unsigned tid = threadIdx.x;
    const u32 k = t.k, tile_doc0 = tile * SA_TILE_DOCS;
    u64 hi = ~0ull;                                                  // keys below hi are still to walk
    auto visit = [&](auto f) {
#pragma unroll
        for (int jj = 0; jj < SA_TILE_DOCS / SA_TERM_THREADS / 4; jj++) {
            const unsigned g = tid + jj * SA_TERM_THREADS;
            const float4 v = reinterpret_cast<const float4 *>(s_tile)[g];
            const float vs[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int e = 0; e < 4; e++) {
                const u64 key = ((u64)__float_as_uint(vs[e]) << 16) | (u64)(0xFFFFu - (g * 4 + e));
                if (vs[e] > 0.0f && key < hi) f(key);
            }
        }
    };
    __syncthreads();                           // the tile as every thread stored it; the fold's dynamic memory is free
    collapse_hash_clear(s_hash, SA_COLLAPSE_TILE_HASH_BITS);
    if (tid == 0) { s_n = 0; s_max = 0; }
    __syncthreads();
    u32 mine = 0;
    visit([&](u64) { mine++; });
    mine = __reduce_add_sync(0xffffffffu, mine);
    if ((tid & 31) == 0 && mine) atomicAdd(&s_n, mine);
    __syncthreads();
    // CTA-uniform: s_n is written only before the barrier above.  Each window gathers through its own counter s_m,
    // which thread 0 clears when every thread is past the previous window's gather (the barriers of the sort and of
    // collapse_window lie between), and which nothing reads but the gather's atomics after the barrier that follows
    // the clear; with lo = 0 no radix select runs, so a shared counter would race with this read of s_n
    u32 n = s_n, taken = 0, w = 0;
    u64 *__restrict__ run = t.tile_cand + ((u64)row * t.n_tiles + tile) * t.slots;
    while (taken < k && n > 0) {
        const u32 m = min(n, (u32)SA_TOPK_DEEP_MAX);
        const u64 lo = n > m ? radix_kth_largest<u64, 48>(m, s_hist, &s_prefix, &s_krem, visit) : 0ull;
        if (tid == 0) s_m = 0;
        __syncthreads();
        visit([&](u64 key) {
            if (key >= lo)
                s_run[atomicAdd(&s_m, 1u)] = ((key >> 16) << 32) |
                                             (u64)(0xFFFFFFFFu - (tile_doc0 + 0xFFFFu - (u32)(key & 0xFFFFu)));
        });
        u32 n2 = 1;
        while (n2 < m) n2 <<= 1;
        __syncthreads();
        for (u32 i = m + tid; i < n2; i += blockDim.x) s_run[i] = 0ull;
        __syncthreads();
        bitonic_sort_desc_smem(s_run, n2);
        taken = collapse_window<SA_TERM_THREADS, SA_TOPK_DEEP_MAX / SA_TERM_THREADS>(
            s_run, m, groups, s_hash, SA_COLLAPSE_TILE_HASH_BITS, taken, k, [&](u32 r, u64 key) {
                run[r] = key;
                if (r == 0) s_max = (u32)(key >> 32);
            });
        n -= m;
        hi = lo;
        w++;
    }
    if (tid == 0) {
        publish_tile(t, row, tile, taken, s_max);
        if (w > 1) atomicAdd(windows, w - 1);
    }
    __syncthreads();
}

// BM25 of tf from the doc's cached length norm (sa_ensure_norm): the last two rounded operations of bm25_one
__device__ __forceinline__ float bm25_from_norm(float tf, float norm, float idf) {
    return __fmul_rn(__fdiv_rn(tf, __fadd_rn(tf, norm)), idf);
}

// The j-th round of "take the warp maximum, then clear it" (REDUX.MAX: one instruction per round on sm_80+).
// Exactly ONE lane gives up its value per round, so equal values are counted with their multiplicity: BM25
// scores are a function of (tf, doc length) only and repeat a lot -- collapsing duplicates used to leave fewer
// than k published values on tiles whose top scores tie, which degenerates the bound to "keep everything".
__device__ __forceinline__ u32 warp_pop_max(u32 &v) {
    const u32 m = __reduce_max_sync(0xffffffffu, v);
    const unsigned holders = __ballot_sync(0xffffffffu, v == m);
    if ((threadIdx.x & 31) == (unsigned)(__ffs(holders) - 1)) v = 0;
    return m;
}

// k-th largest (k <= 32), with multiplicity, of the CTA's thread maxima, from the per-warp top-M lists in shared
// memory (M = 4 or 8, tile_bound_width; exact unless one warp holds more than M of the CTA's top k, in which case
// the result is smaller -- still a valid lower bound of the tile's k-th best score, because thread maxima belong to
// distinct docs).  Every warp computes it redundantly, no extra barrier.
__device__ __forceinline__ u32 cta_kth_bound(const u32 *s_top /*[8][8]*/, u32 k, bool wide = false) {
    const unsigned lane = threadIdx.x & 31;
    u32 v0, v1 = 0;
    if (k <= 10 && !wide) {
        v0 = s_top[(lane >> 2) * 8 + (lane & 3)];
    } else {
        v0 = s_top[lane];
        v1 = s_top[32 + lane];
    }
    u32 kth = 0;
    for (u32 r = 0; r < k; r++) {
        const u32 m0 = __reduce_max_sync(0xffffffffu, max(v0, v1));
        kth = m0;
        if (m0 == 0) break;
        const unsigned holders = __ballot_sync(0xffffffffu, v0 == m0 || v1 == m0);
        if (lane == (unsigned)(__ffs(holders) - 1)) {        // one holder gives up ONE copy
            if (v0 == m0) v0 = 0; else v1 = 0;
        }
    }
    return kth;
}

// The tile bound: every warp publishes the M largest of its threads' values v into s_top (M = 4 or 8,
// tile_bound_width), then, after a barrier, every warp derives the k-th largest of them (cta_kth_bound), at least 1.
// need = false (CTA-uniform): no bound, 1.  With k > 0 thread 0 also clears the tile's candidate count and maximum
// before the barrier.  The barrier is taken either way, so what the CTA stored to shared memory before the call is
// visible after it.  All SA_TERM_THREADS threads call.
__device__ __forceinline__ u32 tile_bound(u32 v, bool need, u32 M, u32 k, u32 *s_top, u32 *s_ncand, u32 *s_tile_max) {
    const unsigned warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (need) {
        for (u32 r = 0; r < M; r++) {
            const u32 m = warp_pop_max(v);
            if (lane == r) s_top[warp * 8 + r] = m;
        }
    }
    if (k && threadIdx.x == 0) { *s_ncand = 0; *s_tile_max = 0; }
    __syncthreads();
    return need ? max(cta_kth_bound(s_top, k, M == 8u), 1u) : 1u;
}

// Candidate-slot overflow caused by TIES at the tile bound (BM25 scores are a function of (tf, doc_len) only, so
// exact ties among thousands of docs are normal): the tile is still in shared memory, so the CTA collects
// again, now breaking ties the way the final ranking does -- lower doc id first.  Scores above the bound are
// all kept; of the docs AT the bound only those with a local index <= the k-th smallest such index (a bound
// derived from the threads' smallest tied docs, which are distinct docs) are kept: a superset of what the
// top-k can take from this tile.  finish: flush_tile_collect's, applied to the tile again.  All SA_TERM_THREADS
// threads call; returns with the slots, *s_ncand and *s_tile_max rewritten (the caller publishes them).  Still
// more than `slots` -> the caller flags the query for the exact host-side re-run, as before.
template <typename F>
__device__ __forceinline__ void tile_collect_ties_retry(const float *s_out, F finish, u32 thr_bits, const TopkCtx &t,
                                                        u64 *__restrict__ my_cand, u32 tile_doc0, u32 *s_top,
                                                        u32 *s_ncand, u32 *s_tile_max) {
    const unsigned tid = threadIdx.x;
    const float thr_f = __uint_as_float(thr_bits);
    u32 best = 0;                                   // 0xFFFFFFFF - smallest tied local doc of this thread (0 = none)
#pragma unroll
    for (int jj = 0; jj < SA_TILE_DOCS / SA_TERM_THREADS / 4; jj++) {
        const unsigned g = tid + jj * SA_TERM_THREADS;
        float4 v = reinterpret_cast<const float4 *>(s_out)[g];
        finish(g, v);
        const float vs[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int e = 0; e < 4; e++)
            if (vs[e] == thr_f) best = max(best, 0xFFFFFFFFu - (g * 4 + e));
    }
    __syncthreads();                                // every thread has read the caller's *s_ncand
    // fewer than k threads hold a tie: the bound is 1, above every local doc -> keep every tie
    const u32 doc_bound = 0xFFFFFFFFu - tile_bound(best, true, 8u, t.k, s_top, s_ncand, s_tile_max);
    u32 cand_max = 0;
#pragma unroll
    for (int jj = 0; jj < SA_TILE_DOCS / SA_TERM_THREADS / 4; jj++) {
        const unsigned g = tid + jj * SA_TERM_THREADS;
        float4 fv = reinterpret_cast<const float4 *>(s_out)[g];
        finish(g, fv);
        const float vs[4] = {fv.x, fv.y, fv.z, fv.w};
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const float v = vs[e];
            if (v > thr_f || (v == thr_f && g * 4 + e <= doc_bound)) {
                u32 slot = atomicAdd(s_ncand, 1u);
                if (slot < t.slots)
                    my_cand[slot] = ((u64)__float_as_uint(v) << 32) | (u64)(0xFFFFFFFFu - (tile_doc0 + g * 4 + e));
                cand_max = max(cand_max, __float_as_uint(v));
            }
        }
    }
    if (cand_max) atomicMax(s_tile_max, cand_max);
    __syncthreads();
}

// How many of its largest thread maxima every warp publishes for the tile bound.  4 per warp are enough for k <= 10
// when all eight warps hold scores; a tile whose scores sit in two or three warps (a few dozen docs) must publish 8 per
// warp, or fewer than k values exist, the bound degenerates to "keep everything" and 65+ docs overflow the 64 slots.
// `n_holders`: how many threads can hold a score (not how many scores there are).
__device__ __forceinline__ u32 tile_bound_width(u32 k, u32 n_holders) { return (k <= 10 && n_holders >= SA_TERM_THREADS) ? 4u : 8u; }

// The finish step of flush_tile_collect that leaves the tile as it is.
struct TileIdentity {
    __device__ __forceinline__ void operator()(unsigned, float4 &) const {}
};

// Flush one shared-memory score tile to its dense row with 16-byte streaming stores and, on the way, collect the
// tile's top-k candidates (private slots, count, maximum): the step every float32 tile kernel ends with.
// finish(g, v) turns float4 g of the tile (docs 4 g .. 4 g + 3) into the final scores that are stored and collected
// (the term kernel's: staged-norm tiles hold negated scores, ALL_DOCS tiles term frequencies); the default,
// TileIdentity, takes the tile as it is.  `my_max` = largest final score bits this thread put into the tile,
// `n_items` = number of scores in the tile, `n_holders` = how many threads can hold one of them.  All SA_TERM_THREADS
// threads must call.
// STORE = false: collect only (out_tile unused); the tile stays in shared memory for the tie retry either way.
// DEEP: k > SA_TOPK_MAX, the tile's candidates from deep_tile_collect (my_max, n_items and n_holders unused); a
// finish other than TileIdentity writes the final scores back to the tile for it.
// ties_retry = false: a tile whose ties at the bound overflow the slots flags its row for the exact re-run at once,
// without the tie retry (which applies finish to the whole tile again).
template <bool STORE = true, bool DEEP = false, typename F = TileIdentity>
__device__ __forceinline__ void flush_tile_collect(float *s_out, float *__restrict__ out_tile, const TopkCtx &t,
                                                   u32 row, u32 tile, u32 my_max, u32 n_items, u32 n_holders, u32 *s_top,
                                                   u32 *s_ncand, u32 *s_tile_max, F finish = F(),
                                                   bool ties_retry = true) {
    constexpr bool FINISH = !std::is_same<F, TileIdentity>::value;
    const unsigned tid = threadIdx.x;
    float4 *s_out4 = reinterpret_cast<float4 *>(s_out);
    if constexpr (DEEP) {
        __syncthreads();                                             // the tile as every thread stored it
#pragma unroll
        for (int jj = 0; jj < SA_TILE_DOCS / SA_TERM_THREADS / 4; jj++) {
            const unsigned g = tid + jj * SA_TERM_THREADS;
            float4 v = s_out4[g];
            finish(g, v);
            if constexpr (STORE) __stcs(reinterpret_cast<float4 *>(out_tile) + tid + jj * SA_TERM_THREADS, v);
            if constexpr (FINISH) s_out4[g] = v;
        }
        if constexpr (FINISH) __syncthreads();                       // the final scores, as every thread wrote them
        deep_tile_collect(s_out, t, row, tile);
        return;
    }
    const u32 k = t.k;
    const u32 tile_doc0 = tile * SA_TILE_DOCS;
    // the barrier inside also orders the tile's stores before the reads below
    const float thr_f = __uint_as_float(tile_bound(my_max, k && n_items > k, tile_bound_width(k, n_holders), k, s_top, s_ncand, s_tile_max));
    u64 *__restrict__ my_cand = k ? t.tile_cand + ((u64)row * t.n_tiles + tile) * t.slots : nullptr;
    float4 *__restrict__ out4 = reinterpret_cast<float4 *>(out_tile);
    u32 cand_max = 0;
#pragma unroll
    for (int jj = 0; jj < SA_TILE_DOCS / SA_TERM_THREADS / 4; jj++) {
        const unsigned g = tid + jj * SA_TERM_THREADS;
        float4 v = s_out4[g];
        finish(g, v);
        if constexpr (STORE) __stcs(out4 + g, v);
        // NaN compares false; scores <= 0 are below thr_f > 0
        if (k && ((v.x >= thr_f) | (v.y >= thr_f) | (v.z >= thr_f) | (v.w >= thr_f))) {
            const float vs[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int e = 0; e < 4; e++) {
                if (vs[e] >= thr_f) {
                    u32 slot = atomicAdd(s_ncand, 1u);
                    if (slot < t.slots)
                        my_cand[slot] = ((u64)__float_as_uint(vs[e]) << 32) | (u64)(0xFFFFFFFFu - (tile_doc0 + g * 4 + e));
                    cand_max = max(cand_max, __float_as_uint(vs[e]));
                }
            }
        }
    }
    if (k) {
        if (cand_max) atomicMax(s_tile_max, cand_max);
        __syncthreads();
        if (ties_retry && *s_ncand > t.slots)                        // CTA-uniform: ties at the bound (see above)
            tile_collect_ties_retry(s_out, finish, __float_as_uint(thr_f), t, my_cand, tile_doc0, s_top, s_ncand,
                                    s_tile_max);
        if (tid == 0) {
            const u32 n = *s_ncand;
            publish_tile(t, row, tile, min(n, t.slots), *s_tile_max, n > t.slots);
        }
    }
    __syncthreads();
}

// The float32 key a float64 score s ranks by when no float32 value is exact: s rounded toward zero, at least the
// smallest subnormal for s > 0 (0 = never ranks: s <= 0 or NaN).  Monotone in s, but distinct scores can share it.
__device__ __forceinline__ u32 f64_proxy_key(double s) {
    return s > 0.0 ? max(1u, __float_as_uint(__double2float_rz(s))) : 0u;
}

// flush_tile_collect for float64 scores ranked by f64_proxy_key (classic similarity, edismax): the tile bound from 8
// maxima per warp, then EVERY position whose key is at or above it -- no tie cut, which would drop positions tied in
// the key by index although their float64 scores can be larger -- with the float64 score bits beside each candidate
// in tile_d (slot for slot), for topk_select_f64_kernel.  key[]: the thread's keys in flush_tile_collect's layout
// (position 4g + e of the tile, g = tid + j * SA_TERM_THREADS), my_max their maximum, n_items the positions of the
// tile; score(local) returns the float64 score of tile position `local` and runs for the stored candidates only.
// More candidates than slots flags the query's overflow: the caller re-runs it with SA_TILE_DOCS slots, which cannot
// overflow.  All SA_TERM_THREADS threads must call.  DEEP (k > SA_TOPK_MAX): the bound is the EXACT k-th largest key
// of the tile (a radix select over the keys in registers; 1 when fewer than k positions rank), and the caller gives
// the tile max(k, 256) slots.
template <bool DEEP = false, typename F>
__device__ __forceinline__ void collect_tile_f64(const u32 (&key)[SA_TILE_DOCS / SA_TERM_THREADS], u32 my_max,
                                                 u32 n_items, const TopkCtx &t, u64 *__restrict__ tile_d, u32 row,
                                                 u32 tile, u32 *s_top, u32 *s_ncand, u32 *s_tile_max, F score) {
    const unsigned tid = threadIdx.x;
    u32 thr;
    if constexpr (DEEP) {
        __shared__ u32 s_hist[256], s_kth, s_krem;
        const u32 kth = radix_kth_largest<u32, 32>(t.k, s_hist, &s_kth, &s_krem, [&](auto f) {
#pragma unroll
            for (int i = 0; i < SA_TILE_DOCS / SA_TERM_THREADS; i++)
                if (key[i]) f(key[i]);
        });
        if (tid == 0) { *s_ncand = 0; *s_tile_max = 0; }
        __syncthreads();
        thr = max(kth, 1u);
    } else {
        thr = tile_bound(my_max, n_items > t.k, 8u, t.k, s_top, s_ncand, s_tile_max);
    }
    const u64 slot0 = ((u64)row * t.n_tiles + tile) * t.slots;
    u32 cand_max = 0;
#pragma unroll
    for (int j = 0; j < SA_TILE_DOCS / SA_TERM_THREADS / 4; j++) {
#pragma unroll
        for (int e = 0; e < 4; e++) {
            if (key[j * 4 + e] >= thr) {
                const u32 local = (tid + j * SA_TERM_THREADS) * 4 + e;
                const u32 slot = atomicAdd(s_ncand, 1u);
                if (slot < t.slots) {
                    t.tile_cand[slot0 + slot] = ((u64)key[j * 4 + e] << 32) | (u64)(0xFFFFFFFFu - (tile * SA_TILE_DOCS + local));
                    tile_d[slot0 + slot] = (u64)__double_as_longlong(score(local));
                }
                cand_max = max(cand_max, key[j * 4 + e]);
            }
        }
    }
    if (cand_max) atomicMax(s_tile_max, cand_max);
    __syncthreads();
    if (tid == 0) publish_tile(t, row, tile, min(*s_ncand, t.slots), *s_tile_max, *s_ncand > t.slots);
}
#endif
