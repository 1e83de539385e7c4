// sa_term.cu -- the term-at-a-time BM25 scan (the headline kernel).
//
// Replaces, fused into one launch per query batch:
//   popcount64_reduce   searcharray/roaringish/popcount.pyx:212-237  (tf by doc)
//   as_dense/scatter    searcharray/roaringish/roaringish_ops.pyx:84-98, scatter_assign.h:8-29
//   bm25_score          searcharray/bm25/bm25.pyx:11-41
//
// Design.  The dense float32[N] score vector is cut into tiles of SA_TILE_DOCS docs; one
// CTA owns one (query, tile) and builds the tile in 32 KB of shared memory:
//   1. the slice [lo,hi) of the term's posting words whose docs fall in the tile comes from the
//      term's tile directory (two loads; built at upload for long lists) or, for short lists,
//      from a warp-cooperative 32-ary search;
//   2. the slice is streamed with coalesced 8-byte loads (4 windows in flight per thread).  Words
//      are sorted by doc, so the words of one doc are adjacent: the thread holding the FIRST word
//      of a doc ("head") adds the popcounts of the doc's run (neighbours via warp shuffle over
//      overlapping 32-lane windows), takes the doc's precomputed BM25 length norm (a gather per
//      pass, issued back to back; dense tiles stage the tile's norms with cp.async instead),
//      evaluates tf/(tf+norm)*idf with individually rounded operations (bit-identical to the
//      reference's x86-64 build) and stores the score into the shared tile.  No atomics, no work
//      for docs that do not contain the term;
//   3. the tile is flushed once with 16-byte streaming stores; while it passes through registers
//      every score >= a running, provably valid lower bound of the k-th best score is appended to
//      the query's top-k candidate list (sa_topk.cu), so the dense vector is never re-read.  This is
//      flush_tile_collect (sa_term.cuh), shared with the other tile kernels; the kernel's finish step
//      forms the final scores on the way.
// The grid is one-dimensional, Q * n_tiles CTAs walked in groups of G consecutive queries: inside a group the query
// runs fastest, then the tile, then the group.  The CTAs in flight (about 6 per SM) then cover about 6 * SMs / G
// neighbouring tiles of G rows: dense terms (issue-bound CTAs) and sparse terms (store-bound CTAs) overlap, and a
// staged tile's norms are read from DRAM about once per group and shared in L2 by its queries.  G = Q (every query of
// the launch, the default) shares them the most; rows in compressible memory want a small G, whose CTAs write few
// rows in long runs of neighbouring tiles (DESIGN §3.1).
// HBM traffic: 8*W (words) + the 32 B sectors holding the 4*df norms + 4*N (scores), less whatever
// the queries of one launch share in L2.  Evaluating BM25 for all 16 docs of every thread under
// divergence with shared-memory atomics was instruction-bound; variants that staged the postings with TMA bulk copies (cp.async.bulk +
// mbarrier), wrote zeros straight to HBM for sparse tiles, or pinned the norm table in L2 measured
// slower and were dropped.
#include <algorithm>
#include <type_traits>

#include "sa_term.cuh"

__device__ __forceinline__ bool payload_keep(u64 w, u64 lo, u64 hi) {
    // reference roaringish_ops.pyx:55: compares the UNSHIFTED masked word
    u64 v = w & SA_MSB_MASK;
    return v >= lo && v <= hi;
}

// DEEP: k > SA_TOPK_MAX, the tile's candidates from deep_tile_collect (through flush_tile_collect).
template <int MODE, bool ALL_DOCS, bool FILTER, bool DEEP>
__global__ void __launch_bounds__(SA_TERM_THREADS, DEEP ? SA_TERM_DEEP_CTAS_PER_SM : SA_TERM_CTAS_PER_SM)
term_tile_kernel(const TermBatchArgs a) {
    __shared__ __align__(16) float s_out[SA_TILE_DOCS];
    __shared__ u32 s_range[2];
    __shared__ u32 s_top[(SA_TERM_THREADS / 32) * 8];
    __shared__ u32 s_ncand, s_tile_max;

    // 1-D grid in groups of G queries: CTA b is in group g = b / (G T); inside it, consecutive CTAs work on the SAME
    // tile of the group's Gg (<= G: the last group may be partial) queries, then on the next tile
    const u32 grp = blockIdx.x / a.group_ctas;
    const u32 rem = blockIdx.x - grp * a.group_ctas;
    const u32 q0 = grp * a.group;
    const u32 gg = min(a.group, a.n_queries - q0);
    const u32 tile = rem / gg;
    const u32 q = q0 + (rem - tile * gg);
    const TermQuery tq = a.queries[q];
    const unsigned tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const u64 *__restrict__ words = a.words + tq.word_off;
    const u32 n_words = (u32)tq.n_words;
    const u32 tile_doc0 = tile * SA_TILE_DOCS;                       // local doc index
    const u32 tile_doc0_abs = (u32)a.doc_base + tile_doc0;           // as stored in the words

    // 1. zero the tile; posting slice [lo, hi) of this tile
#pragma unroll
    for (int i = 0; i < SA_TILE_DOCS / SA_TERM_THREADS / 4; i++)
        reinterpret_cast<float4 *>(s_out)[tid + i * SA_TERM_THREADS] = make_float4(0.f, 0.f, 0.f, 0.f);
    u32 lo, hi;
    bool quads = false;
    // tf-table path (CTA-uniform): the term has (doc, tf) records and nothing has to look inside the words
    const bool use_recs = !FILTER && !ALL_DOCS && a.recs != nullptr && tq.rec_off != SA_NO_DIR && tq.dir_off != SA_NO_DIR;
    if (use_recs) {
        const u32 *dir = a.rec_dir + tq.dir_off + tile;
        lo = __ldg(dir);
        hi = __ldg(dir + 1);
        // L2 prefetch of the records a LATER tile of this query will read: tile + d is dispatched Gg * d CTAs after this
        // one, and launch_term_batch picks d so that this is about one generation of resident CTAs; its record loads --
        // the second of two dependent DRAM round trips (directory, then records) on a memory system saturated with the
        // dense rows' stores -- then hit L2.  One 128-byte line per thread covers any tile (<= 32 KB).
        const u32 pf_tile = tile + a.prefetch_tiles;
        if (a.prefetch_tiles && (u64)pf_tile * SA_TILE_DOCS < a.n_docs) {
            const u32 plo = __ldg(dir + a.prefetch_tiles), phi = __ldg(dir + a.prefetch_tiles + 1);
            const u32 pi = (plo & ~31u) + tid * 32u;
            if (pi < phi) asm volatile("prefetch.global.L2 [%0];" ::"l"(a.recs + tq.rec_off + pi));
        }
        __syncthreads();
        // Four records per thread only when that still leaves >= k threads, in whole warps, holding a score: the
        // tile bound is the k-th largest of (at most 8 per warp) thread maxima, and with fewer than k of them it
        // degenerates to "keep everything" -- 129 records in 32 threads of ONE warp overflowed the 128 slots (the short
        // last tile of a 2.5M-doc shard).  16 * k records = 4 * k quads = k / 8 full warps of 8 published maxima.
        // (the deep collector takes no bound from thread maxima)
        quads = hi - lo >= (DEEP ? a.quad_min_recs : max(a.quad_min_recs, 16u * a.topk.k));
    } else if (tq.dir_off != SA_NO_DIR) {                             // CTA-uniform
        const u32 *dir = a.tile_dir + tq.dir_off + tile;
        lo = __ldg(dir);
        hi = __ldg(dir + 1);
        __syncthreads();
    } else {
        if (warp < 2) {
            u64 key = (u64)tile_doc0_abs + (warp ? SA_TILE_DOCS : 0);
            u64 r = warp_lower_bound_shifted(words, 0, n_words, key, SA_KEY_SHIFT);
            if (lane == 0) s_range[warp] = (u32)r;
        }
        __syncthreads();
        lo = s_range[0];
        hi = s_range[1];
    }

    // Dense tiles (SCORE mode): instead of one dependent norm gather per matching doc, the tile's
    // norms are staged in the score tile itself with asynchronous 16-byte copies (cp.async) issued
    // together with the first posting loads -- one coalesced 32 KB read in place of a second DRAM
    // round trip per pass.  A doc's head reads its norm from the tile and stores the score NEGATED:
    // norms are > 0 here and scores >= +0, so the sign bit tells a score (set) from a leftover norm
    // (clear), which the flush turns into 0.
    const bool staged_norm = MODE == TERM_MODE_SCORE && !ALL_DOCS &&
                             (hi - lo) >= (use_recs ? a.staged_norm_min_recs : a.staged_norm_min_words);
    bool norm_ready = !staged_norm;
    if (staged_norm) {
        const float4 *__restrict__ n4 = reinterpret_cast<const float4 *>(a.norm + tile_doc0);
#pragma unroll
        for (int i = 0; i < SA_TILE_DOCS / SA_TERM_THREADS / 4; i++) {
            const unsigned dst = (unsigned)__cvta_generic_to_shared(reinterpret_cast<float4 *>(s_out) + tid + i * SA_TERM_THREADS);
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(n4 + tid + i * SA_TERM_THREADS) : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    }

    // 2. stream the slice.  Each warp takes windows of 30 owned words and loads 32 (two look-ahead
    //    lanes), so "is the previous / next word the same doc?" is a register shuffle with no
    //    warp-edge special case.  Words are sorted by doc: the thread holding the FIRST word of a
    //    doc ("head") sums the doc's run (<= 3 words via shuffles, longer runs by look-ahead
    //    loads).  SA_TERM_UNROLL windows are loaded before any is processed, and the heads' norm
    //    gathers are issued back to back before any score is computed (memory-level parallelism).
    u32 my_max = 0;
    const float *__restrict__ norm = a.norm + tile_doc0;
    constexpr u32 OWN = 30;
    constexpr u32 WIN = (SA_TERM_THREADS / 32) * OWN;                  // words per CTA pass (240)
    auto windows = [&](auto unroll_tag, const u32 base) {
        constexpr int UN = decltype(unroll_tag)::value;
        u64 w[UN];
#pragma unroll
        for (int u = 0; u < UN; u++) {
            const u32 i = base + (u * (SA_TERM_THREADS / 32) + warp) * OWN + lane;
            // look-ahead lanes may read into the next tile (another doc) but never past the list
            w[u] = (i < n_words && i < hi + 2) ? __ldg(words + i) : ~0ull;
        }
        // rel << 19 | tf, the tf records' layout: tf <= 2^18 (positions < 2^18) needs 19 bits, and rel < 2^13 keeps
        // every packed value below ~0 = not a head
        u32 pk[UN];
        float nr[UN];
#pragma unroll
        for (int u = 0; u < UN; u++) {
            const u32 s = base + (u * (SA_TERM_THREADS / 32) + warp) * OWN;   // window start (warp-uniform)
            const u32 i = s + lane;
            const u32 rel = (u32)(w[u] >> SA_KEY_SHIFT) - tile_doc0_abs;  // >= 2^27 for the ~0 filler
            u32 pc = (u32)__popcll(w[u] & SA_LSB_MASK);
            if (FILTER && !payload_keep(w[u], a.min_payload, a.max_payload)) pc = 0;
            const u32 packed = (rel << 5) | pc;                        // pc <= 18
            u32 prev = __shfl_up_sync(0xffffffffu, packed, 1);
            const u32 next = __shfl_down_sync(0xffffffffu, packed, 1);
            const u32 next2 = __shfl_down_sync(0xffffffffu, packed, 2);
            if (lane == 0) {
                prev = ~0u;                                           // s == lo: previous word is another tile's
                if (s > lo && s < hi) prev = ((u32)(__ldg(words + s - 1) >> SA_KEY_SHIFT) - tile_doc0_abs) << 5;
            }
            pk[u] = ~0u;
            nr[u] = 0.0f;
            const bool owned = lane < OWN && i < hi;
            if (owned && (prev >> 5) != rel && rel < SA_TILE_DOCS) {
                u32 tf = pc;
                if ((next >> 5) == rel) {
                    tf += next & 31u;
                    if ((next2 >> 5) == rel) {
                        tf += next2 & 31u;
                        for (u32 j = i + 3; j < n_words; j++) {        // runs of >= 4 words (rare)
                            const u64 w2 = __ldg(words + j);
                            if ((u32)(w2 >> SA_KEY_SHIFT) - tile_doc0_abs != rel) break;
                            if (!(FILTER && !payload_keep(w2, a.min_payload, a.max_payload))) tf += (u32)__popcll(w2 & SA_LSB_MASK);
                        }
                    }
                }
                pk[u] = (rel << SA_REC_TF_BITS) | tf;
                if (MODE == TERM_MODE_SCORE && !ALL_DOCS && tf && !staged_norm) nr[u] = __ldg(norm + rel);
            }
        }
        if (!norm_ready) {                                 // CTA-uniform: first pass of a staged tile
            asm volatile("cp.async.wait_all;" ::: "memory");
            __syncthreads();
            norm_ready = true;
        }
#pragma unroll
        for (int u = 0; u < UN; u++) {
            if (pk[u] != ~0u) {
                const u32 rel = pk[u] >> SA_REC_TF_BITS, tf = pk[u] & SA_REC_TF_MASK;
                float v;
                if (MODE == TERM_MODE_TF || ALL_DOCS) {
                    v = (float)tf;
                } else {
                    v = 0.0f;
                    if (tf) {
                        const float nrm = staged_norm ? s_out[rel] : nr[u];
                        v = bm25_from_norm((float)tf, nrm, tq.idf);
                        my_max = max(my_max, __float_as_uint(v));
                    }
                }
                s_out[rel] = staged_norm ? -v : v;
            }
        }
    };
    if (use_recs) {
        // 2'. tf-table path: one u32 record per matching doc, (doc - tile_doc0) << 19 | tf, in doc order.  Every
        //     lane takes FOUR records with one 16-byte load (record runs start 16-byte aligned; the slice is
        //     widened to whole quads and the strangers masked); no run detection, no shuffles, no popcount.
        const u32 *__restrict__ recs = a.recs + tq.rec_off;
        if (quads) {                       // with a tile bound over thread maxima at most 4 * k docs reach it
            // quads => staged norms (quad_min_recs >= staged_norm_min_recs, launch_term_batch): no norm gathers here.
            // Two quads are loaded before either is processed (two 16-byte loads in flight per thread).
            constexpr int QU = 2;
            for (u32 base = lo & ~3u; base < hi; base += SA_TERM_THREADS * 4 * QU) {  // CTA-uniform trip count
                uint4 r4[QU];
    #pragma unroll
                for (int u = 0; u < QU; u++) {
                    const u32 i = base + (u * SA_TERM_THREADS + tid) * 4;
                    r4[u] = make_uint4(0u, 0u, 0u, 0u);
                    if (i < hi) r4[u] = __ldg(reinterpret_cast<const uint4 *>(recs + i));
                }
                if (!norm_ready) {                             // CTA-uniform: first pass of a staged tile
                    asm volatile("cp.async.wait_all;" ::: "memory");
                    __syncthreads();
                    norm_ready = true;
                }
    #pragma unroll
                for (int u = 0; u < QU; u++) {
                    const u32 i = base + (u * SA_TERM_THREADS + tid) * 4;
                    const u32 rr[4] = {r4[u].x, r4[u].y, r4[u].z, r4[u].w};
    #pragma unroll
                    for (int e = 0; e < 4; e++) {
                        if (i + e < lo || i + e >= hi) continue;
                        const u32 rel = rr[e] >> SA_REC_TF_BITS, tf = rr[e] & SA_REC_TF_MASK;
                        float v = (float)tf;
                        if (MODE == TERM_MODE_SCORE) {
                            v = 0.0f;
                            if (tf) {
                                v = bm25_from_norm((float)tf, staged_norm ? s_out[rel] : 1.0f, tq.idf);
                                my_max = max(my_max, __float_as_uint(v));
                            }
                        }
                        s_out[rel] = staged_norm ? -v : v;
                    }
                }
            }
        } else {
            // sparse tiles: ONE record per thread, so the threads' maxima (the tile bound of step 3) come from as
            // many distinct docs as possible
            for (u32 base = lo; base < hi; base += SA_TERM_THREADS) {                 // CTA-uniform trip count
                const u32 i = base + tid;
                const bool live = i < hi;
                const u32 r = live ? __ldg(recs + i) : 0u;
                float nrm = 1.0f;
                if (MODE == TERM_MODE_SCORE && !staged_norm && live) nrm = __ldg(norm + (r >> SA_REC_TF_BITS));
                if (!norm_ready) {                         // CTA-uniform: first pass of a staged tile
                    asm volatile("cp.async.wait_all;" ::: "memory");
                    __syncthreads();
                    norm_ready = true;
                }
                if (live) {
                    const u32 rel = r >> SA_REC_TF_BITS, tf = r & SA_REC_TF_MASK;
                    float v = (float)tf;
                    if (MODE == TERM_MODE_SCORE) {
                        v = 0.0f;
                        if (tf) {
                            v = bm25_from_norm((float)tf, staged_norm ? s_out[rel] : nrm, tq.idf);
                            my_max = max(my_max, __float_as_uint(v));
                        }
                    }
                    s_out[rel] = staged_norm ? -v : v;
                }
            }
        }
    } else {
    // CTA-uniform schedule: big slices in 4-window passes, the remainder (and small tiles) in
    // single-window passes so sparse tiles do not pay for empty windows.
    u32 base = lo;
    while (base < hi && hi - base > WIN) {
        windows(std::integral_constant<int, SA_TERM_UNROLL>{}, base);
        base += WIN * SA_TERM_UNROLL;
    }
    while (base < hi) {
        windows(std::integral_constant<int, 1>{}, base);
        base += WIN;
    }
    }

    // 3. flush the tile and collect its top-k candidates.  A tile with no more postings than k needs no bound: every
    //    positive score fits.  (Keeping every positive score of tiles with up to `slots` postings instead was measured
    //    slower, df/N 1e-2: 9.9 vs 9.2 us/query: candidates cost more than the bound.)  Threads that can hold a score:
    //    one per record / posting word, or one per quad of records on the dense tf-table path.
    auto finish = [&](unsigned g, float4 &v) {
        if (staged_norm) {                                  // sign set: a (negated) score; clear: a leftover norm
            v.x = __float_as_int(v.x) < 0 ? -v.x : 0.0f;
            v.y = __float_as_int(v.y) < 0 ? -v.y : 0.0f;
            v.z = __float_as_int(v.z) < 0 ? -v.z : 0.0f;
            v.w = __float_as_int(v.w) < 0 ? -v.w : 0.0f;
        }
        if (ALL_DOCS && MODE == TERM_MODE_SCORE) {
            // bm25.pyx:20-25 over EVERY doc (NaN / inf / -0.0 cases of exotic parameters)
            Bm25Params p = a.bm25;
            p.idf = tq.idf;
            const u64 d = (u64)tile_doc0 + (u64)g * 4;
            const float *dl = a.doc_lens + d;
            v.x = (d + 0 < a.n_docs) ? bm25_one(v.x, dl[0], p) : 0.0f;
            v.y = (d + 1 < a.n_docs) ? bm25_one(v.y, dl[1], p) : 0.0f;
            v.z = (d + 2 < a.n_docs) ? bm25_one(v.z, dl[2], p) : 0.0f;
            v.w = (d + 3 < a.n_docs) ? bm25_one(v.w, dl[3], p) : 0.0f;
        }
    };
    // ALL_DOCS scores take no tie retry, which would evaluate BM25 over the tile again: a tile whose ties overflow
    // sends its query to the exact re-run (the padded row makes the tile always in bounds)
    flush_tile_collect<true, DEEP>(s_out, a.out + (u64)q * a.out_stride + tile_doc0, a.topk, q, tile, my_max, hi - lo,
                                   quads ? (hi - lo) / 4u : hi - lo, s_top, &s_ncand, &s_tile_max, finish,
                                   !(ALL_DOCS && MODE == TERM_MODE_SCORE));
}

// per-doc BM25 length norm, the inner part of bm25.pyx:21-23 with the same rounding sequence
__global__ void norm_kernel(const float *__restrict__ dl, float *__restrict__ norm, u64 n, u64 n_pad,
                            Bm25Params p) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_pad) return;
    float v = 0.0f;
    if (i < n) v = __fmul_rn(p.k1, __fadd_rn(p.one_minus_b, __fmul_rn(p.b, __fdiv_rn(dl[i], p.avg_doc_len))));
    norm[i] = v;
}

int sa_ensure_norm(sa_index *ix, float k1, float b, float avg_doc_len) {
    if (ix->norm_valid && ix->norm_k1 == k1 && ix->norm_b == b && ix->norm_avgdl == avg_doc_len) return SA_OK;
    const u64 n_pad = sa_padded_docs(ix->n_docs);
    if (!ix->d_norm.p) {
        int rc = ix->d_norm.allocate(std::max<u64>(n_pad, 1) * sizeof(float));
        if (rc) return rc;
        ix->device_bytes += n_pad * sizeof(float);
    }
    if (n_pad) {
        norm_kernel<<<(unsigned)((n_pad + 255) / 256), 256, 0, ix->stream>>>(ix->d_doc_lens.as<float>(), ix->d_norm.as<float>(),
                                                                           ix->n_docs, n_pad,
                                                                           make_bm25(0, avg_doc_len, k1, b, ix->doc_lens_nonneg));
        SA_CUDA(cudaGetLastError());
        ix->stats.total_launches++;
    }
    ix->norm_k1 = k1; ix->norm_b = b; ix->norm_avgdl = avg_doc_len;
    ix->norm_valid = true;
    return SA_OK;
}

int launch_term_batch(sa_index *ix, const TermBatchArgs &a_in, u32 n_queries, u32 group) {
    if (n_queries == 0 || a_in.n_docs == 0) return SA_OK;
    TermBatchArgs a = a_in;
    const unsigned n_tiles = sa_n_tiles(a.n_docs);
    SA_CHECK((u64)n_queries * n_tiles <= 0x7fffffffu, "term launch of %u queries x %u tiles exceeds the grid", n_queries,
             n_tiles);
    static const bool env_qmajor = getenv("SA_TERM_QUERY_MAJOR") && atoi(getenv("SA_TERM_QUERY_MAJOR")) != 0;
    if (env_qmajor) group = 1;
    a.n_queries = n_queries;
    a.n_tiles = n_tiles;
    a.group = (group == 0 || group > n_queries) ? n_queries : group;
    a.group_ctas = a.group * n_tiles;
    {
        // tuning knobs, read per launch (a getenv costs nanoseconds; tools/term_buckets.py sweeps them in one process)
        const char *e;
        // the staged-norm thresholds are at least 1: a tile with no records or words must not stage norms, since it
        // would exit with its cp.async copies still in flight
        a.staged_norm_min_words = std::max(1u, (e = getenv("SA_STAGED_NORM_MIN_WORDS")) ? (u32)atol(e) : SA_STAGED_NORM_MIN_WORDS);
        a.staged_norm_min_recs = std::max(1u, (e = getenv("SA_STAGED_NORM_MIN_RECS")) ? (u32)atol(e) : SA_STAGED_NORM_MIN_RECS);
        a.quad_min_recs = (e = getenv("SA_TERM_QUAD_MIN_RECS")) ? (u32)atol(e) : SA_TERM_QUAD_MIN_RECS;
        // tile + d of a query is dispatched group * d CTAs later: d = one generation of resident CTAs, rounded up
        a.prefetch_tiles = (e = getenv("SA_TERM_PREFETCH_TILES"))
                               ? (u32)atol(e)
                               : std::max(1u, ((a.topk.k > SA_TOPK_MAX ? SA_TERM_DEEP_CTAS_PER_SM : SA_TERM_CTAS_PER_SM) *
                                                   (u32)ix->num_sms + a.group - 1) / a.group);
        a.quad_min_recs = std::max(a.quad_min_recs, a.staged_norm_min_recs);   // the quad path reads norms from the staged tile only
    }
    a.tile_dir = ix->d_tile_dir.as<u32>();
    // the tf table describes the index's own lists only
    a.recs = (a.words == ix->d_words.as<u64>()) ? ix->d_recs.as<u32>() : nullptr;
    a.rec_dir = ix->d_rec_dir.as<u32>();
    a.norm = ix->d_norm.as<float>();
    const bool sparse_score = (a.mode == TERM_MODE_SCORE) && a.bm25.sparse_ok;
    if (sparse_score) {
        int rc = sa_ensure_norm(ix, a.bm25.k1, a.bm25.b, a.bm25.avg_doc_len);
        if (rc) return rc;
        a.norm = ix->d_norm.as<float>();
    }
    const dim3 grid(n_queries * n_tiles), block(SA_TERM_THREADS);
    KernelTimer t(ix, 0);
    // top-k launches score without a payload filter (TF-mode and filtered launches collect nothing): the deep
    // instances exist for that case only
    const bool deep = a.topk.k > SA_TOPK_MAX;
    SA_CHECK(!deep || (a.mode == TERM_MODE_SCORE && !a.filter), "a deep top-k term launch scores without a filter");
    if (a.mode == TERM_MODE_TF) {
        if (a.filter) term_tile_kernel<TERM_MODE_TF, false, true, false><<<grid, block, 0, ix->stream>>>(a);
        else term_tile_kernel<TERM_MODE_TF, false, false, false><<<grid, block, 0, ix->stream>>>(a);
    } else if (sparse_score) {
        if (deep) term_tile_kernel<TERM_MODE_SCORE, false, false, true><<<grid, block, 0, ix->stream>>>(a);
        else if (a.filter) term_tile_kernel<TERM_MODE_SCORE, false, true, false><<<grid, block, 0, ix->stream>>>(a);
        else term_tile_kernel<TERM_MODE_SCORE, false, false, false><<<grid, block, 0, ix->stream>>>(a);
    } else {
        if (deep) term_tile_kernel<TERM_MODE_SCORE, true, false, true><<<grid, block, 0, ix->stream>>>(a);
        else if (a.filter) term_tile_kernel<TERM_MODE_SCORE, true, true, false><<<grid, block, 0, ix->stream>>>(a);
        else term_tile_kernel<TERM_MODE_SCORE, true, false, false><<<grid, block, 0, ix->stream>>>(a);
    }
    if (deep) ix->stats.deep_tiles += (u64)n_queries * n_tiles;
    SA_CUDA(cudaGetLastError());
    t.stop();
    ix->stats.term_kernel_launches++;
    ix->stats.term_kernel_queries += n_queries;
    ix->stats.term_kernel_groups += (n_queries + a.group - 1) / a.group;
    ix->stats.total_launches++;
    return SA_OK;
}
