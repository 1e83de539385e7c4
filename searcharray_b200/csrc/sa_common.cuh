// sa_common.cuh -- shared definitions for libsearcharray_b200 (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <algorithm>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <memory>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/searcharray_b200.h"

typedef uint64_t u64;
typedef uint32_t u32;
typedef int64_t i64;

// ---- roaringish bit layout (reference searcharray/roaringish/roaringish.py:30-35) ----
#define SA_KEY_SHIFT 36
#define SA_LSB_BITS 18
#define SA_LSB_MASK 0x3FFFFull
#define SA_HDR_MASK 0xFFFFFFFFFFFC0000ull
#define SA_MSB_MASK 0x0000000FFFFC0000ull
#define SA_BIT17 (1ull << 17)
#define SA_ONE_BLOCK (1ull << SA_LSB_BITS)
#define SA_MAX_POSN ((1u << 18) - 1)                   // reference roaringish.py:86: positions a doc may hold
#define SA_MAX_BLOCK (SA_MAX_POSN / SA_LSB_BITS)       // 14,563: the last block a posting word may carry

#define SA_NUM_SMS_FALLBACK 132          // H100 SXM

// ---- error plumbing -------------------------------------------------------------
void sa_set_error(const char *fmt, ...);

#define SA_CUDA(call)                                                                  \
    do {                                                                               \
        cudaError_t e_ = (call);                                                       \
        if (e_ != cudaSuccess) {                                                       \
            sa_set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
            return SA_ERR_CUDA;                                                        \
        }                                                                              \
    } while (0)

#define SA_CHECK(cond, ...)                                                            \
    do {                                                                               \
        if (!(cond)) {                                                                 \
            sa_set_error(__VA_ARGS__);                                                 \
            return SA_ERR_ARG;                                                         \
        }                                                                              \
    } while (0)

// ---- owned memory ---------------------------------------------------------------------
// Every cudaMalloc / cuMemCreate / cudaHostAlloc of the library is made by a Buffer (apart from sa_host_alloc's, which hands its
// memory to the caller), and the Buffer frees it when its owner goes away, on every return path.  A device buffer is
// destroyed while its device is current: ~sa_index and ~sa_multi set the device first, and locals live inside calls
// that have set it.
inline std::atomic<uint64_t> g_live_dev_buffers{0}, g_live_dev_bytes{0};   // sa_device_allocations

struct DeviceSpace {
    static constexpr const char *name = "cudaMalloc";
    static cudaError_t alloc(void **p, size_t bytes) {
        cudaError_t e = cudaMalloc(p, bytes);
        if (e == cudaSuccess && *p) { g_live_dev_buffers++; g_live_dev_bytes += bytes; }
        return e;
    }
    static void free(void *p, size_t bytes) {
        cudaFree(p);
        g_live_dev_buffers--;
        g_live_dev_bytes -= bytes;
    }
};

struct PinnedSpace {
    static constexpr const char *name = "cudaHostAlloc";
    static cudaError_t alloc(void **p, size_t bytes) { return cudaHostAlloc(p, bytes, cudaHostAllocDefault); }
    static void free(void *p, size_t) { cudaFreeHost(p); }
};

// Device memory the L2 may compress on its way to DRAM (Hopper's generic compute data compression): the term batch's
// score rows, most of whose 128-byte lines are zero.  cuMemCreate with
// CU_MEM_ALLOCATION_COMP_GENERIC, mapped at a reserved address for the current device; plain cudaMalloc where the
// device does not support it, the driver does not grant it, or SA_DENSE_PLAIN=1 (read once per process).  Freeing
// synchronises the device first, as cudaFree does: the rows may still be written on any of the library's streams.
// Contents and addresses behave as cudaMalloc's; sa_device_allocations counts the mapped bytes.  sa_index.cu.
struct CompressibleSpace {
    static constexpr const char *name = "compressible device alloc";
    static cudaError_t alloc(void **p, size_t bytes);
    static void free(void *p, size_t bytes);
    static bool compressible(const void *p);   // p came from cuMemCreate with compression granted
    // bytes a compressible mapping is rounded to; 0 when the current device has no support or SA_DENSE_PLAIN is set
    static size_t granularity();
};

template <typename Space> struct Buffer {
    void *p = nullptr;
    size_t cap = 0;
    Buffer() = default;
    Buffer(const Buffer &) = delete;
    Buffer &operator=(const Buffer &) = delete;
    Buffer(Buffer &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    Buffer &operator=(Buffer &&o) noexcept {
        if (this != &o) {
            reset();
            std::swap(p, o.p);
            std::swap(cap, o.cap);
        }
        return *this;
    }
    ~Buffer() { reset(); }
    // At least `bytes`; the contents are not kept.  Grows geometrically: cudaFree + cudaMalloc synchronise the
    // device, so a buffer that creeps up query by query must not be reallocated on every new maximum.
    int reserve(size_t bytes) {
        if (bytes <= cap) return SA_OK;
        return allocate(std::max(bytes + (bytes >> 3), cap + (cap >> 1)) + 256);
    }
    // Exactly `bytes` (the index's fixed arrays); the contents are not kept.
    int allocate(size_t bytes) {
        reset();
        cudaError_t e = Space::alloc(&p, bytes);
        if (e != cudaSuccess) {
            sa_set_error("%s(%zu) failed: %s", Space::name, bytes, cudaGetErrorString(e));
            p = nullptr;
            return SA_ERR_NOMEM;
        }
        cap = bytes;
        return SA_OK;
    }
    void reset() {
        if (p) Space::free(p, cap);
        p = nullptr;
        cap = 0;
    }
    template <typename T> T *as() const { return (T *)p; }
};
using DevBuf = Buffer<DeviceSpace>;
using PinnedBuf = Buffer<PinnedSpace>;
using RowBuf = Buffer<CompressibleSpace>;
// The term batch scans its rows in compressible memory in query groups of SA_COMP_ROW_GROUP (0 = all), or of
// SA_COMP_ROW_GROUP from the environment, read per launch.  Swept on H100 (DESIGN §6).
#define SA_COMP_ROW_GROUP 16
static_assert(!std::is_copy_constructible<DevBuf>::value, "a DevBuf has exactly one owner");

// The scratch arrays of one call, freed when the set goes out of scope.
struct DevMem {
    std::vector<DevBuf> bufs;
    template <typename T> T *alloc(size_t n) {
        DevBuf b;
        if (b.allocate(std::max<size_t>(n, 1) * sizeof(T) + 64)) return nullptr;
        bufs.push_back(std::move(b));
        return bufs.back().as<T>();
    }
    template <typename T> T *upload(const T *h, size_t n) {
        T *d = alloc<T>(n + 4);                       // pad: staged copies read up to 2 words past a slice
        if (!d || cudaMemset(d + n, 0, 4 * sizeof(T)) != cudaSuccess) return nullptr;
        if (n && cudaMemcpy(d, h, n * sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess) return nullptr;
        return d;
    }
};

// ---- BM25 parameters as the reference passes them to bm25_score ---------------------
struct Bm25Params {
    float idf, avg_doc_len, k1, b, one_minus_b;
    // 1 when a doc with tf == 0 provably scores +0.0f (k1>0, 0<=b<1, finite idf>=+0,
    // doc_lens >= 0, avgdl > 0): the kernel then only touches doc_lens of matching docs.
    // 0 -> the formula is evaluated for every doc like bm25.pyx:20-25 does (NaN/inf/-0.0
    // cases included).
    int sparse_ok;
};

// A query against one shard, as the kernels see it.
#define SA_NO_DIR 0xFFFFFFFFFFFFFFFFull
#define SA_FACET_NONE 0xFFFFu           // a facet column's code of a doc without a value (sa_index::d_facets)
#define SA_FACET_SET_WORDS (SA_FACET_MAX_BUCKETS / 32)   // u32 words of a set of facet codes, one bit per code
struct TermQuery {
    u64 word_off;      // offset of the term's first word in d_words
    u64 n_words;       // 0 => unknown term (zeros)
    u64 dir_off;       // offset of the term's tile directory in d_tile_dir (and d_rec_dir), or SA_NO_DIR
    u64 rec_off;       // offset of the term's (doc, tf) records in d_recs, or SA_NO_DIR
    float idf;
    u32 pad;
};

// (doc, tf) record of the per-term tf table: doc index RELATIVE to its 8192-doc tile in the high 13 bits,
// term frequency (sum of the doc's payload popcounts, < 2^18 + 1) in the low 19
#define SA_REC_TF_BITS 19
#define SA_REC_TF_MASK 0x7FFFFu

// ---- the index handle ---------------------------------------------------------------
struct TimedLaunch { cudaEvent_t e0, e1; int kind; };   // kind: 0 term, 1 topk, 2 phrase (see KernelTimer)
struct BatchState;
struct ViewState;
struct BatchStateDelete { void operator()(BatchState *b) const; };   // sa_index.cu
struct ViewStateDelete { void operator()(ViewState *v) const; };     // sa_view.cu
struct BoolState;
struct BoolStateDelete { void operator()(BoolState *s) const; };     // sa_bool.cu
struct sa_index {
    ~sa_index();
    int device = 0;
    int num_sms = SA_NUM_SMS_FALLBACK;
    u64 n_docs = 0, n_words = 0, doc_base = 0;
    u32 n_terms = 0;
    bool doc_lens_nonneg = true;
    int upload_mode = 0;             // how the posting words reached HBM (sa_index_upload_mode)

    // HBM-resident index
    DevBuf d_words;                  // u64 [n_words + 1] (one readable pad word)
    DevBuf d_doc_lens;               // float [n_docs]
    DevBuf d_df;                     // u32 [n_terms] distinct docs per term (this shard)
    // tile directory of long posting lists: for term t with h_dir_off[t] != SA_NO_DIR,
    // d_tile_dir[h_dir_off[t] + j] = index (within the term's list) of the first word whose
    // doc lies in tile >= j, j = 0..n_tiles  (tile = 4096 docs).  Built on the device at upload.
    DevBuf d_tile_dir;               // u32
    std::vector<u64> h_dir_off;
    // per-term tf table (the analogue of the reference's termfreq_cache, middle_out.py:501-509, built on the
    // device at upload): for every term WITH a tile directory, one u32 record per (term, doc) in doc order,
    // (doc - tile_doc0) << 19 | tf; d_rec_dir mirrors d_tile_dir (same offsets) with indices into the records.
    DevBuf d_recs;                   // u32
    DevBuf d_rec_dir;                // u32
    std::vector<u64> h_rec_off;
    // per-doc BM25 length norm k1*((1-b)+b*dl/avgdl) for the last used (k1, b, avgdl)
    DevBuf d_norm;                   // float [padded n_docs]
    float norm_k1 = 0, norm_b = 0, norm_avgdl = 0;
    bool norm_valid = false;
    // feature columns (sa_index_set_feature, sa_feature.cu): slot s, when bit s of feature_set is set, is
    // d_features[s] (float [padded n_docs], zero past n_docs) and its tile flags d_feature_tiles[s * n_tiles + t]
    // (1: some doc of tile t has a value > 0) and bounds d_feature_bounds[s * n_tiles + t] (the min and max of the
    // tile's values > 0, read by range clauses)
    DevBuf d_features[SA_MAX_FEATURES];
    DevBuf d_feature_tiles;          // u32 [SA_MAX_FEATURES * n_tiles]
    DevBuf d_feature_bounds;         // float2 [SA_MAX_FEATURES * n_tiles]
    u32 feature_set = 0;
    // facet columns (sa_index_set_facet, sa_feature.cu): slot s, when bit s of facet_set is set, is d_facets[s]
    // (uint16 [padded n_docs], a doc's bucket or 0xFFFF for none, 0xFFFF past n_docs) with facet_buckets[s] buckets,
    // and d_facet_tiles[s] the codes present in each tile (u32 [n_tiles][SA_FACET_SET_WORDS], bit c: code c), read by
    // In clauses
    DevBuf d_facets[SA_MAX_FACETS];
    DevBuf d_facet_tiles[SA_MAX_FACETS];
    u32 facet_buckets[SA_MAX_FACETS] = {};
    u32 facet_set = 0;
    // group columns (sa_index_set_group, sa_feature.cu): slot s, when bit s of group_set is set, is d_groups[s]
    // (u32 [padded n_docs], a doc's group or SA_GROUP_NONE, SA_GROUP_NONE past n_docs), read by the collapsed top-k
    DevBuf d_groups[SA_MAX_GROUPS];
    u32 group_set = 0;
    // host mirrors for query set-up
    std::vector<u64> h_off, h_len;
    std::vector<u32> h_df;
    std::vector<unsigned char> h_first0;   // 1 = the term's first word sits at (doc 0, block 0): span-search corner

    // sliced-array filter (FilteredPosns semantics)
    u64 n_rows = 0;                  // number of selected rows
    bool rows_active = false;        // a row filter is installed (n_rows may be 0)
    // one buffer, so that installing a filter allocates once: the row mask (unsigned char [n_docs], 1 if doc selected),
    // then the rows (u64, sorted local doc indices) at row_mask_bytes()
    DevBuf row_filter;
    size_t row_mask_bytes() const { return (std::max<u64>(n_docs, 1) + 15) & ~(size_t)15; }
    unsigned char *d_row_mask() const { return row_filter.as<unsigned char>(); }
    u64 *d_rows() const { return row_filter.p ? (u64 *)(row_filter.as<char>() + row_mask_bytes()) : nullptr; }

    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;   // sa_timer_start / sa_timer_stop
    bool profiling = false;
    std::vector<TimedLaunch> pending_timers;
    std::vector<cudaEvent_t> free_events;
    std::unique_ptr<BatchState, BatchStateDelete> batch;
    std::unique_ptr<ViewState, ViewStateDelete> view;   // buffers of sa_score_batch_topk_sim (sa_view.cu)
    std::unique_ptr<BoolState, BoolStateDelete> boolq;  // buffers of sa_score_batch_topk_bool (sa_bool.cu)
    sa_stats stats;
    std::mutex mu;

    // scratch
    DevBuf dense;        // float [chunk][n_docs_padded]
    RowBuf comp_rows;    // term batch: a chunk's rows in compressible memory, each padded to the granularity (sa_batch_upload)
    DevBuf queries;      // TermQuery[] / phrase descriptors
    DevBuf cand;         // top-k candidates
    DevBuf cand_meta;    // per-query counters / thresholds
    DevBuf topk_out;     // per-query (doc, score) results
    DevBuf phrase_scratch;
    DevBuf filt;         // filtered (sliced / position-filtered) copies of posting lists
    DevBuf misc;
    PinnedBuf h_pinned;  // pinned staging

    // NCCL
    void *nccl_comm = nullptr;
    int rank = 0, world = 1;
    DevBuf gather;

    size_t device_bytes = 0;
};

// Kernel timing without serialising the stream: when profiling is on every timed launch gets
// an event pair from a pool; elapsed times are resolved lazily (sa_stats_get syncs once).
struct KernelTimer {
    sa_index *ix;
    int kind;
    bool on;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    KernelTimer(sa_index *ix_, int kind_);
    void stop();
};
int sa_resolve_timers(sa_index *ix);
// sa_index_create, or with refuse_past_max_posn == false an index that also accepts words whose block lies past
// SA_MAX_BLOCK (sa_op_bigram_freqs: the reference's bigram_freqs takes any word; its count never reads a tf record)
int sa_index_create_blocks(const uint64_t *words, uint64_t n_words,
                           const uint64_t *term_offsets, const uint64_t *term_lengths, uint32_t n_terms,
                           const float *doc_lens, uint64_t n_docs, uint64_t doc_base,
                           int device, bool refuse_past_max_posn, sa_index **index_out);

// ---- device helpers -------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ u64 ld_stream_u64(const u64 *p) {
    u64 v;
    asm volatile("ld.global.nc.L1::no_allocate.u64 %0, [%1];" : "=l"(v) : "l"(p));
    return v;
}

// BM25 exactly as bm25.pyx:20-25 evaluates it on x86-64 without FMA contraction:
// every operation individually rounded to nearest-even float32.
__device__ __forceinline__ float bm25_one(float tf, float dl, const Bm25Params &p) {
    float ratio = __fdiv_rn(dl, p.avg_doc_len);
    float norm = __fmul_rn(p.k1, __fadd_rn(p.one_minus_b, __fmul_rn(p.b, ratio)));
    return __fmul_rn(__fdiv_rn(tf, __fadd_rn(tf, norm)), p.idf);
}

// Warp-cooperative lower bound: first index i in [lo, hi) with (a[i] >> shift) >= key,
// 32-ary search (each round probes 32 evenly spaced elements, ballot picks the bucket).
// All lanes must call; all lanes get the result.
__device__ __forceinline__ u64 warp_lower_bound_shifted(const u64 *__restrict__ a, u64 lo, u64 hi,
                                                        u64 key, int shift) {
    const unsigned lane = threadIdx.x & 31;
    while (hi - lo > 32) {
        u64 step = (hi - lo + 31) >> 5;          // ceil(len/32) >= 2
        u64 probe = lo + (u64)(lane + 1) * step - 1;   // last element of bucket `lane`
        bool below = (probe < hi) && ((__ldg(a + probe) >> shift) < key);
        unsigned m = __ballot_sync(0xffffffffu, below);
        int c = __popc(m);                        // buckets entirely below key (monotone)
        lo = lo + (u64)c * step;
        u64 nhi = lo + step;
        hi = nhi < hi ? nhi : hi;
        if (lo > hi) lo = hi;
    }
    u64 idx = lo + lane;
    bool below = (idx < hi) && ((__ldg(a + idx) >> shift) < key);
    unsigned m = __ballot_sync(0xffffffffu, below);
    return lo + (u64)__popc(m);
}
#endif
