// sa_comm.cu -- the one collective on the scoring path (SURVEY.md section 8e): every rank
// owns a contiguous doc-id range, scores its shard, and the per-shard top-k lists are
// exchanged with a single ncclAllGather per query batch, then merged on the device.
#include <dlfcn.h>
#include <nccl.h>      // types only: the library is bound at run time (see nccl_api)

#include "sa_term.cuh"

// NCCL is dlopen'ed on first use instead of being a link-time dependency: PyTorch bundles its own
// libnccl.so.2 under the same SONAME, and whichever copy a process loads first wins.  Binding
// lazily means this library never forces the (older) system copy on a process that also imports
// torch, and works without torch too.
struct NcclApi {
    ncclResult_t (*GetUniqueId)(ncclUniqueId *);
    ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int);
    ncclResult_t (*CommDestroy)(ncclComm_t);
    ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t);
    ncclResult_t (*AllReduce)(const void *, void *, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t);
    const char *(*GetErrorString)(ncclResult_t);
    bool ok = false;
};

static NcclApi *nccl_api() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        void *h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!h) return;
        api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(h, "ncclGetUniqueId");
        api.CommInitRank = (decltype(api.CommInitRank))dlsym(h, "ncclCommInitRank");
        api.CommDestroy = (decltype(api.CommDestroy))dlsym(h, "ncclCommDestroy");
        api.AllGather = (decltype(api.AllGather))dlsym(h, "ncclAllGather");
        api.AllReduce = (decltype(api.AllReduce))dlsym(h, "ncclAllReduce");
        api.GetErrorString = (decltype(api.GetErrorString))dlsym(h, "ncclGetErrorString");
        api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.AllReduce &&
                 api.GetErrorString;
    });
    return &api;
}

#define ncclGetUniqueId nccl_api()->GetUniqueId
#define ncclCommInitRank nccl_api()->CommInitRank
#define ncclCommDestroy nccl_api()->CommDestroy
#define ncclAllGather nccl_api()->AllGather
#define ncclAllReduce nccl_api()->AllReduce
#define ncclGetErrorString nccl_api()->GetErrorString
#define SA_NEED_NCCL()                                                              \
    do {                                                                            \
        if (!nccl_api()->ok) {                                                      \
            sa_set_error("libnccl.so.2 could not be loaded (%s)", dlerror());       \
            return SA_ERR_NCCL;                                                     \
        }                                                                           \
    } while (0)

#define SA_NCCL(call)                                                                  \
    do {                                                                               \
        ncclResult_t r_ = (call);                                                      \
        if (r_ != ncclSuccess) {                                                       \
            sa_set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call, ncclGetErrorString(r_)); \
            return SA_ERR_NCCL;                                                        \
        }                                                                              \
    } while (0)

extern "C" int sa_comm_unique_id(void *id128_out) {
    SA_CHECK(id128_out, "id buffer is NULL");
    SA_NEED_NCCL();
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    ncclUniqueId id;
    SA_NCCL(ncclGetUniqueId(&id));
    memcpy(id128_out, &id, sizeof(id));
    return SA_OK;
}

extern "C" int sa_comm_init(sa_index *ix, const void *id128, int rank, int world_size) {
    SA_CHECK(ix && id128, "NULL argument");
    SA_CHECK(world_size >= 1 && rank >= 0 && rank < world_size, "bad rank/world");
    SA_NEED_NCCL();
    std::lock_guard<std::mutex> g(ix->mu);
    SA_CUDA(cudaSetDevice(ix->device));
    ncclUniqueId id;
    memcpy(&id, id128, sizeof(id));
    ncclComm_t comm;
    SA_NCCL(ncclCommInitRank(&comm, world_size, id, rank));
    ix->nccl_comm = comm;
    ix->rank = rank;
    ix->world = world_size;
    return SA_OK;
}

extern "C" int sa_comm_destroy(sa_index *ix) {
    if (ix && ix->nccl_comm) {
        ncclCommDestroy((ncclComm_t)ix->nccl_comm);
        ix->nccl_comm = nullptr;
    }
    return SA_OK;
}

extern "C" int sa_comm_barrier(sa_index *ix) {
    SA_CHECK(ix && ix->nccl_comm, "communicator not initialised");
    std::lock_guard<std::mutex> g(ix->mu);
    SA_CUDA(cudaSetDevice(ix->device));
    int rc = ix->misc.reserve(256);
    if (rc) return rc;
    SA_CUDA(cudaMemsetAsync(ix->misc.p, 0, sizeof(float), ix->stream));
    SA_NCCL(ncclAllReduce(ix->misc.p, ix->misc.p, 1, ncclFloat, ncclSum, (ncclComm_t)ix->nccl_comm, ix->stream));
    SA_CUDA(cudaStreamSynchronize(ix->stream));
    return SA_OK;
}

extern "C" int sa_comm_allreduce_max(sa_index *ix, double *inout) {
    SA_CHECK(ix && ix->nccl_comm && inout, "communicator not initialised");
    std::lock_guard<std::mutex> g(ix->mu);
    SA_CUDA(cudaSetDevice(ix->device));
    int rc = ix->misc.reserve(256);
    if (rc) return rc;
    SA_CUDA(cudaMemcpyAsync(ix->misc.p, inout, sizeof(double), cudaMemcpyHostToDevice, ix->stream));
    SA_NCCL(ncclAllReduce(ix->misc.p, ix->misc.p, 1, ncclDouble, ncclMax, (ncclComm_t)ix->nccl_comm, ix->stream));
    SA_CUDA(cudaMemcpyAsync(inout, ix->misc.p, sizeof(double), cudaMemcpyDeviceToHost, ix->stream));
    SA_CUDA(cudaStreamSynchronize(ix->stream));
    return SA_OK;
}

// enqueue: all-gather the per-shard result blocks (keys + summary tail) and merge (async on the library stream)
static int enqueue_allgather_merge(sa_index *ix, size_t nq, u32 k) {
    const size_t nk = nq * k, blk = nk + SA_BATCH_TAIL;
    int rc;
    if ((rc = ix->gather.reserve(((size_t)ix->world * blk + nk + 8) * sizeof(u64)))) return rc;
    u64 *d_all = ix->gather.as<u64>();
    u64 *d_merged = d_all + (size_t)ix->world * blk;
    SA_NCCL(ncclAllGather(ix->topk_out.p, d_all, blk, ncclUint64, (ncclComm_t)ix->nccl_comm, ix->stream));
    if (nk == 0) return SA_OK;
    return launch_topk_merge(ix, d_all, blk, (u32)ix->world, (u32)nq, k, d_merged);
}

extern "C" int sa_batch_execute_allgather(sa_index *ix) {
    SA_CHECK(ix && ix->nccl_comm, "communicator not initialised (sa_comm_init)");
    std::lock_guard<std::mutex> g(ix->mu);
    int rc = sa_batch_execute_locked(ix);
    if (rc) return rc;
    u32 nq, k;
    sa_batch_dims(ix, &nq, &k);
    return enqueue_allgather_merge(ix, nq, k);
}

// merged keys + every rank's summary tail in one synchronise
static int download_merged(sa_index *ix, size_t nq, u32 k, uint32_t *out_docs, float *out_scores, u64 *redo_all, u64 *redo_mine,
                           bool count_stats) {
    const size_t nk = nq * k, blk = nk + SA_BATCH_TAIL;
    int rc;
    if ((rc = ix->h_pinned.reserve((nk + (size_t)ix->world * SA_BATCH_TAIL) * sizeof(u64)))) return rc;
    u64 *h = ix->h_pinned.as<u64>();
    const u64 *d_all = ix->gather.as<u64>();
    const u64 *d_merged = d_all + (size_t)ix->world * blk;
    if (nk) SA_CUDA(cudaMemcpyAsync(h, d_merged, nk * sizeof(u64), cudaMemcpyDeviceToHost, ix->stream));
    SA_CUDA(cudaMemcpy2DAsync(h + nk, SA_BATCH_TAIL * sizeof(u64), d_all + nk, blk * sizeof(u64), SA_BATCH_TAIL * sizeof(u64),
                              (size_t)ix->world, cudaMemcpyDeviceToHost, ix->stream));
    SA_CUDA(cudaStreamSynchronize(ix->stream));
    sa_unpack_keys(h, nk, out_docs, out_scores);
    *redo_all = 0;
    for (int r = 0; r < ix->world; r++) *redo_all += h[nk + (size_t)r * SA_BATCH_TAIL];
    *redo_mine = h[nk + (size_t)ix->rank * SA_BATCH_TAIL];
    if (count_stats) {
        ix->stats.phrase_cont_words += h[nk + (size_t)ix->rank * SA_BATCH_TAIL + 1];
        ix->stats.phrase_matched_docs += h[nk + (size_t)ix->rank * SA_BATCH_TAIL + 2];
    }
    return SA_OK;
}

extern "C" int sa_batch_download_allgather(sa_index *ix, uint32_t *out_docs, float *out_scores,
                                           uint32_t *n_overflow) {
    SA_CHECK(ix && ix->nccl_comm && out_docs && out_scores, "NULL argument / no communicator");
    std::lock_guard<std::mutex> g(ix->mu);
    u32 nq, k, redone = 0;
    sa_batch_dims(ix, &nq, &k);
    if (n_overflow) *n_overflow = 0;
    // every rank sees every rank's "queries to re-run" count (it travelled with the all-gathered keys), so all ranks
    // take the same path without a separate collective
    u64 redo_all = 0, redo_mine = 0;
    int rc = download_merged(ix, nq, k, out_docs, out_scores, &redo_all, &redo_mine, true);
    if (rc || redo_all == 0) return rc;
    if (redo_mine && (rc = sa_batch_fix_overflow_locked(ix, &redone))) return rc;
    if (n_overflow) *n_overflow = redone;
    // the repaired keys sit in topk_out; clear this rank's tail so the second gather reports a clean batch
    SA_CUDA(cudaMemsetAsync(ix->topk_out.as<u64>() + (size_t)nq * k, 0, SA_BATCH_TAIL * sizeof(u64), ix->stream));
    if ((rc = enqueue_allgather_merge(ix, nq, k))) return rc;
    return download_merged(ix, nq, k, out_docs, out_scores, &redo_all, &redo_mine, false);
}

extern "C" int sa_score_batch_topk_allgather(sa_index *ix, const uint32_t *terms, const uint32_t *term_starts,
                                             const float *idf, uint32_t n_queries, uint32_t slop,
                                             float avg_doc_len, float k1, float b, uint32_t k,
                                             uint32_t *out_docs, float *out_scores) {
    SA_CHECK(ix && out_docs && out_scores, "NULL argument");
    int rc = sa_batch_upload(ix, terms, term_starts, idf, n_queries, slop, avg_doc_len, k1, b, k);
    if (rc) return rc;
    if ((rc = sa_batch_execute_allgather(ix))) return rc;
    return sa_batch_download_allgather(ix, out_docs, out_scores, nullptr);
}

extern "C" int sa_comm_allreduce_sum_u64(sa_index *ix, uint64_t *inout, uint64_t n) {
    SA_CHECK(ix && ix->nccl_comm && (inout || n == 0), "communicator not initialised");
    std::lock_guard<std::mutex> g(ix->mu);
    SA_CUDA(cudaSetDevice(ix->device));
    if (n == 0) return SA_OK;
    int rc = ix->misc.reserve(n * sizeof(u64));
    if (rc) return rc;
    SA_CUDA(cudaMemcpyAsync(ix->misc.p, inout, n * sizeof(u64), cudaMemcpyHostToDevice, ix->stream));
    SA_NCCL(ncclAllReduce(ix->misc.p, ix->misc.p, n, ncclUint64, ncclSum, (ncclComm_t)ix->nccl_comm, ix->stream));
    SA_CUDA(cudaMemcpyAsync(inout, ix->misc.p, n * sizeof(u64), cudaMemcpyDeviceToHost, ix->stream));
    SA_CUDA(cudaStreamSynchronize(ix->stream));
    return SA_OK;
}
