// sa_index.cu -- index upload into HBM, per-term document frequencies, and the C-ABI entry
// points of the term path (see include/searcharray_b200.h for the reference mapping).
#include <cuda.h>
#include <cudaTypedefs.h>
#include <stdarg.h>
#include <algorithm>
#include <unordered_map>

#include "sa_term.cuh"
#include "sa_phrase.cuh"
#include "sa_scan.cuh"
#include "sa_sim.cuh"
#include "sa_span.cuh"

// ------------------------------------------------------------------ error text
static thread_local char g_err[1024] = "";

void sa_set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" const char *sa_last_error(void) { return g_err; }

extern "C" int sa_device_count(int *n_out) {
    SA_CHECK(n_out, "n_out is NULL");
    int n = 0;
    SA_CUDA(cudaGetDeviceCount(&n));
    *n_out = n;
    return SA_OK;
}

extern "C" int sa_host_alloc(void **ptr_out, uint64_t bytes) {
    SA_CHECK(ptr_out, "ptr_out is NULL");
    SA_CUDA(cudaHostAlloc(ptr_out, bytes ? bytes : 1, cudaHostAllocDefault));
    return SA_OK;
}

extern "C" int sa_host_free(void *ptr) {
    if (ptr) SA_CUDA(cudaFreeHost(ptr));
    return SA_OK;
}

extern "C" int sa_device_allocations(uint64_t *live_buffers, uint64_t *live_bytes) {
    SA_CHECK(live_buffers && live_bytes, "NULL argument");
    *live_buffers = g_live_dev_buffers;
    *live_bytes = g_live_dev_bytes;
    return SA_OK;
}

// --------------------------------------------------------------- compressible score rows (CompressibleSpace)
// The driver's virtual memory calls are reached through the runtime, so the library links against cudart alone.
namespace {
struct VmmApi {
    PFN_cuDeviceGetAttribute_v2000 getAttribute = nullptr;
    PFN_cuMemGetAllocationGranularity_v10020 granularity = nullptr;
    PFN_cuMemCreate_v10020 create = nullptr;
    PFN_cuMemGetAllocationPropertiesFromHandle_v10020 properties = nullptr;
    PFN_cuMemRelease_v10020 release = nullptr;
    PFN_cuMemAddressReserve_v10020 reserve = nullptr;
    PFN_cuMemAddressFree_v10020 addressFree = nullptr;
    PFN_cuMemMap_v10020 map = nullptr;
    PFN_cuMemUnmap_v10020 unmap = nullptr;
    PFN_cuMemSetAccess_v10020 setAccess = nullptr;
    bool ok = false;
};

template <typename F> bool driver_entry(const char *symbol, F *fn) {
    cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
    return cudaGetDriverEntryPointByVersion(symbol, (void **)fn, 12000, cudaEnableDefault, &q) == cudaSuccess &&
           q == cudaDriverEntryPointSuccess && *fn;
}

// nullptr when SA_DENSE_PLAIN=1 or the driver lacks an entry point
const VmmApi *vmm_api() {
    static const VmmApi api = [] {
        VmmApi a;
        if (getenv("SA_DENSE_PLAIN") && atoi(getenv("SA_DENSE_PLAIN")) != 0) return a;
        a.ok = driver_entry("cuDeviceGetAttribute", &a.getAttribute) &&
               driver_entry("cuMemGetAllocationGranularity", &a.granularity) && driver_entry("cuMemCreate", &a.create) &&
               driver_entry("cuMemGetAllocationPropertiesFromHandle", &a.properties) &&
               driver_entry("cuMemRelease", &a.release) && driver_entry("cuMemAddressReserve", &a.reserve) &&
               driver_entry("cuMemAddressFree", &a.addressFree) && driver_entry("cuMemMap", &a.map) &&
               driver_entry("cuMemUnmap", &a.unmap) && driver_entry("cuMemSetAccess", &a.setAccess);
        return a;
    }();
    return api.ok ? &api : nullptr;
}

// The live compressible mappings: base address -> mapped bytes (the request rounded up to the granularity).
std::mutex g_vmm_mu;
std::unordered_map<const void *, size_t> g_vmm_maps;

// The current device's compressible allocation properties and their granularity, or 0 when it has none.
size_t compressible_prop(const VmmApi &api, CUmemAllocationProp *prop) {
    int device = 0, supported = 0;
    if (cudaGetDevice(&device) != cudaSuccess || cudaSetDevice(device) != cudaSuccess ||   // primary context current
        api.getAttribute(&supported, CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED, device) != CUDA_SUCCESS ||
        !supported)
        return 0;
    *prop = {};
    prop->type = CU_MEM_ALLOCATION_TYPE_PINNED;
    prop->location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    prop->location.id = device;
    prop->allocFlags.compressionType = CU_MEM_ALLOCATION_COMP_GENERIC;
    size_t gran = 0;
    if (api.granularity(&gran, prop, CU_MEM_ALLOC_GRANULARITY_MINIMUM) != CUDA_SUCCESS) return 0;
    return gran;
}

// cuMemCreate + reserve + map + access with compression granted, or nullptr (nothing left behind).
void *map_compressible(const VmmApi &api, size_t bytes, size_t *mapped) {
    CUmemAllocationProp prop;
    const size_t gran = compressible_prop(api, &prop);
    if (!gran) return nullptr;
    const size_t size = (bytes + gran - 1) / gran * gran;
    CUmemGenericAllocationHandle h;
    if (api.create(&h, size, &prop, 0) != CUDA_SUCCESS) return nullptr;
    CUmemAllocationProp got = {};
    CUdeviceptr va = 0;
    bool ok = api.properties(&got, h) == CUDA_SUCCESS && got.allocFlags.compressionType == CU_MEM_ALLOCATION_COMP_GENERIC;
    ok = ok && api.reserve(&va, size, gran, 0, 0) == CUDA_SUCCESS;
    bool mapped_ok = ok && api.map(va, size, 0, h, 0) == CUDA_SUCCESS;
    api.release(h);                                   // the mapping keeps the memory until it is unmapped
    CUmemAccessDesc access = {};
    access.location = prop.location;
    access.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    if (mapped_ok && api.setAccess(va, size, &access, 1) == CUDA_SUCCESS) {
        *mapped = size;
        return (void *)va;
    }
    if (mapped_ok) api.unmap(va, size);
    if (va) api.addressFree(va, size);
    return nullptr;
}
}  // namespace

cudaError_t CompressibleSpace::alloc(void **p, size_t bytes) {
    if (const VmmApi *api = vmm_api()) {
        size_t mapped = 0;
        if (void *va = map_compressible(*api, bytes, &mapped)) {
            std::lock_guard<std::mutex> lk(g_vmm_mu);
            g_vmm_maps[va] = mapped;
            *p = va;
            g_live_dev_buffers++;
            g_live_dev_bytes += mapped;
            return cudaSuccess;
        }
    }
    return DeviceSpace::alloc(p, bytes);
}

void CompressibleSpace::free(void *p, size_t bytes) {
    size_t mapped = 0;
    {
        std::lock_guard<std::mutex> lk(g_vmm_mu);
        auto it = g_vmm_maps.find(p);
        if (it != g_vmm_maps.end()) {
            mapped = it->second;
            g_vmm_maps.erase(it);
        }
    }
    if (!mapped) return DeviceSpace::free(p, bytes);
    const VmmApi *api = vmm_api();
    cudaDeviceSynchronize();                          // cudaFree's implicit synchronisation: no kernel still writes p
    api->unmap((CUdeviceptr)p, mapped);
    api->addressFree((CUdeviceptr)p, mapped);
    g_live_dev_buffers--;
    g_live_dev_bytes -= mapped;
}

size_t CompressibleSpace::granularity() {
    const VmmApi *api = vmm_api();
    CUmemAllocationProp prop;
    return api ? compressible_prop(*api, &prop) : 0;
}

bool CompressibleSpace::compressible(const void *p) {
    std::lock_guard<std::mutex> lk(g_vmm_mu);
    return p && g_vmm_maps.count(p);
}

// --------------------------------------------------------------- bulk upload
// SURVEY 8f-2: the posting words usually sit in pageable memory -- a numpy array, or the np.memmap of the
// reference's MemoryMappedArrays `.dat` file (phrase/memmap_arrays.py:145-208).  A plain cudaMemcpy from pageable
// memory crawls through the driver's small staging buffers; instead the source range is page-locked IN PLACE
// (cudaHostRegister, read-only: works on a read-only file mapping too) and copied by DMA at PCIe rate straight from
// the page cache / the array.  If the range cannot be registered (old kernels, exotic mappings) the copy is pipelined
// through two pinned bounce buffers.  mode_out: 0 plain copy (small), 1 registered in place, 2 pinned bounce.
static int upload_bulk(void *dst, const void *src, size_t bytes, cudaStream_t stream, int *mode_out) {
    *mode_out = 0;
    if (bytes == 0) return SA_OK;
    static const bool no_register = getenv("SA_NO_HOST_REGISTER") && atoi(getenv("SA_NO_HOST_REGISTER")) != 0;
    if (bytes >= (32u << 20)) {
        if (!no_register && cudaHostRegister((void *)src, bytes, cudaHostRegisterReadOnly) == cudaSuccess) {
            cudaError_t e = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
            cudaHostUnregister((void *)src);
            if (e != cudaSuccess) { sa_set_error("registered upload failed: %s", cudaGetErrorString(e)); return SA_ERR_CUDA; }
            *mode_out = 1;
            return SA_OK;
        }
        cudaGetLastError();                                   // registration refused: clear the error, bounce instead
        const size_t CH = 32u << 20;
        struct EventDestroy { void operator()(cudaEvent_t e) const { cudaEventDestroy(e); } };
        PinnedBuf pin[2];
        std::unique_ptr<CUevent_st, EventDestroy> ev[2];
        bool ok = pin[0].allocate(CH) == SA_OK && pin[1].allocate(CH) == SA_OK;
        for (int i = 0; i < 2 && ok; i++) {
            cudaEvent_t e = nullptr;
            ok = cudaEventCreate(&e) == cudaSuccess;
            ev[i].reset(e);
        }
        if (ok) {
            size_t at = 0;
            int b = 0;
            cudaError_t e = cudaSuccess;
            while (at < bytes && e == cudaSuccess) {
                const size_t n = std::min(CH, bytes - at);
                e = cudaEventSynchronize(ev[b].get());        // the previous copy out of this buffer is done
                if (e != cudaSuccess) break;
                memcpy(pin[b].p, (const char *)src + at, n);
                e = cudaMemcpyAsync((char *)dst + at, pin[b].p, n, cudaMemcpyHostToDevice, stream);
                if (e == cudaSuccess) e = cudaEventRecord(ev[b].get(), stream);
                at += n;
                b ^= 1;
            }
            if (e == cudaSuccess) e = cudaStreamSynchronize(stream);
            if (e != cudaSuccess) { sa_set_error("bounce upload failed: %s", cudaGetErrorString(e)); return SA_ERR_CUDA; }
            *mode_out = 2;
            return SA_OK;
        }
        cudaGetLastError();
    }
    SA_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream));
    return SA_OK;
}

// --------------------------------------------------------------- df, tile directories and the tf table at upload
// The upload kernels run one thread per posting word of the whole index; a word finds its term through the slots
// (the terms' slices, sorted by offset, covering `words` exactly).

// slot = last j with term_off_sorted[j] <= i   (slots cover [off, off+len) disjointly)
__device__ __forceinline__ u32 slot_of_word(const u64 *__restrict__ term_off_sorted, u32 n_slots, u64 i) {
    u32 lo = 0, hi = n_slots;
    while (hi - lo > 1) {
        u32 mid = (lo + hi) >> 1;
        if (term_off_sorted[mid] <= i) lo = mid; else hi = mid;
    }
    return lo;
}

// word i is a "doc head" when it starts its term's list (at `start`) or its doc id differs from its predecessor's
__device__ __forceinline__ bool is_doc_head(const u64 *__restrict__ words, u64 i, u64 start) {
    return i == start || (words[i] >> SA_KEY_SHIFT) != (words[i - 1] >> SA_KEY_SHIFT);
}

__device__ __forceinline__ u32 tile_of_word(u64 w, u64 doc_base) {
    return (u32)(((w >> SA_KEY_SHIFT) - doc_base) / SA_TILE_DOCS);
}

// The directory entries that word i of the list [start, start + len) fills: dir[t] = value for the tiles after its
// predecessor's, up to its own (from tile 0 for the list's first word), and dir[t] = end for the tiles after the list's
// last word.  A word of the same doc as its predecessor fills no tile of the first kind.
__device__ __forceinline__ void fill_tile_dir(u32 *__restrict__ dir, const u64 *__restrict__ words, u64 i, u64 start,
                                              u64 len, u32 value, u32 end, u64 doc_base, u32 n_tiles) {
    const u32 t_i = tile_of_word(words[i], doc_base);
    const u32 t0 = i == start ? 0 : tile_of_word(words[i - 1], doc_base) + 1;
    for (u32 t = t0; t <= t_i && t <= n_tiles; t++) dir[t] = value;
    if (i == start + len - 1)
        for (u32 t = t_i + 1; t <= n_tiles; t++) dir[t] = end;
}

// docfreq = number of distinct doc ids among a term's words (reference: unique(words >> 36)
// .size, roaringish/unique.pyx:87-104 via middle_out.py:521-528) = its doc heads.  A word whose block lies past
// MAX_POSN's sets *past_max_posn (one ballot per warp; an atomic only on a violation).
__global__ void df_kernel(const u64 *__restrict__ words, u64 n_words,
                          const u64 *__restrict__ term_off_sorted, const u32 *__restrict__ term_of_slot,
                          u32 n_slots, u32 *__restrict__ df, u32 *__restrict__ past_max_posn) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < n_words;
    u32 lo = 0;
    bool head = false;
    if (live) {
        lo = slot_of_word(term_off_sorted, n_slots, i);
        head = is_doc_head(words, i, term_off_sorted[lo]);
    }
    const bool past = live && ((words[i] >> SA_LSB_BITS) & SA_LSB_MASK) > SA_MAX_BLOCK;
    if (__ballot_sync(0xffffffffu, past) && (threadIdx.x & 31) == 0) atomicOr(past_max_posn, 1u);
    // a warp's 32 consecutive words almost always belong to one term: one atomic per (warp, term) instead of one
    // per doc head (a billion same-address atomics on a 10M-doc index)
    const unsigned heads = __ballot_sync(0xffffffffu, head);
    if (heads == 0) return;
    const unsigned peers = __match_any_sync(0xffffffffu, live ? lo : 0xFFFFFFFFu);
    const unsigned mine = heads & peers;
    if (live && mine && (threadIdx.x & 31) == (unsigned)(__ffs(peers) - 1)) atomicAdd(&df[term_of_slot[lo]], (u32)__popc(mine));
}

// Tile directory of a long posting list: dir[j] = index (within the list) of the first word whose
// doc falls in tile >= j, for j = 0..n_tiles.
__global__ void tile_dir_kernel(const u64 *__restrict__ words, u64 n_words,
                                const u64 *__restrict__ term_off_sorted, const u64 *__restrict__ slot_len,
                                const u64 *__restrict__ slot_dir_off, u32 n_slots,
                                u32 *__restrict__ dir, u64 doc_base, u32 n_tiles) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_words) return;
    const u32 slot = slot_of_word(term_off_sorted, n_slots, i);
    const u64 doff = slot_dir_off[slot];
    if (doff == SA_NO_DIR) return;
    const u64 start = term_off_sorted[slot], len = slot_len[slot];
    fill_tile_dir(dir + doff, words, i, start, len, (u32)(i - start), (u32)len, doc_base, n_tiles);
}

// ---- tf table (see sa_index::d_recs).  Pass 1 counts the doc heads of every 1024-word block, a one-CTA scan
// (cta_scan_kernel, sa_scan.cuh) turns the counts into ranks in place, pass 2 writes each head's record at (term's
// record offset + rank within the term) and fills the term's record directory with the heads' ranks.
#define REC_BLOCK 1024

__global__ void __launch_bounds__(256)
rec_count_kernel(const u64 *__restrict__ words, u64 n_words, const u64 *__restrict__ term_off_sorted, u32 n_slots,
                 u64 *__restrict__ bcount) {
    __shared__ u32 s_cnt;
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    u32 mine = 0;
    for (int e = 0; e < REC_BLOCK / 256; e++) {
        const u64 i = (u64)blockIdx.x * REC_BLOCK + e * 256 + threadIdx.x;
        if (i >= n_words) break;
        if (is_doc_head(words, i, term_off_sorted[slot_of_word(term_off_sorted, n_slots, i)])) mine++;
    }
    mine = __reduce_add_sync(0xffffffffu, mine);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(&s_cnt, mine);
    __syncthreads();
    if (threadIdx.x == 0) bcount[blockIdx.x] = s_cnt;
}

__global__ void __launch_bounds__(256)
rec_write_kernel(const u64 *__restrict__ words, u64 n_words, const u64 *__restrict__ term_off_sorted,
                 const u64 *__restrict__ slot_len, const u64 *__restrict__ slot_dir_off,
                 const u64 *__restrict__ slot_rec_off, const u64 *__restrict__ slot_head_base,
                 const u32 *__restrict__ slot_df, u32 n_slots, const u64 *__restrict__ bbase,
                 u32 *__restrict__ recs, u32 *__restrict__ rec_dir, u64 doc_base, u32 n_tiles) {
    __shared__ u32 s_warp[8];
    u32 run = 0;                                                                      // heads of the earlier rounds
    for (int e = 0; e < REC_BLOCK / 256; e++) {
        const u64 i = (u64)blockIdx.x * REC_BLOCK + e * 256 + threadIdx.x;
        bool head = false;
        u32 slot = 0;
        u64 start = 0;
        if (i < n_words) {
            slot = slot_of_word(term_off_sorted, n_slots, i);
            start = term_off_sorted[slot];
            head = is_doc_head(words, i, start);
        }
        u32 round_total;
        const u64 g = bbase[blockIdx.x] + run + block_exclusive_sum<256>(head ? 1u : 0u, s_warp, round_total);   // global head rank
        run += round_total;
        if (i < n_words && slot_dir_off[slot] != SA_NO_DIR) {
            const u64 len = slot_len[slot];
            const u32 rank = (u32)(g - slot_head_base[slot]);                         // within the term
            if (head) {
                const u64 w = words[i];
                u32 tf = 0;
                for (u64 j = i; j < start + len; j++) {                                // the doc's run of words
                    const u64 w2 = words[j];
                    if ((w2 >> SA_KEY_SHIFT) != (w >> SA_KEY_SHIFT)) break;
                    tf += (u32)__popcll(w2 & SA_LSB_MASK);
                }
                const u64 doc = (w >> SA_KEY_SHIFT) - doc_base;
                recs[slot_rec_off[slot] + rank] = ((u32)(doc % SA_TILE_DOCS) << SA_REC_TF_BITS) | (tf & SA_REC_TF_MASK);
            }
            fill_tile_dir(rec_dir + slot_dir_off[slot], words, i, start, len, rank, slot_df[slot], doc_base, n_tiles);
        }
    }
}

extern "C" int sa_index_create(const uint64_t *words, uint64_t n_words,
                               const uint64_t *term_offsets, const uint64_t *term_lengths, uint32_t n_terms,
                               const float *doc_lens, uint64_t n_docs, uint64_t doc_base,
                               int device, sa_index **index_out) {
    return sa_index_create_blocks(words, n_words, term_offsets, term_lengths, n_terms, doc_lens, n_docs, doc_base,
                                  device, true, index_out);
}

int sa_index_create_blocks(const uint64_t *words, uint64_t n_words,
                           const uint64_t *term_offsets, const uint64_t *term_lengths, uint32_t n_terms,
                           const float *doc_lens, uint64_t n_docs, uint64_t doc_base,
                           int device, bool refuse_past_max_posn, sa_index **index_out) {
    SA_CHECK(index_out, "index_out is NULL");
    SA_CHECK(n_words == 0 || words, "words is NULL");
    SA_CHECK(n_terms == 0 || (term_offsets && term_lengths), "term tables are NULL");
    SA_CHECK(n_docs == 0 || doc_lens, "doc_lens is NULL");
    SA_CHECK(doc_base + n_docs <= (1ull << 28), "doc ids exceed the 28-bit key space");
    for (u32 t = 0; t < n_terms; t++)
        SA_CHECK(term_offsets[t] + term_lengths[t] <= n_words, "term %u slice out of range", t);
    SA_CUDA(cudaSetDevice(device));

    std::unique_ptr<sa_index> ix(new sa_index());
    ix->device = device;
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) ix->num_sms = prop.multiProcessorCount;
    ix->n_docs = n_docs;
    ix->n_words = n_words;
    ix->n_terms = n_terms;
    ix->doc_base = doc_base;
    memset(&ix->stats, 0, sizeof(ix->stats));
    ix->h_off.assign(term_offsets, term_offsets + n_terms);
    ix->h_len.assign(term_lengths, term_lengths + n_terms);
    ix->h_df.assign(n_terms, 0);
    ix->h_dir_off.assign(n_terms, SA_NO_DIR);
    ix->h_first0.assign(n_terms, 0);
    ix->h_rec_off.assign(n_terms, SA_NO_DIR);
    for (u32 t = 0; t < n_terms; t++)
        if (term_lengths[t] && (words[term_offsets[t]] & SA_HDR_MASK) == 0) ix->h_first0[t] = 1;

    // a host table in a new device buffer of exactly its size, copied on the index's stream
    auto upload_table = [&](DevBuf &d, const auto &h) -> int {
        const size_t bytes = h.size() * sizeof(h[0]);
        int rc = d.allocate(bytes);
        if (rc) return rc;
        SA_CUDA(cudaMemcpyAsync(d.p, h.data(), bytes, cudaMemcpyHostToDevice, ix->stream));
        return SA_OK;
    };
    int rc;
    SA_CUDA(cudaStreamCreateWithFlags(&ix->stream, cudaStreamNonBlocking));
    SA_CUDA(cudaEventCreate(&ix->ev0));
    SA_CUDA(cudaEventCreate(&ix->ev1));
    if ((rc = ix->d_words.allocate((n_words + 4) * sizeof(u64)))) return rc;
    SA_CUDA(cudaMemsetAsync(ix->d_words.as<u64>() + n_words, 0, 4 * sizeof(u64), ix->stream));
    if (n_words && (rc = upload_bulk(ix->d_words.p, words, n_words * sizeof(u64), ix->stream, &ix->upload_mode))) return rc;
    if ((rc = ix->d_doc_lens.allocate((n_docs + 1) * sizeof(float)))) return rc;
    if (n_docs)
        SA_CUDA(cudaMemcpyAsync(ix->d_doc_lens.p, doc_lens, n_docs * sizeof(float), cudaMemcpyHostToDevice, ix->stream));
    if ((rc = ix->d_df.allocate((size_t)(n_terms + 1) * sizeof(u32)))) return rc;
    SA_CUDA(cudaMemsetAsync(ix->d_df.p, 0, (size_t)(n_terms + 1) * sizeof(u32), ix->stream));
    DevBuf d_past;
    u32 past_max_posn = 0;
    if ((rc = d_past.allocate(sizeof(u32)))) return rc;
    SA_CUDA(cudaMemsetAsync(d_past.p, 0, sizeof(u32), ix->stream));
    ix->device_bytes = (n_words + 1) * sizeof(u64) + (n_docs + 1) * sizeof(float) + (size_t)(n_terms + 1) * 4;

    ix->doc_lens_nonneg = true;
    for (u64 i = 0; i < n_docs; i++)
        if (!(doc_lens[i] >= 0.0f)) { ix->doc_lens_nonneg = false; break; }

    // df per term on the device
    if (n_words && n_terms) {
        std::vector<u32> order;
        order.reserve(n_terms);
        for (u32 t = 0; t < n_terms; t++) if (term_lengths[t]) order.push_back(t);
        std::sort(order.begin(), order.end(), [&](u32 a, u32 b) { return term_offsets[a] < term_offsets[b]; });
        // slices must be disjoint for the head test to be per-term; also cover gaps
        std::vector<u64> off_sorted;
        std::vector<u32> term_of_slot;
        u64 covered = 0;
        bool full_cover = true;
        for (u32 t : order) {
            if (term_offsets[t] != covered) { full_cover = false; break; }
            off_sorted.push_back(term_offsets[t]);
            term_of_slot.push_back(t);
            covered += term_lengths[t];
        }
        SA_CHECK(full_cover && covered == n_words, "term slices must tile `words` exactly (ArrayDict.compact layout)");
        u32 n_slots = (u32)off_sorted.size();
        // tile directories for long lists (short ones are searched: they stay cache resident)
        const u32 n_tiles = sa_n_tiles(n_docs);
        const u64 dir_min_words = std::max<u64>(1024, n_tiles / 2);
        std::vector<u64> slot_len(n_slots), slot_dir(n_slots, SA_NO_DIR);
        u64 dir_words = 0;
        for (u32 sI = 0; sI < n_slots; sI++) {
            u32 t = term_of_slot[sI];
            slot_len[sI] = term_lengths[t];
            if (term_lengths[t] >= dir_min_words && term_lengths[t] < 0xFFFFFFFFull) {
                slot_dir[sI] = dir_words;
                ix->h_dir_off[t] = dir_words;
                dir_words += (u64)n_tiles + 1;
            }
        }
        DevBuf d_off, d_slot, d_slot_len, d_slot_dir;
        if ((rc = upload_table(d_off, off_sorted)) || (rc = upload_table(d_slot, term_of_slot))) return rc;
        unsigned blocks = (unsigned)((n_words + 255) / 256);
        df_kernel<<<blocks, 256, 0, ix->stream>>>(ix->d_words.as<u64>(), n_words, d_off.as<u64>(), d_slot.as<u32>(), n_slots,
                                                  ix->d_df.as<u32>(), d_past.as<u32>());
        SA_CUDA(cudaGetLastError());
        ix->stats.total_launches++;
        SA_CUDA(cudaMemcpyAsync(ix->h_df.data(), ix->d_df.p, n_terms * sizeof(u32), cudaMemcpyDeviceToHost, ix->stream));
        SA_CUDA(cudaMemcpyAsync(&past_max_posn, d_past.p, sizeof(u32), cudaMemcpyDeviceToHost, ix->stream));
        if (dir_words) {
            if ((rc = ix->d_tile_dir.allocate(dir_words * sizeof(u32)))) return rc;
            ix->device_bytes += dir_words * sizeof(u32);
            if ((rc = upload_table(d_slot_len, slot_len)) || (rc = upload_table(d_slot_dir, slot_dir))) return rc;
            tile_dir_kernel<<<blocks, 256, 0, ix->stream>>>(ix->d_words.as<u64>(), n_words, d_off.as<u64>(),
                                                           d_slot_len.as<u64>(), d_slot_dir.as<u64>(), n_slots,
                                                           ix->d_tile_dir.as<u32>(), doc_base, n_tiles);
            SA_CUDA(cudaGetLastError());
            ix->stats.total_launches++;
        }
        SA_CUDA(cudaStreamSynchronize(ix->stream));         // h_df is final from here on
        // a block past MAX_POSN's would carry a doc's tf past the 19 bits of its record (and of the words path's count)
        SA_CHECK(!(refuse_past_max_posn && past_max_posn),
                 "posting words hold positions past MAX_POSN = %u (block > %u): the index counts at most %u positions per doc",
                 SA_MAX_POSN, SA_MAX_BLOCK, SA_MAX_POSN + 1);
        // tf table for the terms that have a directory (the long lists: that is where the scan's time goes)
        static const bool no_tf_table = getenv("SA_NO_TF_TABLE") && atoi(getenv("SA_NO_TF_TABLE")) != 0;
        ix->h_rec_off.assign(n_terms, SA_NO_DIR);
        if (dir_words && !no_tf_table) {
            std::vector<u64> slot_rec(n_slots, SA_NO_DIR), slot_head_base(n_slots, 0);
            std::vector<u32> slot_df(n_slots, 0);
            u64 total_recs = 0, heads = 0;
            for (u32 sI = 0; sI < n_slots; sI++) {
                const u32 t = term_of_slot[sI];
                slot_head_base[sI] = heads;
                slot_df[sI] = ix->h_df[t];
                heads += ix->h_df[t];
                if (slot_dir[sI] != SA_NO_DIR) {
                    slot_rec[sI] = total_recs;
                    ix->h_rec_off[t] = total_recs;
                    total_recs += ((u64)ix->h_df[t] + 3) / 4 * 4;          // 16-byte aligned record runs
                }
            }
            const u32 n_rblocks = (u32)((n_words + REC_BLOCK - 1) / REC_BLOCK);
            DevBuf d_bbase, d_slot_rec, d_slot_hb, d_slot_df;
            if ((rc = ix->d_recs.allocate((total_recs + 8) * sizeof(u32)))) return rc;
            SA_CUDA(cudaMemsetAsync(ix->d_recs.p, 0, (total_recs + 8) * sizeof(u32), ix->stream));
            if ((rc = ix->d_rec_dir.allocate(dir_words * sizeof(u32)))) return rc;
            ix->device_bytes += (total_recs + 8) * sizeof(u32) + dir_words * sizeof(u32);
            if ((rc = d_bbase.allocate((size_t)(n_rblocks + 1) * sizeof(u64))) || (rc = upload_table(d_slot_rec, slot_rec)) ||
                (rc = upload_table(d_slot_hb, slot_head_base)) || (rc = upload_table(d_slot_df, slot_df)))
                return rc;
            rec_count_kernel<<<n_rblocks, 256, 0, ix->stream>>>(ix->d_words.as<u64>(), n_words, d_off.as<u64>(), n_slots,
                                                                d_bbase.as<u64>());
            cta_scan_kernel<1024><<<1, 1024, 0, ix->stream>>>(d_bbase.as<u64>(), n_rblocks, d_bbase.as<u64>() + n_rblocks);
            rec_write_kernel<<<n_rblocks, 256, 0, ix->stream>>>(
                ix->d_words.as<u64>(), n_words, d_off.as<u64>(), d_slot_len.as<u64>(), d_slot_dir.as<u64>(), d_slot_rec.as<u64>(),
                d_slot_hb.as<u64>(), d_slot_df.as<u32>(), n_slots, d_bbase.as<u64>(), ix->d_recs.as<u32>(), ix->d_rec_dir.as<u32>(),
                doc_base, n_tiles);
            SA_CUDA(cudaGetLastError());
            ix->stats.total_launches += 3;
            SA_CUDA(cudaStreamSynchronize(ix->stream));
        }
    } else {
        SA_CUDA(cudaStreamSynchronize(ix->stream));
    }
    *index_out = ix.release();
    return SA_OK;
}

// Order matters: the stream drains before anything it uses is freed; the members (every device buffer, the batch
// and view states, the pinned staging) free themselves after this body, with the device still current.
sa_index::~sa_index() {
    cudaSetDevice(device);
    if (stream) cudaStreamSynchronize(stream);
    sa_comm_destroy(this);
    for (auto &t : pending_timers) { cudaEventDestroy(t.e0); cudaEventDestroy(t.e1); }
    for (auto e : free_events) cudaEventDestroy(e);
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
    if (stream) cudaStreamDestroy(stream);
}

extern "C" int sa_index_destroy(sa_index *ix) {
    delete ix;
    return SA_OK;
}

extern "C" int sa_index_info(const sa_index *ix, uint64_t *n_docs, uint64_t *n_words,
                             uint32_t *n_terms, uint64_t *device_bytes) {
    SA_CHECK(ix, "index is NULL");
    if (n_docs) *n_docs = ix->n_docs;
    if (n_words) *n_words = ix->n_words;
    if (n_terms) *n_terms = ix->n_terms;
    if (device_bytes) *device_bytes = ix->device_bytes;
    return SA_OK;
}

extern "C" int sa_index_upload_mode(const sa_index *ix, int *mode_out) {
    SA_CHECK(ix && mode_out, "NULL argument");
    *mode_out = ix->upload_mode;
    return SA_OK;
}

extern "C" int sa_index_dense_compressible(const sa_index *ix, int *compressible_out) {
    SA_CHECK(ix && compressible_out, "NULL argument");
    *compressible_out = CompressibleSpace::compressible(ix->comp_rows.p) ? 1 : 0;
    return SA_OK;
}

extern "C" int sa_docfreq(sa_index *ix, uint32_t term_id, uint64_t *df_out) {
    SA_CHECK(ix && df_out, "NULL argument");
    if (term_id == SA_NO_TERM) { *df_out = 0; return SA_OK; }
    int rc = sa_check_term_ids(ix, &term_id, 1);
    if (rc) return rc;
    *df_out = ix->h_df[term_id];
    return SA_OK;
}

extern "C" int sa_stats_reset(sa_index *ix) {
    SA_CHECK(ix, "index is NULL");
    std::lock_guard<std::mutex> g(ix->mu);
    sa_resolve_timers(ix);
    memset(&ix->stats, 0, sizeof(ix->stats));
    return SA_OK;
}

extern "C" int sa_stats_get(sa_index *ix, sa_stats *out) {
    SA_CHECK(ix && out, "NULL argument");
    std::lock_guard<std::mutex> g(ix->mu);
    int rc = sa_resolve_timers(ix);
    if (rc) return rc;
    *out = ix->stats;
    return SA_OK;
}

extern "C" int sa_set_profiling(sa_index *ix, int enabled) {
    SA_CHECK(ix, "index is NULL");
    std::lock_guard<std::mutex> g(ix->mu);
    ix->profiling = enabled != 0;
    return SA_OK;
}

// ----------------------------------------------------------------- term path
static int single_term(sa_index *ix, uint32_t term_id, int mode, const Bm25Params &p,
                       u64 min_payload, u64 max_payload, float *out_host) {
    SA_CHECK(ix && out_host, "NULL argument");
    int rc = sa_check_term_ids(ix, &term_id, 1);
    if (rc) return rc;
    std::lock_guard<std::mutex> g(ix->mu);
    SA_CUDA(cudaSetDevice(ix->device));
    if (ix->n_docs == 0) return SA_OK;
    const bool rows = ix->rows_active;
    SA_CHECK(!(rows && mode == TERM_MODE_SCORE), "score on a sliced array: call termfreqs + bm25 (the Python layer does)");
    if ((rc = ix->dense.reserve(sa_padded_docs(ix->n_docs) * sizeof(float)))) return rc;
    if ((rc = ix->queries.reserve(sizeof(TermQuery)))) return rc;
    TermQuery tq = make_term_query(ix, term_id, p.idf);
    TopkCtx none;
    memset(&none, 0, sizeof(none));
    TermBatchArgs a = make_term_args(ix, ix->queries.as<TermQuery>(), p, none);
    a.min_payload = min_payload;
    a.max_payload = max_payload;
    a.filter = !(min_payload == 0 && max_payload == SA_ALL_BITS);
    a.mode = mode;
    if (rows && term_id != SA_NO_TERM) {
        // sliced array: run on the materialised FilteredPosns list (rows and block filter applied)
        std::vector<u64> offs, lens;
        if ((rc = sa_filter_terms(ix, &term_id, 1, true, min_payload, max_payload, a.filter, offs, lens))) return rc;
        a.words = ix->filt.as<u64>();
        tq.word_off = offs[0];
        tq.n_words = lens[0];
        tq.dir_off = SA_NO_DIR;
        tq.rec_off = SA_NO_DIR;
        a.filter = 0;
    }
    SA_CUDA(cudaMemcpyAsync(ix->queries.p, &tq, sizeof(tq), cudaMemcpyHostToDevice, ix->stream));
    if ((rc = launch_term_batch(ix, a, 1))) return rc;
    return sa_copy_out_dense(ix, out_host);
}

extern "C" int sa_termfreqs(sa_index *ix, uint32_t term_id, uint64_t min_payload, uint64_t max_payload,
                            float *out_host) {
    SA_CHECK(ix, "index is NULL");
    Bm25Params p = make_bm25(0, 1, 1, 0, ix->doc_lens_nonneg);
    return single_term(ix, term_id, TERM_MODE_TF, p, min_payload, max_payload, out_host);
}

extern "C" int sa_score_term(sa_index *ix, uint32_t term_id, float idf, float avg_doc_len,
                             float k1, float b, uint64_t min_payload, uint64_t max_payload,
                             float *out_host) {
    SA_CHECK(ix, "index is NULL");
    if (avg_doc_len == 0.0f) {   // similarity.py:31-32: zeros_like(term_freqs)
        SA_CHECK(out_host, "out is NULL");
        memset(out_host, 0, ix->n_docs * sizeof(float));
        return SA_OK;
    }
    Bm25Params p = make_bm25(idf, avg_doc_len, k1, b, ix->doc_lens_nonneg);
    return single_term(ix, term_id, TERM_MODE_SCORE, p, min_payload, max_payload, out_host);
}

// ------------------------------------------------ batched, HBM-resident top-k
// A prepared batch: query descriptors live in HBM; sa_batch_execute only enqueues kernels.
// Queries are processed in the chunks of sa_plan_rows (bounded dense-vector memory).  Inside a chunk the term queries
// take dense rows [0, nT) (one fused launch) and the phrase queries rows [nT, nT + nP) (phrase
// kernel + tile scan); one select launch covers the chunk and writes each result at its
// original query index.
struct BatchChunk {
    u32 row0 = 0;          // first row (in the permuted "row space") of this chunk
    u32 n_term = 0, n_phrase = 0;
    u32 term0 = 0, phrase0 = 0;     // offsets into the batch-wide TermQuery / PhraseQuery (slop > 0: SpanQuery) arrays
    Bm25Params params;
    DocChunks phrase_chunks{};      // doc ranges of every phrase query
    u64 arena_words = 64;
    // phrase queries by regime (indices relative to phrase0, stored at B.d_sel + sel0: search first, then conjunction)
    u32 sel0 = 0, n_search = 0, n_conj = 0;
    SpanPlan span;                  // slop > 0: the chunk's multi-term queries as span queries
};

struct BatchState {
    u32 nq = 0, k = 0, slots = 0, chunk = 0, slop = 0;
    float avg_doc_len = 0, k1 = 0, b = 0;
    bool ready = false;
    std::vector<TermQuery> tqs;               // all term queries, chunk by chunk
    std::vector<PhraseQuery> pqs;             // all phrase queries, chunk by chunk
    std::vector<u32> row_query;               // row -> original query index
    std::vector<u32> term_query, phrase_query;  // index in tqs / pqs -> original query index
    std::vector<u32> phrase_missing;          // 1 = a term is unknown: result stays empty
    std::vector<BatchChunk> chunks;
    u64 comp_stride = 0;                      // term rows in ix->comp_rows, floats from one to the next; 0: in ix->dense
    DevBuf d_sq, d_scounts;                   // slop > 0: every chunk's span descriptors, concatenated, and counts
    DevBuf d_tq, d_pq, d_row_query;
    DevBuf d_meta;                            // u32 overflow[nq] (row space)
    DevBuf d_pstats;                          // PhraseStats[#phrase queries]
    std::vector<u32> sel;                     // per chunk: search-regime then conjunction-regime phrase indices
    DevBuf d_sel;
    DevBuf d_missing;                         // phrase_missing on the device (batch_summary_kernel)
};

int sa_batch_upload_locked(sa_index *ix, const uint32_t *terms, const uint32_t *term_starts,
                           const float *idf, uint32_t n_queries, uint32_t slop,
                           float avg_doc_len, float k1, float b, uint32_t k) {
    SA_CHECK(ix && (n_queries == 0 || (terms && term_starts && idf)), "NULL argument");
    SA_CHECK(k >= 1 && k <= SA_TOPK_DEEP_MAX, "k must be in [1, %d]", SA_TOPK_DEEP_MAX);
    SA_CUDA(cudaSetDevice(ix->device));
    if (!ix->batch) ix->batch.reset(new BatchState());
    BatchState &B = *ix->batch;
    B.ready = false;
    B.nq = n_queries;
    B.k = k;
    B.slots = sa_topk_slots(k);
    B.avg_doc_len = avg_doc_len;
    B.k1 = k1;
    B.b = b;
    B.slop = slop;
    B.tqs.clear(); B.pqs.clear(); B.row_query.clear(); B.term_query.clear(); B.phrase_query.clear();
    B.phrase_missing.clear(); B.chunks.clear(); B.sel.clear();
    int rc;
    if ((rc = ix->topk_out.reserve(std::max<size_t>(((size_t)n_queries * k + SA_BATCH_TAIL) * sizeof(u64), 256)))) return rc;
    if (n_queries == 0) { B.ready = true; return SA_OK; }
    for (u32 q = 0; q < n_queries; q++) {
        const u32 nt = term_starts[q + 1] - term_starts[q];
        SA_CHECK(nt >= 1 && nt <= SA_MAX_PHRASE_TERMS, "query %u: bad number of terms", q);
        if ((rc = sa_check_term_ids(ix, terms + term_starts[q], nt))) return rc;
    }
    RowPlan plan = sa_plan_rows(ix->n_docs, term_starts, n_queries);
    const u64 stride = sa_padded_docs(std::max<u64>(ix->n_docs, 1));
    B.chunk = plan.chunk;
    B.row_query = std::move(plan.row_query);
    // A term row is mostly zero 128-byte lines (72 % at df/N = 1e-2), which compressible memory keeps off DRAM when
    // the CTAs in flight write neighbouring tiles of few rows: the term launch walks the rows in query groups of
    // SA_COMP_ROW_GROUP (sa_term.cu, DESIGN §3.1).  So where compressible memory is available the chunks' term rows
    // live in ix->comp_rows, the phrase rows in ix->dense.  A row that spans many granules starts on one of its own:
    // written a group's time apart, neighbouring rows sharing one would be slow to compress.  The padding is kept to at
    // most 1/8 of the row (always so for rows of >= 8 granules, 16 MiB); other rows stay packed -- a group's few short
    // rows are in flight together anyway -- so a chunk's rows stay within sa_plan_rows' budget plus that 1/8.
    u32 max_term = 0;
    for (const RowChunk &R : plan.chunks) max_term = std::max(max_term, R.n_term);
    const size_t gran = max_term ? CompressibleSpace::granularity() : 0;
    B.comp_stride = 0;
    if (gran) {
        const size_t packed = stride * sizeof(float), padded = (packed + gran - 1) / gran * gran;
        const size_t row_bytes = padded - packed <= packed / 8 ? padded : packed;
        if (ix->comp_rows.reserve((size_t)max_term * row_bytes) == SA_OK && CompressibleSpace::compressible(ix->comp_rows.p)) {
            B.comp_stride = row_bytes / sizeof(float);
        } else {
            // plain rows in ix->dense instead; a failed fallback cudaMalloc must not fail the batch's next launch check
            ix->comp_rows.reset();
            (void)cudaGetLastError();
        }
    }
    u32 max_dense_rows = 1;
    u64 max_arena = 64;
    size_t max_span_scratch = 0;
    u32 n_span = 0;
    for (const RowChunk &R : plan.chunks) {
        BatchChunk C;
        C.row0 = R.row0;
        C.n_term = R.n_term;
        C.n_phrase = R.n_phrase;
        C.term0 = (u32)B.tqs.size();
        C.phrase0 = slop > 0 ? n_span : (u32)B.pqs.size();
        C.params = make_bm25(1.0f, avg_doc_len, k1, b, ix->doc_lens_nonneg);
        max_dense_rows = std::max(max_dense_rows, (B.comp_stride ? 0 : R.n_term) + R.n_phrase);
        for (u32 r = R.row0; r < R.row0 + R.n_term + R.n_phrase; r++) {
            const u32 q = B.row_query[r];
            const u32 nt = term_starts[q + 1] - term_starts[q];
            const u32 *tids = terms + term_starts[q];
            u64 offs[SA_MAX_PHRASE_TERMS], lens[SA_MAX_PHRASE_TERMS], dirs[SA_MAX_PHRASE_TERMS];
            bool missing, literal;
            if ((rc = sa_resolve_terms(ix, tids, nt, offs, lens, dirs, &missing, &literal))) return rc;
            if (!make_bm25(idf[q], avg_doc_len, k1, b, ix->doc_lens_nonneg).sparse_ok) C.params.sparse_ok = 0;
            if (nt == 1) {
                B.tqs.push_back(make_term_query(ix, tids[0], idf[q]));
                B.term_query.push_back(q);
            } else if (slop > 0) {
                // phrase with slop: span search (spans.py:171-187) on the index's own lists
                sa_span_plan_add(C.span, offs, lens, dirs, nt, slop, idf[q], literal, missing ? 0 : ix->n_docs);
                B.phrase_query.push_back(q);
            } else {
                PhraseQuery pq = make_phrase_query(tids, nt, offs, lens, dirs, idf[q], missing);
                pq.use_conj = !missing && sa_phrase_use_conjunction(pq, ix->n_docs);
                B.pqs.push_back(pq);
                B.phrase_query.push_back(q);
                B.phrase_missing.push_back(missing);
            }
        }
        if (slop > 0) {
            n_span += C.n_phrase;
            max_span_scratch = std::max(max_span_scratch, sa_span_scratch_bytes(C.span));
            B.chunks.push_back(std::move(C));
            continue;
        }
        if (C.n_phrase) {
            C.sel0 = (u32)B.sel.size();
            for (u32 i = 0; i < C.n_phrase; i++) if (!B.pqs[C.phrase0 + i].use_conj) B.sel.push_back(i);
            C.n_search = (u32)B.sel.size() - C.sel0;
            for (u32 i = 0; i < C.n_phrase; i++) if (B.pqs[C.phrase0 + i].use_conj) B.sel.push_back(i);
            C.n_conj = C.n_phrase - C.n_search;
            C.phrase_chunks = phrase_doc_chunks(ix, C.n_search, 16);
            for (u32 i = 0; i < C.n_phrase; i++)                     // only the search regime bump-allocates
                if (!B.pqs[C.phrase0 + i].use_conj)
                    C.arena_words += sa_phrase_arena_words(B.pqs[C.phrase0 + i], C.phrase_chunks.n_chunks);
            max_arena = std::max(max_arena, C.arena_words);
        }
        B.chunks.push_back(std::move(C));
    }
    SA_CHECK(B.chunks.empty() || B.chunks[0].params.sparse_ok || (B.pqs.empty() && n_span == 0),
             "phrase queries in a batch need ordinary BM25 parameters (k1 > 0, 0 <= b < 1, finite idf)");
    if ((rc = ix->dense.reserve((size_t)max_dense_rows * stride * sizeof(float)))) return rc;
    if ((rc = ix->cand.reserve(cand_bytes(sa_n_tiles(ix->n_docs), B.chunk, B.slots)))) return rc;
    if ((rc = B.d_tq.reserve(std::max<size_t>(B.tqs.size() * sizeof(TermQuery), 64)))) return rc;
    if ((rc = B.d_pq.reserve(std::max<size_t>(B.pqs.size() * sizeof(PhraseQuery), 64)))) return rc;
    if ((rc = B.d_row_query.reserve((size_t)n_queries * sizeof(u32)))) return rc;
    if ((rc = B.d_meta.reserve((size_t)n_queries * sizeof(u32)))) return rc;
    if ((rc = B.d_pstats.reserve(std::max<size_t>(B.pqs.size() * sizeof(PhraseStats), 64)))) return rc;
    if ((rc = B.d_sel.reserve(std::max<size_t>(B.sel.size() * sizeof(u32), 64)))) return rc;
    if ((rc = B.d_missing.reserve(std::max<size_t>(B.phrase_missing.size() * sizeof(u32), 64)))) return rc;
    if (!B.pqs.empty() && (rc = ix->phrase_scratch.reserve(max_arena * sizeof(u64) + 64))) return rc;
    if (n_span) {
        if ((rc = ix->phrase_scratch.reserve(max_span_scratch))) return rc;
        if ((rc = B.d_sq.reserve((size_t)n_span * sizeof(SpanQuery)))) return rc;
        if ((rc = B.d_scounts.reserve((size_t)n_span * sizeof(SpanCounts)))) return rc;
        for (const BatchChunk &C : B.chunks) {
            if (C.span.qs.empty()) continue;
            SA_CUDA(cudaMemcpyAsync(B.d_sq.as<SpanQuery>() + C.phrase0, C.span.qs.data(), C.span.qs.size() * sizeof(SpanQuery),
                                    cudaMemcpyHostToDevice, ix->stream));
        }
        SA_CUDA(cudaStreamSynchronize(ix->stream));      // the plans' host vectors may be reallocated later
    }
    if (!B.tqs.empty())
        SA_CUDA(cudaMemcpyAsync(B.d_tq.p, B.tqs.data(), B.tqs.size() * sizeof(TermQuery), cudaMemcpyHostToDevice, ix->stream));
    if (!B.pqs.empty()) {
        SA_CUDA(cudaMemcpyAsync(B.d_pq.p, B.pqs.data(), B.pqs.size() * sizeof(PhraseQuery), cudaMemcpyHostToDevice, ix->stream));
        SA_CUDA(cudaMemcpyAsync(B.d_sel.p, B.sel.data(), B.sel.size() * sizeof(u32), cudaMemcpyHostToDevice, ix->stream));
        SA_CUDA(cudaMemcpyAsync(B.d_missing.p, B.phrase_missing.data(), B.phrase_missing.size() * sizeof(u32),
                                cudaMemcpyHostToDevice, ix->stream));
    }
    SA_CUDA(cudaMemcpyAsync(B.d_row_query.p, B.row_query.data(), (size_t)n_queries * sizeof(u32), cudaMemcpyHostToDevice, ix->stream));
    B.ready = true;
    return SA_OK;
}

// Last kernel of a batch: how many queries need the exact re-run, and the phrase roofline counters.  The same-term
// speculation of every phrase query is verified here exactly as sa_phrase_guess_ok does on the host.
__global__ void __launch_bounds__(256)
batch_summary_kernel(const u32 *__restrict__ ovf, u32 nq, const PhraseQuery *__restrict__ pqs,
                     const PhraseStats *__restrict__ st, const u32 *__restrict__ missing, u32 n_phrase,
                     u64 *__restrict__ tail) {
    __shared__ unsigned long long s_acc[3];
    if (threadIdx.x < 3) s_acc[threadIdx.x] = 0;
    __syncthreads();
    unsigned long long redo = 0, cont = 0, match = 0;
    for (u32 i = threadIdx.x; i < nq; i += blockDim.x) redo += ovf[i] ? 1 : 0;
    for (u32 i = threadIdx.x; i < n_phrase; i += blockDim.x) {
        const PhraseQuery &pq = pqs[i];
        const PhraseStats &s = st[i];
        cont += s.n_cont;
        match += s.n_match;
        bool bad = s.overflow != 0;
        if (!bad && !missing[i]) {
            const u32 n = pq.n_terms;
            // every step the plan runs (sa_phrase.cu step_order): LR 1..n-1, RL 0..n-2, middle-out 1..split-1 and split..n-2
            u32 s0 = 1, s1 = n;
            if (pq.mode == SA_PHRASE_MODE_RL) { s0 = 0; s1 = n - 1; }
            else if (pq.mode == SA_PHRASE_MODE_MID) { s0 = 1; s1 = n - 1; }
            for (u32 step = s0; step < s1 && !bad; step++) {
                const bool actual = s.n_inner[step] > 0 && s.n_diff[step] == 0;
                const bool guess = (pq.same_guess >> step) & 1u;
                if (actual != guess) bad = true;
            }
        }
        // a wrong guess also sets the query's overflow flag?  No: the host re-derives which queries to redo; here
        // only the COUNT matters (non-zero -> the host takes the slow path)
        if (bad) redo++;
    }
    if (redo) atomicAdd(&s_acc[0], redo);
    if (cont) atomicAdd(&s_acc[1], cont);
    if (match) atomicAdd(&s_acc[2], match);
    __syncthreads();
    if (threadIdx.x < 3) tail[threadIdx.x] = s_acc[threadIdx.x];
    if (threadIdx.x == 3) tail[3] = 0;
}

int sa_batch_execute_locked(sa_index *ix) {
    SA_CHECK(ix && ix->batch && ix->batch->ready, "no batch uploaded (sa_batch_upload)");
    BatchState &B = *ix->batch;
    SA_CUDA(cudaSetDevice(ix->device));
    u64 *d_keys = ix->topk_out.as<u64>();
    if (B.nq == 0) {
        SA_CUDA(cudaMemsetAsync(d_keys, 0, SA_BATCH_TAIL * sizeof(u64), ix->stream));
        return SA_OK;
    }
    if (ix->n_docs == 0 || B.avg_doc_len == 0.0f) {
        SA_CUDA(cudaMemsetAsync(d_keys, 0, ((size_t)B.nq * B.k + SA_BATCH_TAIL) * sizeof(u64), ix->stream));
        return SA_OK;
    }
    const u64 stride = sa_padded_docs(ix->n_docs);
    const char *e = getenv("SA_COMP_ROW_GROUP");
    const u32 comp_group = e ? (u32)atol(e) : SA_COMP_ROW_GROUP;
    u32 *d_ovf = B.d_meta.as<u32>();
    SA_CUDA(cudaMemsetAsync(d_ovf, 0, (size_t)B.nq * sizeof(u32), ix->stream));
    if (!B.pqs.empty())
        SA_CUDA(cudaMemsetAsync(B.d_pstats.p, 0, B.pqs.size() * sizeof(PhraseStats), ix->stream));
    int rc;
    for (const BatchChunk &C : B.chunks) {
        const u32 Q = C.n_term + C.n_phrase;
        TopkCtx t = make_topk_ctx(ix->cand.p, sa_n_tiles(ix->n_docs), Q, B.slots, B.k, d_ovf + C.row0);
        const u32 n_plain = B.comp_stride ? 0 : C.n_term;   // term rows in ix->dense; the phrase rows follow them
        if (C.n_term) {
            TermBatchArgs a = make_term_args(ix, B.d_tq.as<TermQuery>() + C.term0, C.params, t);
            if (B.comp_stride) {
                a.out = ix->comp_rows.as<float>();
                a.out_stride = B.comp_stride;
            }
            if ((rc = launch_term_batch(ix, a, C.n_term, B.comp_stride ? comp_group : 0))) return rc;
        }
        if (B.slop > 0) {
            if (C.n_phrase) {
                // span matches become records; one tile pass writes the rows (zeros + BM25) and collects top-k
                float *rows = ix->dense.as<float>() + (u64)n_plain * stride;
                if ((rc = sa_ensure_norm(ix, B.k1, B.b, B.avg_doc_len))) return rc;
                if ((rc = sa_span_enqueue(ix, ix->d_words.as<u64>(), C.span, B.d_sq.as<SpanQuery>() + C.phrase0,
                                          B.d_scounts.as<SpanCounts>() + C.phrase0, ix->phrase_scratch.p, rows, stride,
                                          &t, C.n_term))) return rc;
            }
        } else if (C.n_phrase) {
            float *rows = ix->dense.as<float>() + (u64)n_plain * stride;
            unsigned long long *d_used = (unsigned long long *)ix->phrase_scratch.p;
            SA_CUDA(cudaMemsetAsync(d_used, 0, 64, ix->stream));
            // the phrase kernel materialises its dense rows (zeros + matches) and their top-k candidates
            PhraseSplit sp;
            sp.d_search = B.d_sel.as<u32>() + C.sel0;
            sp.n_search = C.n_search;
            sp.d_conj = sp.d_search + C.n_search;
            sp.n_conj = C.n_conj;
            if ((rc = sa_phrase_enqueue(ix, B.d_pq.as<PhraseQuery>() + C.phrase0, B.d_pstats.as<PhraseStats>() + C.phrase0,
                                        C.n_phrase, rows, stride, C.phrase_chunks, (u64 *)ix->phrase_scratch.p + 8,
                                        d_used, C.arena_words, 1, C.params, &t, C.n_term, &sp))) return rc;
        }
        if ((rc = launch_topk_select(ix, t, Q, ix->doc_base, d_keys, B.d_row_query.as<u32>() + C.row0))) return rc;
    }
    const u32 n_phr = B.slop > 0 ? 0u : (u32)B.pqs.size();
    batch_summary_kernel<<<1, 256, 0, ix->stream>>>(d_ovf, B.nq, B.d_pq.as<PhraseQuery>(), B.d_pstats.as<PhraseStats>(),
                                                   B.d_missing.as<u32>(), n_phr, d_keys + (size_t)B.nq * B.k);
    SA_CUDA(cudaGetLastError());
    ix->stats.total_launches++;
    return SA_OK;
}

// Re-run one query exactly (synchronously): a tile overflowed its candidate slots, or a phrase's
// same-term speculation was wrong.  Uses a slot per doc of the tile -- cannot overflow.  A phrase or span query
// writes its raw counts into ix->dense row 0, and the BM25 tile pass (launch_sim_tiles) scores and collects them:
// bm25_one performs the rounded operations of the batch kernels' BM25 in the same order, and a zero count scores +0
// (a batch with phrase queries has ordinary parameters, sa_batch_upload_locked), so the scores are the batch's bits.
static int redo_query(sa_index *ix, BatchState &B, bool is_phrase, u32 idx, u32 q, const SpanQuery *sq = nullptr) {
    int rc;
    const u32 n_tiles = sa_n_tiles(ix->n_docs);
    if ((rc = ix->cand.reserve(cand_bytes(n_tiles, 1, SA_TILE_DOCS)))) return rc;
    SA_CUDA(cudaMemsetAsync(B.d_meta.p, 0, sizeof(u32), ix->stream));
    TopkCtx t = make_topk_ctx(ix->cand.p, n_tiles, 1, SA_TILE_DOCS, B.k, B.d_meta.as<u32>());
    if (!is_phrase) {
        Bm25Params p = make_bm25(B.tqs[idx].idf, B.avg_doc_len, B.k1, B.b, ix->doc_lens_nonneg);
        TermBatchArgs a = make_term_args(ix, B.d_tq.as<TermQuery>() + idx, p, t);
        if ((rc = launch_term_batch(ix, a, 1))) return rc;
    } else {
        const Bm25Params p = make_bm25(sq ? sq->idf : B.pqs[idx].idf, B.avg_doc_len, B.k1, B.b, ix->doc_lens_nonneg);
        if (sq) {
            if ((rc = sa_span_run(ix, ix->d_words.as<u64>(), sq->off, sq->len, sq->dir_off, sq->n_terms, sq->slop,
                                  sq->literal != 0))) return rc;
        } else {
            std::vector<PhraseQuery> one(1, B.pqs[idx]);
            PhraseDump nodump;
            memset(&nodump, 0, sizeof(nodump));
            // loops until the guess holds
            if ((rc = sa_phrase_run_sync(ix, one, ix->d_words.as<u64>(), 0, p, nodump, false))) return rc;
            B.pqs[idx] = one[0];
        }
        const double idf = p.idf;
        if ((rc = ix->misc.reserve(sizeof(double)))) return rc;
        SA_CUDA(cudaMemcpyAsync(ix->misc.p, &idf, sizeof(double), cudaMemcpyHostToDevice, ix->stream));
        if ((rc = launch_sim_tiles(ix, SA_SIM_BM25, ix->dense.as<float>(), nullptr, ix->d_doc_lens.as<float>(), ix->n_docs, p,
                                   SimParams{}, ix->misc.as<double>(), 1, 0, t, nullptr))) return rc;
    }
    SA_CUDA(cudaMemcpyAsync(B.d_row_query.p, &q, sizeof(u32), cudaMemcpyHostToDevice, ix->stream));
    if ((rc = launch_topk_select(ix, t, 1, ix->doc_base, ix->topk_out.as<u64>(), B.d_row_query.as<u32>()))) return rc;
    SA_CUDA(cudaStreamSynchronize(ix->stream));
    return SA_OK;
}

// After execute: repair (synchronously) the queries that need it.
int sa_batch_fix_overflow_locked(sa_index *ix, u32 *n_redone) {
    BatchState &B = *ix->batch;
    if (n_redone) *n_redone = 0;
    if (B.nq == 0 || ix->n_docs == 0 || B.avg_doc_len == 0.0f) return SA_OK;
    int rc;
    const size_t ovf_bytes = (size_t)B.nq * sizeof(u32), st_bytes = B.pqs.size() * sizeof(PhraseStats);
    if ((rc = ix->h_pinned.reserve(std::max<size_t>(ovf_bytes + st_bytes, 4096)))) return rc;
    SA_CUDA(cudaMemcpyAsync(ix->h_pinned.p, B.d_meta.p, ovf_bytes, cudaMemcpyDeviceToHost, ix->stream));
    if (st_bytes)
        SA_CUDA(cudaMemcpyAsync(ix->h_pinned.as<char>() + ovf_bytes, B.d_pstats.p, st_bytes, cudaMemcpyDeviceToHost, ix->stream));
    SA_CUDA(cudaStreamSynchronize(ix->stream));
    std::vector<u32> ovf(ix->h_pinned.as<const u32>(), ix->h_pinned.as<const u32>() + B.nq);       // row space
    std::vector<PhraseStats> st(B.pqs.size());
    if (st_bytes) memcpy(st.data(), ix->h_pinned.as<char>() + ovf_bytes, st_bytes);

    struct Redo { bool phrase; u32 idx, q; const SpanQuery *sq; };
    std::vector<Redo> redo;
    for (const BatchChunk &C : B.chunks) {
        for (u32 i = 0; i < C.n_term; i++)
            if (ovf[C.row0 + i]) redo.push_back({false, C.term0 + i, B.term_query[C.term0 + i], nullptr});
        if (B.slop > 0) {
            for (u32 i = 0; i < C.n_phrase; i++)
                if (ovf[C.row0 + C.n_term + i])
                    redo.push_back({true, C.phrase0 + i, B.phrase_query[C.phrase0 + i], &C.span.qs[i]});
            continue;
        }
        for (u32 i = 0; i < C.n_phrase; i++) {
            const u32 pi = C.phrase0 + i;
            SA_CHECK(st[pi].overflow != 1, "phrase scratch arena exhausted (internal sizing error)");
            PhraseQuery trial = B.pqs[pi];
            bool ok = st[pi].overflow == 0 && (B.phrase_missing[pi] || sa_phrase_guess_ok(trial, st[pi]));
            if (!ok || ovf[C.row0 + C.n_term + i]) redo.push_back({true, pi, B.phrase_query[pi], nullptr});
        }
    }
    if (redo.empty()) return SA_OK;
    for (const Redo &r : redo)
        if ((rc = redo_query(ix, B, r.phrase, r.idx, r.q, r.sq))) return rc;
    // the repair buffers are larger than the batch's: restore the normal ones and descriptors
    if ((rc = ix->cand.reserve(cand_bytes(sa_n_tiles(ix->n_docs), B.chunk, B.slots)))) return rc;
    SA_CUDA(cudaMemcpyAsync(B.d_row_query.p, B.row_query.data(), (size_t)B.nq * sizeof(u32), cudaMemcpyHostToDevice, ix->stream));
    if (!B.pqs.empty())
        SA_CUDA(cudaMemcpyAsync(B.d_pq.p, B.pqs.data(), B.pqs.size() * sizeof(PhraseQuery), cudaMemcpyHostToDevice, ix->stream));
    if (B.slop > 0) {
        size_t need = 0;
        for (const BatchChunk &C : B.chunks) need = std::max(need, sa_span_scratch_bytes(C.span));
        if ((rc = ix->phrase_scratch.reserve(need))) return rc;
    }
    SA_CUDA(cudaStreamSynchronize(ix->stream));
    if (n_redone) *n_redone = (u32)redo.size();
    return SA_OK;
}

void sa_unpack_keys(const u64 *keys, u64 n, uint32_t *out_docs, float *out_scores) {
    for (u64 i = 0; i < n; i++) {
        u64 key = keys[i];
        if (key == 0) { out_docs[i] = SA_NO_DOC; out_scores[i] = 0.0f; continue; }
        out_docs[i] = 0xFFFFFFFFu - (u32)(key & 0xFFFFFFFFull);
        u32 bits = (u32)(key >> 32);
        memcpy(&out_scores[i], &bits, 4);
    }
}

// keys + the batch's summary tail in ONE device-to-host copy and ONE synchronise
static int download_keys(sa_index *ix, const u64 *d_keys, size_t nk, uint32_t *out_docs, float *out_scores, u64 *tail) {
    int rc;
    if ((rc = ix->h_pinned.reserve((nk + SA_BATCH_TAIL) * sizeof(u64)))) return rc;
    SA_CUDA(cudaMemcpyAsync(ix->h_pinned.p, d_keys, (nk + SA_BATCH_TAIL) * sizeof(u64), cudaMemcpyDeviceToHost, ix->stream));
    SA_CUDA(cudaStreamSynchronize(ix->stream));
    sa_unpack_keys(ix->h_pinned.as<const u64>(), nk, out_docs, out_scores);
    if (tail) memcpy(tail, ix->h_pinned.as<const u64>() + nk, SA_BATCH_TAIL * sizeof(u64));
    return SA_OK;
}

int sa_batch_download_locked(sa_index *ix, uint32_t *out_docs, float *out_scores, uint32_t *n_overflow) {
    BatchState &B = *ix->batch;
    const size_t nk = (size_t)B.nq * B.k;
    u64 tail[SA_BATCH_TAIL] = {0, 0, 0, 0};
    if (n_overflow) *n_overflow = 0;
    int rc = download_keys(ix, ix->topk_out.as<u64>(), nk, out_docs, out_scores, tail);
    if (rc) return rc;
    ix->stats.phrase_cont_words += tail[1];
    ix->stats.phrase_matched_docs += tail[2];
    if (tail[0] == 0) return SA_OK;              // the common case: nothing to repair
    if ((rc = sa_batch_fix_overflow_locked(ix, n_overflow))) return rc;
    return download_keys(ix, ix->topk_out.as<u64>(), nk, out_docs, out_scores, nullptr);
}

extern "C" int sa_batch_upload(sa_index *ix, const uint32_t *terms, const uint32_t *term_starts,
                               const float *idf, uint32_t n_queries, uint32_t slop,
                               float avg_doc_len, float k1, float b, uint32_t k) {
    SA_CHECK(ix, "index is NULL");
    std::lock_guard<std::mutex> g(ix->mu);
    return sa_batch_upload_locked(ix, terms, term_starts, idf, n_queries, slop, avg_doc_len, k1, b, k);
}

extern "C" int sa_batch_execute(sa_index *ix) {
    SA_CHECK(ix, "index is NULL");
    std::lock_guard<std::mutex> g(ix->mu);
    return sa_batch_execute_locked(ix);
}

extern "C" int sa_batch_download(sa_index *ix, uint32_t *out_docs, float *out_scores, uint32_t *n_overflow) {
    SA_CHECK(ix && ix->batch && ix->batch->ready, "no batch uploaded");
    SA_CHECK(out_docs && out_scores, "NULL argument");
    std::lock_guard<std::mutex> g(ix->mu);
    return sa_batch_download_locked(ix, out_docs, out_scores, n_overflow);
}

extern "C" int sa_score_batch_topk(sa_index *ix, const uint32_t *terms, const uint32_t *term_starts,
                                   const float *idf, uint32_t n_queries, uint32_t slop,
                                   float avg_doc_len, float k1, float b, uint32_t k,
                                   uint32_t *out_docs, float *out_scores) {
    SA_CHECK(ix && out_docs && out_scores, "NULL argument");
    std::lock_guard<std::mutex> g(ix->mu);
    int rc = sa_batch_upload_locked(ix, terms, term_starts, idf, n_queries, slop, avg_doc_len, k1, b, k);
    if (rc) return rc;
    if ((rc = sa_batch_execute_locked(ix))) return rc;
    return sa_batch_download_locked(ix, out_docs, out_scores, nullptr);
}

// ------------------------------------------------------------------- timers
KernelTimer::KernelTimer(sa_index *ix_, int kind_) : ix(ix_), kind(kind_), on(ix_->profiling) {
    if (!on) return;
    auto get = [&]() {
        cudaEvent_t e = nullptr;
        if (!ix->free_events.empty()) { e = ix->free_events.back(); ix->free_events.pop_back(); }
        else cudaEventCreate(&e);
        return e;
    };
    e0 = get();
    e1 = get();
    cudaEventRecord(e0, ix->stream);
}

void KernelTimer::stop() {
    if (!on) return;
    cudaEventRecord(e1, ix->stream);
    ix->pending_timers.push_back(TimedLaunch{e0, e1, kind});
    on = false;
}

int sa_resolve_timers(sa_index *ix) {
    if (ix->pending_timers.empty()) return SA_OK;
    SA_CUDA(cudaStreamSynchronize(ix->stream));
    for (auto &t : ix->pending_timers) {
        float ms = 0;
        cudaEventElapsedTime(&ms, t.e0, t.e1);
        if (t.kind == 0) ix->stats.term_kernel_ms += ms;
        else if (t.kind == 1) ix->stats.topk_kernel_ms += ms;
        else ix->stats.phrase_kernel_ms += ms;
        ix->free_events.push_back(t.e0);
        ix->free_events.push_back(t.e1);
    }
    ix->pending_timers.clear();
    return SA_OK;
}

extern "C" int sa_timer_start(sa_index *ix) {
    SA_CHECK(ix, "index is NULL");
    std::lock_guard<std::mutex> g(ix->mu);
    SA_CUDA(cudaSetDevice(ix->device));
    SA_CUDA(cudaStreamSynchronize(ix->stream));
    SA_CUDA(cudaEventRecord(ix->ev0, ix->stream));
    return SA_OK;
}

extern "C" int sa_timer_stop(sa_index *ix, double *ms_out) {
    SA_CHECK(ix && ms_out, "NULL argument");
    std::lock_guard<std::mutex> g(ix->mu);
    SA_CUDA(cudaSetDevice(ix->device));
    SA_CUDA(cudaEventRecord(ix->ev1, ix->stream));
    SA_CUDA(cudaEventSynchronize(ix->ev1));
    float ms = 0;
    SA_CUDA(cudaEventElapsedTime(&ms, ix->ev0, ix->ev1));
    *ms_out = ms;
    return SA_OK;
}

void BatchStateDelete::operator()(BatchState *b) const { delete b; }

void sa_batch_dims(sa_index *ix, u32 *nq, u32 *k) {
    *nq = ix->batch ? ix->batch->nq : 0;
    *k = ix->batch ? ix->batch->k : 0;
}
