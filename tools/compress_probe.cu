// compress_probe.cu -- does Hopper's generic compressible memory make zero-heavy score rows cheaper to write?
//
// Writes 4 GB of float rows at the corpus's document densities (random non-zero floats at density p, zeros
// elsewhere, as synth.py draws them) into cudaMalloc memory and into cuMemCreate memory that asks for
// CU_MEM_ALLOCATION_COMP_GENERIC, with streaming (st.global.cs) and plain stores, and reads them back once;
// a third write kernel stores whole 32 KB tiles per CTA as the term scan does.  Best of 5 after a warm-up.
// Prints the card, its power limit and what compression the driver granted.
//
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a tools/compress_probe.cu -o compress_probe -ldl
#include <cstdio>
#include <cstdint>
#include <dlfcn.h>
#include <cuda.h>
#include <cuda_runtime.h>
#include <cudaTypedefs.h>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { \
    printf("%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); return 1; } } while (0)
#define CU(x) do { CUresult r_ = (x); if (r_ != CUDA_SUCCESS) { \
    printf("%s:%d %s: CUresult %d\n", __FILE__, __LINE__, #x, (int)r_); return 1; } } while (0)

__device__ __forceinline__ uint32_t mix32(uint32_t x) {   // lowbias32
    x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16; return x;
}
// Doc d is non-zero with probability thresh / 2^32; its value is a float in [1, 2).
__device__ __forceinline__ float doc_value(uint32_t d, uint64_t thresh, uint32_t seed) {
    uint32_t h = mix32(d ^ seed);
    return (uint64_t)h < thresh ? __uint_as_float(0x3f800000u | (mix32(h) >> 9)) : 0.f;
}
template <bool kStreaming>
__global__ void write_rows(float4 *p, size_t n4, uint64_t thresh, uint32_t seed) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, s = (size_t)gridDim.x * blockDim.x;
    for (; i < n4; i += s) {
        uint32_t d = (uint32_t)(i * 4);
        float4 v = make_float4(doc_value(d, thresh, seed), doc_value(d + 1, thresh, seed),
                               doc_value(d + 2, thresh, seed), doc_value(d + 3, thresh, seed));
        if (kStreaming) __stcs(p + i, v); else p[i] = v;
    }
}
// One CTA writes whole 32 KB tiles (8,192 docs), the shape in which the term scan flushes its rows.
__global__ void write_tiles(float4 *p, size_t n4, uint64_t thresh, uint32_t seed) {
    const size_t tile4 = 2048, n_tiles = n4 / tile4;
    for (size_t t = blockIdx.x; t < n_tiles; t += gridDim.x)
        for (size_t i = t * tile4 + threadIdx.x; i < (t + 1) * tile4; i += blockDim.x) {
            uint32_t d = (uint32_t)(i * 4);
            __stcs(p + i, make_float4(doc_value(d, thresh, seed), doc_value(d + 1, thresh, seed),
                                      doc_value(d + 2, thresh, seed), doc_value(d + 3, thresh, seed)));
        }
}
__global__ void read_rows(const float4 *p, size_t n4, float *sink) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, s = (size_t)gridDim.x * blockDim.x;
    float acc = 0.f;
    for (; i < n4; i += s) { float4 v = __ldcs(p + i); acc += v.x + v.y + v.z + v.w; }
    if (acc == -1.f) *sink = acc;   // never true; keeps the loads
}

template <typename F> static bool entry(const char *sym, F *fn) {
    cudaDriverEntryPointQueryResult q;
    return cudaGetDriverEntryPointByVersion(sym, (void **)fn, 12000, cudaEnableDefault, &q) == cudaSuccess &&
           q == cudaDriverEntryPointSuccess;
}

static void print_power_limit() {   // NVML through dlopen, so the probe links against cudart alone
    void *h = dlopen("libnvidia-ml.so.1", RTLD_NOW);
    if (!h) { printf("power limit: unknown (no NVML)\n"); return; }
    typedef int (*init_t)(); typedef int (*handle_t)(unsigned, void **);
    typedef int (*limit_t)(void *, unsigned *); typedef int (*clock_t_)(void *, int, unsigned *);
    auto init = (init_t)dlsym(h, "nvmlInit_v2");
    auto get = (handle_t)dlsym(h, "nvmlDeviceGetHandleByIndex_v2");
    auto lim = (limit_t)dlsym(h, "nvmlDeviceGetEnforcedPowerLimit");
    auto clk = (clock_t_)dlsym(h, "nvmlDeviceGetMaxClockInfo");
    void *dev = nullptr; unsigned mw = 0, mhz = 0;
    int dev_index = 0;
    cudaGetDevice(&dev_index);
    if (init && get && lim && init() == 0 && get((unsigned)dev_index, &dev) == 0 && lim(dev, &mw) == 0) {
        if (clk) clk(dev, 1 /* NVML_CLOCK_SM */, &mhz);
        printf("power limit: %.0f W, max SM clock %u MHz\n", mw / 1000.0, mhz);
    } else {
        printf("power limit: unknown\n");
    }
}

int main() {
    const size_t bytes = (size_t)4 << 30, n4 = bytes / 16;
    cudaDeviceProp prop; CK(cudaGetDeviceProperties(&prop, 0));
    printf("device: %s, %d SMs\n", prop.name, prop.multiProcessorCount);
    print_power_limit();

    PFN_cuDeviceGetAttribute_v2000 getAttr; PFN_cuMemCreate_v10020 memCreate;
    PFN_cuMemGetAllocationGranularity_v10020 granularity; PFN_cuMemAddressReserve_v10020 reserve;
    PFN_cuMemMap_v10020 map; PFN_cuMemSetAccess_v10020 setAccess;
    PFN_cuMemGetAllocationPropertiesFromHandle_v10020 propsOf;
    CK(cudaFree(nullptr));
    if (!entry("cuDeviceGetAttribute", &getAttr) || !entry("cuMemCreate", &memCreate) ||
        !entry("cuMemGetAllocationGranularity", &granularity) || !entry("cuMemAddressReserve", &reserve) ||
        !entry("cuMemMap", &map) || !entry("cuMemSetAccess", &setAccess) ||
        !entry("cuMemGetAllocationPropertiesFromHandle", &propsOf)) {
        printf("driver entry points missing\n"); return 1;
    }
    int supported = 0;
    CU(getAttr(&supported, CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED, 0));
    printf("CU_DEVICE_ATTRIBUTE_GENERIC_COMPRESSION_SUPPORTED = %d\n", supported);

    CUmemAllocationProp ap = {};
    ap.type = CU_MEM_ALLOCATION_TYPE_PINNED;
    ap.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
    ap.location.id = 0;
    ap.allocFlags.compressionType = CU_MEM_ALLOCATION_COMP_GENERIC;
    size_t gran = 0;
    CU(granularity(&gran, &ap, CU_MEM_ALLOC_GRANULARITY_MINIMUM));
    size_t mapped = (bytes + gran - 1) / gran * gran;
    CUmemGenericAllocationHandle hdl;
    CU(memCreate(&hdl, mapped, &ap, 0));
    CUmemAllocationProp got = {};
    CU(propsOf(&got, hdl));
    printf("granularity %zu B; compressionType requested %d, granted %d\n", gran,
           (int)CU_MEM_ALLOCATION_COMP_GENERIC, (int)got.allocFlags.compressionType);
    CUdeviceptr va;
    CU(reserve(&va, mapped, gran, 0, 0));
    CU(map(va, mapped, 0, hdl, 0));
    CUmemAccessDesc acc = {};
    acc.location = ap.location; acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
    CU(setAccess(va, mapped, &acc, 1));

    float4 *plain; CK(cudaMalloc(&plain, bytes));
    float *sink; CK(cudaMalloc(&sink, 4));
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    auto best_ms = [&](auto f) {
        f(); cudaDeviceSynchronize();
        float best = 1e9f;
        for (int r = 0; r < 5; r++) {
            cudaEventRecord(e0); f(); cudaEventRecord(e1); cudaEventSynchronize(e1);
            float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms;
        }
        return best;
    };
    const int blocks = prop.multiProcessorCount * 16, threads = 256;
    struct Arm { const char *name; float4 *p; } arms[2] = {{"cudaMalloc", plain}, {"compressible", (float4 *)va}};
    const double densities[] = {1, 0.3, 0.1, 0.03, 0.01, 1e-3, 1e-4, 0};
    printf("\n4 GB rows, grid %d x %d, best of 5; GB/s counts 4 GB per pass\n", blocks, threads);
    printf("%-8s %-13s %10s %10s %10s %10s %10s\n", "density", "memory", "st.cs ms", "st ms", "tile ms", "read ms",
           "st.cs GB/s");
    for (double d : densities) {
        uint64_t thresh = (uint64_t)(d * 4294967296.0);
        for (const Arm &a : arms) {
            float cs = best_ms([&] { write_rows<true><<<blocks, threads>>>(a.p, n4, thresh, 12345u); });
            float st = best_ms([&] { write_rows<false><<<blocks, threads>>>(a.p, n4, thresh, 12345u); });
            float tl = best_ms([&] { write_tiles<<<blocks, threads>>>(a.p, n4, thresh, 12345u); });
            float rd = best_ms([&] { read_rows<<<blocks, threads>>>(a.p, n4, sink); });
            printf("%-8g %-13s %10.3f %10.3f %10.3f %10.3f %10.1f\n", d, a.name, cs, st, tl, rd, bytes / cs / 1e6);
        }
    }
    for (const Arm &a : arms)
        printf("cudaMemsetAsync(0), %-13s %8.3f ms\n", a.name, best_ms([&] { cudaMemsetAsync(a.p, 0, bytes); }));
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    print_power_limit();
    return 0;
}
