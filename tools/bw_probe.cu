// bw_probe.cu -- what HBM bandwidth does a write-dominated stream reach on this H100?
// (fill / copy / 70-30 mix), to put the term kernel's 4N-write-dominated traffic in context.
#include <cstdio>
#include <cuda_runtime.h>
__global__ void fill(float4 *p, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, s = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += s) __stcs(p + i, make_float4(0, 0, 0, 0));
}
__global__ void fill_plain(float4 *p, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, s = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += s) p[i] = make_float4(0, 0, 0, 0);
}
__global__ void copyk(const float4 *a, float4 *b, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, s = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += s) b[i] = a[i];
}
// reads n_r float4, writes n float4 (read fraction = n_r / n)
__global__ void mix(const float4 *a, float4 *b, size_t n, size_t n_r) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, s = (size_t)gridDim.x * blockDim.x;
    for (; i < n; i += s) {
        float4 v = make_float4(0, 0, 0, 0);
        if (i < n_r) v = a[i];
        __stcs(b + i, v);
    }
}
int main() {
    size_t n = (size_t)1 << 28;   // 4 GiB of float4
    float4 *a, *b;
    cudaMalloc(&a, n * 16); cudaMalloc(&b, n * 16);
    cudaMemset(a, 1, n * 16);
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    auto time = [&](const char *name, auto f, double bytes) {
        f(); cudaDeviceSynchronize();
        float best = 1e9;
        for (int r = 0; r < 5; r++) { cudaEventRecord(e0); f(); cudaEventRecord(e1); cudaEventSynchronize(e1);
            float ms; cudaEventElapsedTime(&ms, e0, e1); if (ms < best) best = ms; }
        printf("%-28s %8.3f ms  %8.1f GB/s\n", name, best, bytes / best / 1e6);
    };
    for (int blocks : {132 * 8, 132 * 16, 132 * 64}) {
        printf("grid %d x 256\n", blocks);
        time("fill (st.cs)", [&] { fill<<<blocks, 256>>>(b, n); }, n * 16.0);
        time("fill (plain st)", [&] { fill_plain<<<blocks, 256>>>(b, n); }, n * 16.0);
        time("copy", [&] { copyk<<<blocks, 256>>>(a, b, n); }, n * 32.0);
        time("mix 30% read / 100% write", [&] { mix<<<blocks, 256>>>(a, b, n, n * 3 / 10); }, n * 16.0 * 1.3);
    }
    time("cudaMemsetAsync", [&] { cudaMemsetAsync(b, 0, n * 16); }, n * 16.0);
    time("cudaMemcpyAsync D2D", [&] { cudaMemcpyAsync(b, a, n * 16, cudaMemcpyDeviceToDevice); }, n * 32.0);
    return 0;
}
