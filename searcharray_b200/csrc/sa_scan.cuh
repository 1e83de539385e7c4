// sa_scan.cuh -- the exclusive prefix sum behind every ordered compaction of the library.
//
// Three layers, each built on the one before:
//   block_exclusive_sum   one CTA, one value per thread: warp shuffle scan, then the warp totals through shared memory;
//   cta_exclusive_scan    one CTA scans an array of any length in place, in rounds of NT with a running carry;
//   scan_flags            a device-wide scan of u32 flags: 1,024-entry tiles, a one-CTA scan of the tile sums, and
//                         the tile sums added back (sa_setops.cu).
#pragma once
#include "sa_common.cuh"

// Every thread of the NT-thread CTA calls.  Returns the sum of v over the threads before this one; `total` = the
// sum over the CTA.  The leading barrier protects warp_sums from the previous call, so a caller may call repeatedly.
template <int NT, typename T>
__device__ __forceinline__ T block_exclusive_sum(T v, T *warp_sums, T &total) {
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    T incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        T t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    __syncthreads();
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    T base = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < NT / 32; w++) {
        T s = warp_sums[w];
        if (w < (int)warp) base += s;
        tot += s;
    }
    total = tot;
    return base + incl - v;
}

// Every thread of the NT-thread CTA calls.  a[i] becomes the sum of a[0, i); *total = the sum of a[0, n).
template <int NT, typename T>
__device__ __forceinline__ void cta_exclusive_scan(T *__restrict__ a, u32 n, T *__restrict__ total) {
    __shared__ T warp_sums[NT / 32];
    T carry = 0;
    for (u32 b0 = 0; b0 < n; b0 += NT) {
        const u32 i = b0 + threadIdx.x;
        const T v = i < n ? a[i] : T(0);
        T tot;
        const T excl = block_exclusive_sum<NT>(v, warp_sums, tot);
        if (i < n) a[i] = carry + excl;
        carry += tot;
    }
    if (threadIdx.x == 0) *total = carry;
}

template <int NT, typename T>
__global__ void __launch_bounds__(NT) cta_scan_kernel(T *__restrict__ a, u32 n, T *__restrict__ total) {
    cta_exclusive_scan<NT>(a, n, total);
}

// offs[i] = number of set flags before i; *total = number of set flags (on the host when the call returns).  Scratch
// comes from m.  Defined in sa_setops.cu.
int scan_flags(DevMem &m, const u32 *d_flags, u32 *d_offs, u64 n, u64 *total, cudaStream_t stream);
