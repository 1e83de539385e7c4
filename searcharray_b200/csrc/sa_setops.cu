// sa_setops.cu -- device versions of the reference's native sorted-set ops (SURVEY 8a row 10, 8b).
//
// Replaces, op for op (reference paths relative to softwaredoug/searcharray):
//   intersect / adjacent / intersect_with_adjacents   searcharray/roaringish/intersect.pyx:32-390
//   merge / sort_merge_counts                         searcharray/roaringish/merge.pyx:54-232
//   unique                                            searcharray/roaringish/unique.pyx:87-145
//   popcount64 / popcount_reduce_at / key_sum_over    searcharray/roaringish/popcount.pyx:71-204
//   payload_slice / as_dense                          searcharray/roaringish/roaringish_ops.pyx:46-98
//
// The reference walks both lists with a galloping two-pointer loop and returns INDEX arrays; on inputs
// sorted by the masked value its output is plain set semantics with first-occurrence indices (SURVEY 8a
// row 10: 3,000 random trials; re-checked against the golden tables in tests/test_setops_gpu.py), so any
// parallel intersection is admissible.  Here:
//   * the intersect family is ONE kernel (`partner_kernel`): a CTA takes 1,024 consecutive lhs elements,
//     finds the rhs range that can hold their partners with two warp-cooperative 32-ary searches (ballots),
//     STAGES that range block by block in shared memory with TMA bulk copies (cp.async.bulk + mbarrier) and
//     resolves every element by a binary search in shared memory.  When the rhs range is far longer than the
//     tile (|lhs| << |rhs|) staging would read words nobody needs, so the CTA searches global memory instead;
//   * merges are rank computations (merge-path: an element's output slot is its own index plus its rank in
//     the other list); grouped sums are head flags + a scan + integer atomics (deterministic);
//   * everything that compacts goes through one flags -> exclusive scan -> ordered write pipeline; the scan is
//     sa_scan.cuh's device-wide `scan_flags`.
// Host in, host out: these exports exist for kernel-level parity tests; the scoring path proper keeps its
// data in HBM.
#include <algorithm>
#include <vector>

#include "sa_common.cuh"
#include "sa_scan.cuh"
#include "sa_tma.cuh"

#define SO_THREADS 256
#define SO_ITEMS 4
#define SO_TILE (SO_THREADS * SO_ITEMS)
#define SO_STAGE_WORDS 4096            // rhs words staged per round (32 KB)
#define SO_NONE 0xFFFFFFFFFFFFFFFFull

// CTAs of the calling thread's last intersect-family call, by path: staged, global search, empty partner range
static thread_local uint64_t g_last_paths[3] = {0, 0, 0};

#define SO_ALLOC_CHECK(p)                                              \
    do {                                                               \
        if (!(p)) {                                                    \
            sa_set_error("device allocation / upload failed");         \
            return SA_ERR_NOMEM;                                       \
        }                                                              \
    } while (0)

// ------------------------------------------------------------------ exclusive scan of u32 flags (sa_scan.cuh)
__global__ void __launch_bounds__(SO_THREADS)
scan_block_kernel(const u32 *__restrict__ flags, u32 *__restrict__ offs, u64 n, u32 *__restrict__ bsum) {
    __shared__ u32 warp_sums[SO_THREADS / 32];
    const u64 base = (u64)blockIdx.x * SO_TILE + (u64)threadIdx.x * SO_ITEMS;
    u32 v[SO_ITEMS], sum = 0;
#pragma unroll
    for (int e = 0; e < SO_ITEMS; e++) {
        v[e] = (base + e < n) ? flags[base + e] : 0u;
        sum += v[e];
    }
    u32 total;
    u32 run = block_exclusive_sum<SO_THREADS>(sum, warp_sums, total);
#pragma unroll
    for (int e = 0; e < SO_ITEMS; e++) {
        if (base + e < n) offs[base + e] = run;
        run += v[e];
    }
    if (threadIdx.x == 0) bsum[blockIdx.x] = total;
}

__global__ void add_bsums_kernel(u32 *__restrict__ offs, u64 n, const u32 *__restrict__ bsum) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) offs[i] += bsum[i / SO_TILE];
}

// offs[i] = number of set flags before i; *total = number of set flags
int scan_flags(DevMem &m, const u32 *d_flags, u32 *d_offs, u64 n, u64 *total, cudaStream_t stream) {
    *total = 0;
    if (n == 0) return SA_OK;
    SA_CHECK(n < (1ull << 32), "array too long for the per-op exports");
    const u32 n_blocks = (u32)((n + SO_TILE - 1) / SO_TILE);
    u32 *d_bsum = m.alloc<u32>(n_blocks + 1);
    SO_ALLOC_CHECK(d_bsum);
    scan_block_kernel<<<n_blocks, SO_THREADS, 0, stream>>>(d_flags, d_offs, n, d_bsum);
    cta_scan_kernel<1024><<<1, 1024, 0, stream>>>(d_bsum, n_blocks, d_bsum + n_blocks);
    add_bsums_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(d_offs, n, d_bsum);
    SA_CUDA(cudaGetLastError());
    u32 t = 0;
    SA_CUDA(cudaMemcpyAsync(&t, d_bsum + n_blocks, sizeof(u32), cudaMemcpyDeviceToHost, stream));
    SA_CUDA(cudaStreamSynchronize(stream));
    *total = t;
    return SA_OK;
}

namespace {

// ------------------------------------------------------------------ the intersect kernel
// warp-cooperative lower bound on masked values: first i in [lo, hi) with (a[i] & mask) >= key
__device__ __forceinline__ u64 warp_lower_bound_masked(const u64 *__restrict__ a, u64 lo, u64 hi, u64 key, u64 mask) {
    const unsigned lane = threadIdx.x & 31;
    while (hi - lo > 32) {
        const u64 step = (hi - lo + 31) >> 5;
        const u64 probe = lo + (u64)(lane + 1) * step - 1;
        const bool below = (probe < hi) && ((__ldg(a + probe) & mask) < key);
        const int c = __popc(__ballot_sync(0xffffffffu, below));
        lo = lo + (u64)c * step;
        const u64 nhi = lo + step;
        hi = nhi < hi ? nhi : hi;
        if (lo > hi) lo = hi;
    }
    const u64 idx = lo + lane;
    const bool below = (idx < hi) && ((__ldg(a + idx) & mask) < key);
    return lo + (u64)__popc(__ballot_sync(0xffffffffu, below));
}

// For every lhs element i: pos[i] = index of the FIRST rhs element whose masked value equals
// (lhs[i] & mask) + add, or SO_NONE; first[i] = 1 iff i is the first lhs element with its masked value.
// add == 0: intersect (intersect.pyx:32-128); add == lowest set bit of mask: adjacent (:131-190, :213-275).
__global__ void __launch_bounds__(SO_THREADS)
partner_kernel(const u64 *__restrict__ lhs, u64 nl, const u64 *__restrict__ rhs, u64 nr, u64 mask, u64 add,
               u64 *__restrict__ pos_out, u32 *__restrict__ first_out, u32 *__restrict__ n_path_ctas /*[3]*/) {
    __shared__ __align__(16) u64 s_blk[SO_STAGE_WORDS + 4];
    __shared__ __align__(8) u64 s_bar;
    __shared__ u64 s_r[2];
    const unsigned tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const u64 i0 = (u64)blockIdx.x * SO_TILE;
    const u64 i1 = min(nl, i0 + SO_TILE);
    // targets of my elements (consecutive, so one thread's run is sorted)
    u64 tgt[SO_ITEMS], pos[SO_ITEMS];
    bool live[SO_ITEMS];
#pragma unroll
    for (int e = 0; e < SO_ITEMS; e++) {
        const u64 i = i0 + (u64)tid * SO_ITEMS + e;
        live[e] = i < i1;
        pos[e] = SO_NONE;
        tgt[e] = 0;
        if (live[e]) {
            const u64 a = __ldg(lhs + i) & mask;
            tgt[e] = a + add;
            if (tgt[e] < a || (tgt[e] & mask) != tgt[e]) live[e] = false;      // a + delta left the masked field
            first_out[i] = (i == 0 || (__ldg(lhs + i - 1) & mask) != a) ? 1u : 0u;
        }
    }
    // rhs range that can hold partners of this tile: [lower_bound(t_lo), lower_bound(t_hi + 1))
    if (warp < 2) {
        const u64 a = __ldg(lhs + (warp == 0 ? i0 : i1 - 1)) & mask;
        u64 key = a + add;
        u64 r;
        if (key < a) r = nr;                                                    // overflow: nothing can match
        else if (warp == 0) r = warp_lower_bound_masked(rhs, 0, nr, key, mask);
        else r = (key == SO_NONE) ? nr : warp_lower_bound_masked(rhs, 0, nr, key + 1, mask);
        if (lane == 0) s_r[warp] = r;
    }
    if (tid == 0) {
        sa_mbar_init(&s_bar, 1);
        sa_mbar_fence_init();
    }
    __syncthreads();
    const u64 r0 = s_r[0], r1 = max(s_r[1], s_r[0]);
    if (r1 == r0) {
        if (tid == 0) atomicAdd(n_path_ctas + 2, 1u);
        goto done;
    }
    if (r1 - r0 <= 8ull * SO_TILE) {
        // ---- staged: the rhs range passes through shared memory in TMA-copied blocks
        if (tid == 0) atomicAdd(n_path_ctas + 0, 1u);
        u32 phase = 0;
        for (u64 b0 = r0; b0 < r1; b0 += SO_STAGE_WORDS) {
            const u32 nb = (u32)min((u64)SO_STAGE_WORDS, r1 - b0);
            u32 head = (u32)(((uintptr_t)(rhs + b0) >> 3) & 1u);
            if (tid == 0) {
                sa_fence_proxy_async();
                sa_mbar_expect_tx(&s_bar, sa_stage_bytes(rhs, b0, nb));
                sa_stage_issue(s_blk, rhs, b0, nb, &s_bar);
            }
            sa_mbar_wait(&s_bar, phase);
            phase ^= 1u;
            const u64 *blk = s_blk + head;
            const u64 v_first = blk[0] & mask, v_last = blk[nb - 1] & mask;
#pragma unroll
            for (int e = 0; e < SO_ITEMS; e++) {
                if (!live[e] || pos[e] != SO_NONE || tgt[e] < v_first || tgt[e] > v_last) continue;
                u32 lo = 0, hi = nb;
                while (lo < hi) {
                    const u32 mid = (lo + hi) >> 1;
                    if ((blk[mid] & mask) < tgt[e]) lo = mid + 1; else hi = mid;
                }
                if (lo < nb && (blk[lo] & mask) == tgt[e]) pos[e] = b0 + lo;
            }
            __syncthreads();                         // everyone is done with the block before it is overwritten
        }
    } else {
        // ---- skewed (|lhs tile| << |rhs range|): search global memory, touching only the probed sectors
        if (tid == 0) atomicAdd(n_path_ctas + 1, 1u);
#pragma unroll
        for (int e = 0; e < SO_ITEMS; e++) {
            if (!live[e]) continue;
            u64 lo = r0, hi = r1;
            while (lo < hi) {
                const u64 mid = (lo + hi) >> 1;
                if ((__ldg(rhs + mid) & mask) < tgt[e]) lo = mid + 1; else hi = mid;
            }
            if (lo < r1 && (__ldg(rhs + lo) & mask) == tgt[e]) pos[e] = lo;
        }
    }
done:
#pragma unroll
    for (int e = 0; e < SO_ITEMS; e++) {
        const u64 i = i0 + (u64)tid * SO_ITEMS + e;
        if (i < i1) pos_out[i] = pos[e];
    }
}

__global__ void pair_flag_kernel(const u64 *__restrict__ pos, const u32 *__restrict__ first, u64 n, int need_first,
                                 u32 *__restrict__ flag) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) flag[i] = (pos[i] != SO_NONE && (!need_first || first[i])) ? 1u : 0u;
}

__global__ void pair_write_kernel(const u64 *__restrict__ pos, const u32 *__restrict__ flag, const u32 *__restrict__ offs,
                                  u64 n, u64 *__restrict__ out_idx, u64 *__restrict__ out_partner) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && flag[i]) {
        out_idx[offs[i]] = i;
        if (out_partner) out_partner[offs[i]] = pos[i];
    }
}

// One (lhs -> rhs) partner pass; results compacted to the host.  out_partner may be NULL (membership only).
// need_first (one pair per masked value) follows the reference's drop loops, which start `last` at all ones
// (intersect.pyx:40,145,224): a pair whose masked value equals the mask is skipped while no pair precedes it.  That
// value is the largest there is, so this drops it exactly when it is the only pair.
int run_partner(DevMem &m, const u64 *h_lhs, const u64 *d_lhs, u64 nl, const u64 *d_rhs, u64 nr, u64 mask, u64 add,
                int need_first, u64 *h_idx, u64 *h_partner, u64 *n_out) {
    *n_out = 0;
    if (nl == 0 || nr == 0) return SA_OK;
    u64 *d_pos = m.alloc<u64>(nl);
    u32 *d_first = m.alloc<u32>(nl), *d_flag = m.alloc<u32>(nl), *d_offs = m.alloc<u32>(nl), *d_cnt = m.alloc<u32>(3);
    SO_ALLOC_CHECK(d_pos && d_first && d_flag && d_offs && d_cnt);
    SA_CUDA(cudaMemset(d_cnt, 0, 3 * sizeof(u32)));
    const unsigned tiles = (unsigned)((nl + SO_TILE - 1) / SO_TILE), blocks = (unsigned)((nl + 255) / 256);
    partner_kernel<<<tiles, SO_THREADS>>>(d_lhs, nl, d_rhs, nr, mask, add, d_pos, d_first, d_cnt);
    pair_flag_kernel<<<blocks, 256>>>(d_pos, d_first, nl, need_first, d_flag);
    SA_CUDA(cudaGetLastError());
    u64 total = 0;
    int rc = scan_flags(m, d_flag, d_offs, nl, &total, 0);
    if (rc) return rc;
    if (total) {
        u64 *d_oi = m.alloc<u64>(total), *d_op = h_partner ? m.alloc<u64>(total) : nullptr;
        SO_ALLOC_CHECK(d_oi && (d_op || !h_partner));
        pair_write_kernel<<<blocks, 256>>>(d_pos, d_flag, d_offs, nl, d_oi, d_op);
        SA_CUDA(cudaGetLastError());
        SA_CUDA(cudaMemcpy(h_idx, d_oi, total * sizeof(u64), cudaMemcpyDeviceToHost));
        if (h_partner) SA_CUDA(cudaMemcpy(h_partner, d_op, total * sizeof(u64), cudaMemcpyDeviceToHost));
    }
    u32 paths[3];
    SA_CUDA(cudaMemcpy(paths, d_cnt, sizeof(paths), cudaMemcpyDeviceToHost));
    for (int k = 0; k < 3; k++) g_last_paths[k] += paths[k];
    if (need_first && total == 1 && (h_lhs[h_idx[0]] & mask) == mask) total = 0;
    *n_out = total;
    return SA_OK;
}

// ------------------------------------------------------------------ ranks (merge-path)
#define SO_UNPAIRED 0xFFFFFFFFu

__device__ __forceinline__ u64 bound(const u64 *__restrict__ a, u64 lo, u64 hi, u64 x, bool upper) {
    while (lo < hi) {
        const u64 mid = (lo + hi) >> 1;
        const u64 y = __ldg(a + mid);
        if (upper ? (y <= x) : (y < x)) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// rank[i] = number of b elements < a[i] (upper == 0) or <= a[i] (upper == 1).  The reference's two-pointer merge
// pairs the k-th copy of a value in a with the k-th copy in b (merge.pyx:64-77): pair[i] = the index in b of a[i]'s
// partner, or SO_UNPAIRED when b holds fewer copies of the value than come up to a[i] in a.
__global__ void rank_kernel(const u64 *__restrict__ a, u64 na, const u64 *__restrict__ b, u64 nb, int upper,
                            u32 *__restrict__ rank, u32 *__restrict__ pair) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= na) return;
    const u64 x = a[i];
    const u64 lo = bound(b, 0, nb, x, false), hi = bound(b, lo, nb, x, true);
    rank[i] = (u32)(upper ? hi : lo);
    const u64 p = lo + (i - bound(a, 0, i, x, false));               // a[i] is copy number i - first of its value
    pair[i] = p < hi ? (u32)p : SO_UNPAIRED;
}

__global__ void unpaired_kernel(const u32 *__restrict__ pair, u32 *__restrict__ out, u64 n) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = pair[i] == SO_UNPAIRED ? 1u : 0u;
}

// merged[i + kept_before(rank_l[i])] = lhs[i];  merged[kept_before(j) + rank_r[j]] = rhs[j] (kept rhs only).  Inside
// a run of equal values the lhs copies come first, the paired ones first among them, then the kept rhs copies: the
// order the reference's merge writes them in.
__global__ void merge_write_kernel(const u64 *__restrict__ lhs, u64 nl, const u64 *__restrict__ rhs, u64 nr,
                                   const u32 *__restrict__ rank_l, const u32 *__restrict__ rank_r,
                                   const u32 *__restrict__ keep_r, const u32 *__restrict__ kept_before /*[nr + 1]*/,
                                   const float *__restrict__ lcnt, const float *__restrict__ rcnt,
                                   const u32 *__restrict__ pair_l,
                                   u64 *__restrict__ out, float *__restrict__ out_cnt) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nl) {
        const u32 r = rank_l[i];
        const u64 at = i + (kept_before ? kept_before[r] : r);
        out[at] = lhs[i];
        if (out_cnt) out_cnt[at] = (pair_l && pair_l[i] != SO_UNPAIRED) ? __fadd_rn(lcnt[i], rcnt[pair_l[i]]) : lcnt[i];
    } else if (i < nl + nr) {
        const u64 j = i - nl;
        if (keep_r && !keep_r[j]) return;
        const u64 at = (kept_before ? kept_before[j] : j) + rank_r[j];
        out[at] = rhs[j];
        if (out_cnt) out_cnt[at] = rcnt[j];
    }
}

// ------------------------------------------------------------------ grouped ops
__global__ void head_flag_kernel(const u64 *__restrict__ a, u64 n, u64 rshift, u32 *__restrict__ flag) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) flag[i] = (i == 0 || (a[i] >> rshift) != (a[i - 1] >> rshift)) ? 1u : 0u;
}

__global__ void unique_write_kernel(const u64 *__restrict__ a, u64 n, u64 rshift, const u32 *__restrict__ flag,
                                    const u32 *__restrict__ offs, u64 *__restrict__ out) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && flag[i]) out[offs[i]] = a[i] >> rshift;
}

// group index of element i = offs[i] + flag[i] - 1 (offs = exclusive scan of the head flags)
__global__ void group_sum_kernel(const u64 *__restrict__ ids, const u64 *__restrict__ val, u64 n, int popcount,
                                 const u32 *__restrict__ flag, const u32 *__restrict__ offs,
                                 u64 *__restrict__ ids_out, unsigned long long *__restrict__ sums) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u32 g = offs[i] + flag[i] - 1u;
    if (flag[i]) ids_out[g] = ids[i];
    const unsigned long long v = popcount ? (unsigned long long)__popcll(val[i]) : (unsigned long long)val[i];
    if (v) atomicAdd(&sums[g], v);
}

__global__ void u64_to_f32_kernel(const unsigned long long *__restrict__ in, float *__restrict__ out, u64 n) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (float)in[i];
}

__global__ void popcount64_kernel(const u64 *__restrict__ a, u64 n, u64 *__restrict__ out) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = (u64)__popcll(a[i]);
}

__global__ void payload_flag_kernel(const u64 *__restrict__ a, u64 n, u64 msb_mask, u64 lo, u64 hi, u32 *__restrict__ flag) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const u64 v = a[i] & msb_mask;             // UNSHIFTED, like roaringish_ops.pyx:55 (SURVEY quirk vi)
        flag[i] = (v >= lo && v <= hi) ? 1u : 0u;
    }
}

__global__ void copy_flagged_kernel(const u64 *__restrict__ a, u64 n, const u32 *__restrict__ flag,
                                    const u32 *__restrict__ offs, u64 *__restrict__ out) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && flag[i]) out[offs[i]] = a[i];
}

// scatter_assign.h:8-29: out[idx[i]] = val[i], later duplicates win.  For the sorted index lists the
// reference passes (doc ids ascending) "later wins" == "the last element of a run writes": deterministic.
__global__ void dense_scatter_kernel(const u64 *__restrict__ idx, const float *__restrict__ val, u64 n, u64 size,
                                     float *__restrict__ out) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const u64 d = idx[i];
    if (d < size && (i + 1 == n || idx[i + 1] != d)) out[d] = val[i];
}

unsigned blocks_for(u64 n) { return (unsigned)((n + 255) / 256); }

}  // namespace

// ================================================================== C ABI
extern "C" int sa_op_intersect(const uint64_t *lhs, uint64_t n_lhs, const uint64_t *rhs, uint64_t n_rhs,
                               uint64_t mask, int drop_duplicates, int device,
                               uint64_t *lhs_idx_out, uint64_t *rhs_idx_out,
                               uint64_t *n_lhs_out, uint64_t *n_rhs_out) {
    SA_CHECK(lhs_idx_out && rhs_idx_out && n_lhs_out && n_rhs_out, "NULL argument");
    SA_CHECK(mask != 0, "Mask cannot be zero");                       // intersect.pyx:291-292 (ValueError)
    g_last_paths[0] = g_last_paths[1] = g_last_paths[2] = 0;
    *n_lhs_out = *n_rhs_out = 0;
    if (n_lhs == 0 || n_rhs == 0) return SA_OK;
    SA_CHECK(lhs && rhs, "NULL argument");
    SA_CUDA(cudaSetDevice(device));
    DevMem m;
    u64 *d_l = m.upload(lhs, n_lhs), *d_r = m.upload(rhs, n_rhs);
    SO_ALLOC_CHECK(d_l && d_r);
    int rc;
    if (drop_duplicates) {
        // one pair per distinct common masked value: first occurrence on both sides (intersect.pyx:32-74)
        if ((rc = run_partner(m, lhs, d_l, n_lhs, d_r, n_rhs, mask, 0, 1, lhs_idx_out, rhs_idx_out, n_lhs_out))) return rc;
        *n_rhs_out = *n_lhs_out;
        return SA_OK;
    }
    // keep: every lhs index whose value occurs in rhs, every rhs index whose value occurs in lhs (:77-128)
    if ((rc = run_partner(m, lhs, d_l, n_lhs, d_r, n_rhs, mask, 0, 0, lhs_idx_out, nullptr, n_lhs_out))) return rc;
    return run_partner(m, rhs, d_r, n_rhs, d_l, n_lhs, mask, 0, 0, rhs_idx_out, nullptr, n_rhs_out);
}

extern "C" int sa_op_adjacent(const uint64_t *lhs, uint64_t n_lhs, const uint64_t *rhs, uint64_t n_rhs,
                              uint64_t mask, int device, uint64_t *lhs_idx_out, uint64_t *rhs_idx_out,
                              uint64_t *n_out) {
    SA_CHECK(lhs_idx_out && rhs_idx_out && n_out, "NULL argument");
    SA_CHECK(mask != 0, "Mask cannot be zero");
    g_last_paths[0] = g_last_paths[1] = g_last_paths[2] = 0;
    *n_out = 0;
    if (n_lhs == 0 || n_rhs == 0) return SA_OK;
    SA_CHECK(lhs && rhs, "NULL argument");
    SA_CUDA(cudaSetDevice(device));
    DevMem m;
    u64 *d_l = m.upload(lhs, n_lhs), *d_r = m.upload(rhs, n_rhs);
    SO_ALLOC_CHECK(d_l && d_r);
    const u64 delta = mask & (~mask + 1);                            // lowest set bit (intersect.pyx:140)
    return run_partner(m, lhs, d_l, n_lhs, d_r, n_rhs, mask, delta, 1, lhs_idx_out, rhs_idx_out, n_out);
}

extern "C" int sa_op_intersect_with_adjacents(const uint64_t *lhs, uint64_t n_lhs, const uint64_t *rhs, uint64_t n_rhs,
                                              uint64_t mask, int device,
                                              uint64_t *lhs_idx_out, uint64_t *rhs_idx_out, uint64_t *n_out,
                                              uint64_t *adj_lhs_idx_out, uint64_t *adj_rhs_idx_out, uint64_t *n_adj_out) {
    SA_CHECK(lhs_idx_out && rhs_idx_out && n_out && adj_lhs_idx_out && adj_rhs_idx_out && n_adj_out, "NULL argument");
    SA_CHECK(mask != 0, "Mask cannot be zero");
    g_last_paths[0] = g_last_paths[1] = g_last_paths[2] = 0;
    *n_out = *n_adj_out = 0;
    if (n_lhs == 0 || n_rhs == 0) return SA_OK;
    SA_CHECK(lhs && rhs, "NULL argument");
    SA_CUDA(cudaSetDevice(device));
    DevMem m;
    u64 *d_l = m.upload(lhs, n_lhs), *d_r = m.upload(rhs, n_rhs);
    SO_ALLOC_CHECK(d_l && d_r);
    const u64 delta = mask & (~mask + 1);
    int rc = run_partner(m, lhs, d_l, n_lhs, d_r, n_rhs, mask, 0, 1, lhs_idx_out, rhs_idx_out, n_out);
    if (rc) return rc;
    return run_partner(m, lhs, d_l, n_lhs, d_r, n_rhs, mask, delta, 1, adj_lhs_idx_out, adj_rhs_idx_out, n_adj_out);
}

// merge.pyx:54-158: sorted two-way merge; an element present in both lists appears twice unless drop_duplicates,
// which drops the rhs copies paired with an lhs copy
static int merge_common(const u64 *lhs, u64 nl, const u64 *rhs, u64 nr, int drop, const float *lcnt, const float *rcnt,
                        int device, u64 *out, float *out_cnt, u64 *n_out) {
    *n_out = 0;
    SA_CUDA(cudaSetDevice(device));
    if (nl + nr == 0) return SA_OK;
    SA_CHECK(nl + nr < (1ull << 32), "array too long for the per-op exports");
    DevMem m;
    u64 *d_l = m.upload(lhs, nl), *d_r = m.upload(rhs, nr);
    float *d_lc = lcnt ? m.upload(lcnt, nl) : nullptr, *d_rc = rcnt ? m.upload(rcnt, nr) : nullptr;
    u32 *rank_l = m.alloc<u32>(nl), *pair_l = m.alloc<u32>(nl), *rank_r = m.alloc<u32>(nr), *pair_r = m.alloc<u32>(nr);
    SO_ALLOC_CHECK(d_l && d_r && rank_l && pair_l && rank_r && pair_r && (!lcnt || (d_lc && d_rc)));
    if (nl) rank_kernel<<<blocks_for(nl), 256>>>(d_l, nl, d_r, nr, 0, rank_l, pair_l);         // # rhs <  lhs[i]
    if (nr) rank_kernel<<<blocks_for(nr), 256>>>(d_r, nr, d_l, nl, 1, rank_r, pair_r);         // # lhs <= rhs[j]
    SA_CUDA(cudaGetLastError());
    u32 *keep_r = nullptr, *kept_before = nullptr;
    u64 kept = nr;
    if (drop && nr) {
        keep_r = m.alloc<u32>(nr);
        kept_before = m.alloc<u32>(nr + 1);
        SO_ALLOC_CHECK(keep_r && kept_before);
        unpaired_kernel<<<blocks_for(nr), 256>>>(pair_r, keep_r, nr);
        int rc = scan_flags(m, keep_r, kept_before, nr, &kept, 0);
        if (rc) return rc;
        const u32 k32 = (u32)kept;
        SA_CUDA(cudaMemcpy(kept_before + nr, &k32, sizeof(u32), cudaMemcpyHostToDevice));
    }
    const u64 total = nl + kept;
    u64 *d_out = m.alloc<u64>(total);
    float *d_oc = out_cnt ? m.alloc<float>(total) : nullptr;
    SO_ALLOC_CHECK(d_out && (d_oc || !out_cnt));
    merge_write_kernel<<<blocks_for(nl + nr), 256>>>(d_l, nl, d_r, nr, rank_l, rank_r, keep_r, kept_before, d_lc, d_rc,
                                                     out_cnt ? pair_l : nullptr, d_out, d_oc);
    SA_CUDA(cudaGetLastError());
    SA_CUDA(cudaMemcpy(out, d_out, total * sizeof(u64), cudaMemcpyDeviceToHost));
    if (out_cnt) SA_CUDA(cudaMemcpy(out_cnt, d_oc, total * sizeof(float), cudaMemcpyDeviceToHost));
    *n_out = total;
    return SA_OK;
}

extern "C" int sa_op_merge(const uint64_t *lhs, uint64_t n_lhs, const uint64_t *rhs, uint64_t n_rhs,
                           int drop_duplicates, int device, uint64_t *out, uint64_t *n_out) {
    SA_CHECK(out && n_out && (lhs || !n_lhs) && (rhs || !n_rhs), "NULL argument");
    return merge_common(lhs, n_lhs, rhs, n_rhs, drop_duplicates, nullptr, nullptr, device, out, nullptr, n_out);
}

// merge.pyx:161-232: union of two (id, count) lists sorted by id, counts of a shared id added (float32)
extern "C" int sa_op_sort_merge_counts(const uint64_t *lhs_ids, const float *lhs_counts, uint64_t n_lhs,
                                       const uint64_t *rhs_ids, const float *rhs_counts, uint64_t n_rhs,
                                       int device, uint64_t *ids_out, float *counts_out, uint64_t *n_out) {
    SA_CHECK(ids_out && counts_out && n_out && (lhs_ids || !n_lhs) && (rhs_ids || !n_rhs), "NULL argument");
    SA_CHECK((lhs_counts || !n_lhs) && (rhs_counts || !n_rhs), "NULL argument");
    static const float zero = 0.0f;
    return merge_common(lhs_ids, n_lhs, rhs_ids, n_rhs, 1, lhs_counts ? lhs_counts : &zero, rhs_counts ? rhs_counts : &zero,
                        device, ids_out, counts_out, n_out);
}

// unique.pyx:87-145: run-length dedup of (arr >> rshift) on a sorted array
extern "C" int sa_op_unique(const uint64_t *arr, uint64_t n, uint64_t rshift, int device, uint64_t *out, uint64_t *n_out) {
    SA_CHECK(out && n_out && (arr || !n), "NULL argument");
    SA_CHECK(rshift < 64, "rshift must be < 64");
    *n_out = 0;
    if (n == 0) return SA_OK;
    SA_CUDA(cudaSetDevice(device));
    DevMem m;
    u64 *d_a = m.upload(arr, n);
    u32 *flag = m.alloc<u32>(n), *offs = m.alloc<u32>(n);
    SO_ALLOC_CHECK(d_a && flag && offs);
    head_flag_kernel<<<blocks_for(n), 256>>>(d_a, n, rshift, flag);
    u64 total = 0;
    int rc = scan_flags(m, flag, offs, n, &total, 0);
    if (rc) return rc;
    u64 *d_out = m.alloc<u64>(total);
    SO_ALLOC_CHECK(d_out);
    unique_write_kernel<<<blocks_for(n), 256>>>(d_a, n, rshift, flag, offs, d_out);
    SA_CUDA(cudaGetLastError());
    SA_CUDA(cudaMemcpy(out, d_out, total * sizeof(u64), cudaMemcpyDeviceToHost));
    *n_out = total;
    return SA_OK;
}

extern "C" int sa_op_popcount64(const uint64_t *arr, uint64_t n, int device, uint64_t *out) {
    SA_CHECK((arr && out) || !n, "NULL argument");
    if (n == 0) return SA_OK;
    SA_CUDA(cudaSetDevice(device));
    DevMem m;
    u64 *d_a = m.upload(arr, n), *d_o = m.alloc<u64>(n);
    SO_ALLOC_CHECK(d_a && d_o);
    popcount64_kernel<<<blocks_for(n), 256>>>(d_a, n, d_o);
    SA_CUDA(cudaGetLastError());
    SA_CUDA(cudaMemcpy(out, d_o, n * sizeof(u64), cudaMemcpyDeviceToHost));
    return SA_OK;
}

// popcount.pyx:124-204: runs of equal ids -> (id, sum); zero sums are KEPT (SURVEY quirk iv)
static int grouped(const u64 *ids, const u64 *val, u64 n, int popcount, int device, u64 *ids_out, float *cnt_out, u64 *n_out) {
    *n_out = 0;
    if (n == 0) return SA_OK;
    SA_CUDA(cudaSetDevice(device));
    DevMem m;
    u64 *d_i = m.upload(ids, n), *d_v = m.upload(val, n);
    u32 *flag = m.alloc<u32>(n), *offs = m.alloc<u32>(n);
    SO_ALLOC_CHECK(d_i && d_v && flag && offs);
    head_flag_kernel<<<blocks_for(n), 256>>>(d_i, n, 0, flag);
    u64 total = 0;
    int rc = scan_flags(m, flag, offs, n, &total, 0);
    if (rc) return rc;
    u64 *d_io = m.alloc<u64>(total);
    unsigned long long *d_s = m.alloc<unsigned long long>(total);
    float *d_c = m.alloc<float>(total);
    SO_ALLOC_CHECK(d_io && d_s && d_c);
    SA_CUDA(cudaMemset(d_s, 0, total * sizeof(unsigned long long)));
    group_sum_kernel<<<blocks_for(n), 256>>>(d_i, d_v, n, popcount, flag, offs, d_io, d_s);
    u64_to_f32_kernel<<<blocks_for(total), 256>>>(d_s, d_c, total);
    SA_CUDA(cudaGetLastError());
    SA_CUDA(cudaMemcpy(ids_out, d_io, total * sizeof(u64), cudaMemcpyDeviceToHost));
    SA_CUDA(cudaMemcpy(cnt_out, d_c, total * sizeof(float), cudaMemcpyDeviceToHost));
    *n_out = total;
    return SA_OK;
}

extern "C" int sa_op_popcount_reduce_at(const uint64_t *ids, const uint64_t *payload, uint64_t n, int device,
                                        uint64_t *ids_out, float *counts_out, uint64_t *n_out) {
    SA_CHECK(ids_out && counts_out && n_out && ((ids && payload) || !n), "NULL argument");
    return grouped(ids, payload, n, 1, device, ids_out, counts_out, n_out);
}

extern "C" int sa_op_key_sum_over(const uint64_t *ids, const uint64_t *counts, uint64_t n, int device,
                                  uint64_t *ids_out, float *counts_out, uint64_t *n_out) {
    SA_CHECK(ids_out && counts_out && n_out && ((ids && counts) || !n), "NULL argument");
    return grouped(ids, counts, n, 0, device, ids_out, counts_out, n_out);
}

// popcount.pyx:212-237,271-278 (popcount64_reduce with key_shift 36, value_mask 0x3FFFF): grouped() over (doc id,
// position bits).  The sum per doc is exact in 64 bits and rounded to float32 once, as the reference's `(float)acc`;
// a doc's count is not bounded by the 19-bit tf of the index's records (up to 18 * 2^18 positions per doc).
extern "C" int sa_op_popcount64_reduce(const uint64_t *words, uint64_t n, int device,
                                       uint64_t *keys_out, float *counts_out, uint64_t *n_out) {
    SA_CHECK(keys_out && counts_out && n_out && (words || !n), "NULL argument");
    std::vector<u64> docs(n), bits(n);
    for (u64 i = 0; i < n; i++) {
        docs[i] = words[i] >> SA_KEY_SHIFT;
        bits[i] = words[i] & SA_LSB_MASK;
    }
    return grouped(docs.data(), bits.data(), n, 1, device, keys_out, counts_out, n_out);
}

extern "C" int sa_op_payload_slice(const uint64_t *arr, uint64_t n, uint64_t msb_mask, uint64_t min_payload,
                                   uint64_t max_payload, int device, uint64_t *out, uint64_t *n_out) {
    SA_CHECK(out && n_out && (arr || !n), "NULL argument");
    *n_out = 0;
    if (n == 0) return SA_OK;
    SA_CUDA(cudaSetDevice(device));
    DevMem m;
    u64 *d_a = m.upload(arr, n);
    u32 *flag = m.alloc<u32>(n), *offs = m.alloc<u32>(n);
    SO_ALLOC_CHECK(d_a && flag && offs);
    payload_flag_kernel<<<blocks_for(n), 256>>>(d_a, n, msb_mask, min_payload, max_payload, flag);
    u64 total = 0;
    int rc = scan_flags(m, flag, offs, n, &total, 0);
    if (rc) return rc;
    u64 *d_out = m.alloc<u64>(total);
    SO_ALLOC_CHECK(d_out);
    copy_flagged_kernel<<<blocks_for(n), 256>>>(d_a, n, flag, offs, d_out);
    SA_CUDA(cudaGetLastError());
    SA_CUDA(cudaMemcpy(out, d_out, total * sizeof(u64), cudaMemcpyDeviceToHost));
    *n_out = total;
    return SA_OK;
}

// roaringish_ops.pyx:84-98 (as_dense): zeros(size) then out[indices] = values (ValueError on length mismatch is the
// Python wrapper's job); indices sorted ascending as every reference caller passes them
extern "C" int sa_op_as_dense(const uint64_t *indices, const float *values, uint64_t n, uint64_t size, int device,
                              float *out) {
    SA_CHECK((out || !size) && ((indices && values) || !n), "NULL argument");
    if (size == 0) return SA_OK;
    SA_CUDA(cudaSetDevice(device));
    DevMem m;
    float *d_o = m.alloc<float>(size);
    SO_ALLOC_CHECK(d_o);
    SA_CUDA(cudaMemset(d_o, 0, size * sizeof(float)));
    if (n) {
        u64 *d_i = m.upload(indices, n);
        float *d_v = m.upload(values, n);
        SO_ALLOC_CHECK(d_i && d_v);
        dense_scatter_kernel<<<blocks_for(n), 256>>>(d_i, d_v, n, size, d_o);
        SA_CUDA(cudaGetLastError());
    }
    SA_CUDA(cudaMemcpy(out, d_o, size * sizeof(float), cudaMemcpyDeviceToHost));
    return SA_OK;
}

// how many CTAs of this thread's last intersect-family call took the TMA-staged path (test hook)
extern "C" uint64_t sa_op_last_staged_ctas(void) { return g_last_paths[0]; }

// ... and how many took each path: staged, global search, empty partner range (test hook)
extern "C" void sa_op_last_path_ctas(uint64_t out[3]) {
    for (int k = 0; k < 3; k++) out[k] = g_last_paths[k];
}
