// sa_topk.cu -- exact top-k over the candidates the scoring kernels collected.
//
// Replaces the reference idiom np.argpartition(scores, -N)[-N:] (searcharray/utils/sort.py:24)
// for the HBM-resident batched path.  The scoring kernels append every score that is >= a
// running, provably-valid lower bound of the k-th best score (sa_term.cu step 4), so the
// candidate list is a superset of the true top-k and is normally a few hundred entries.
// Here one CTA per query selects the exact k best by (score desc, doc id asc): a tight threshold
// (k-th largest of the per-tile maxima) prefilters the per-tile candidate slots to ~k survivors,
// which are sorted in shared memory (bitonic); a radix select handles massive ties.
#include "sa_term.cuh"

#define SEL_THREADS 512
#define SEL_SMEM_KEYS 4096

// visit every candidate key of query q whose tile can hold a key with score bits >= min_score.  RUNS: each tile's
// candidates are sorted descending (deep_tile_collect), so the visit stops at the first key below min_score.
template <bool RUNS, typename F>
__device__ __forceinline__ void for_each_candidate(const TopkCtx &t, u32 q, u32 min_score, F f) {
    const u32 *cnt = t.tile_cnt + (u64)q * t.n_tiles;
    const u32 *tmax = t.tile_max + (u64)q * t.n_tiles;
    const u64 *cand = t.tile_cand + (u64)q * t.n_tiles * t.slots;
    for (u32 tile = threadIdx.x; tile < t.n_tiles; tile += blockDim.x) {
        if (tmax[tile] < min_score) continue;
        const u32 n = cnt[tile];
        const u64 *c = cand + (u64)tile * t.slots;
        for (u32 j = 0; j < n; j++) {
            if (RUNS && (u32)(c[j] >> 32) < min_score) break;
            f(c[j]);
        }
    }
}

template <bool RUNS>
__global__ void __launch_bounds__(SEL_THREADS)
topk_select_kernel(TopkCtx t, u64 doc_base, u64 *__restrict__ out_keys, const u32 *__restrict__ out_index) {
    __shared__ u64 s_keys[SEL_SMEM_KEYS];
    __shared__ u32 s_hist[256];
    __shared__ u64 s_prefix;
    __shared__ u32 s_krem, s_n;

    const u32 q = blockIdx.x;
    const u32 k = t.k;
    const u32 T = t.n_tiles;

    // A. a tight valid threshold: the k-th largest of the per-tile(-group) best scores (they
    //    belong to distinct docs).  The tile maxima were written by the scoring kernel, so this
    //    is one coalesced read of 4*T bytes; 4-pass 8-bit radix select in shared memory.
    u32 *s_max = reinterpret_cast<u32 *>(s_keys);                   // [G] reuse (2 * SEL_SMEM_KEYS u32)
    const u32 GMAX = 2 * SEL_SMEM_KEYS;
    const u32 gs = (T + GMAX - 1) / GMAX;                            // tiles per group
    const u32 G = (T + gs - 1) / gs;
    {
        const u32 *tmax = t.tile_max + (u64)q * T;
        for (u32 g = threadIdx.x; g < G; g += blockDim.x) {
            u32 m = 0;
            for (u32 tile = g * gs; tile < min(T, (g + 1) * gs); tile++) m = max(m, tmax[tile]);
            s_max[g] = m;
        }
    }
    if (threadIdx.x == 0) { s_prefix = 0; s_krem = k; }
    __syncthreads();
    for (int shift = 24; shift >= 0; shift -= 8) {
        for (u32 i = threadIdx.x; i < 256; i += blockDim.x) s_hist[i] = 0;
        __syncthreads();
        const u32 prefix = (u32)s_prefix;
        for (u32 g = threadIdx.x; g < G; g += blockDim.x) {
            u32 key = s_max[g];
            bool match = (shift == 24) || ((key >> (shift + 8)) == (prefix >> (shift + 8)));
            if (match) atomicAdd(&s_hist[(key >> shift) & 255], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            u32 rem = s_krem;
            int b;
            radix_pick(s_hist, rem, b);
            s_krem = rem;
            s_prefix = (u64)(prefix | ((u32)b << shift));
        }
        __syncthreads();
    }
    u32 thr_score = (u32)s_prefix;      // 0 when fewer than k tile groups hold a candidate
    if (thr_score == 0) thr_score = 1;
    __syncthreads();

    // B. survivors with score >= thr_score (a superset of the true top-k, normally ~k of them);
    //    tiles whose best score is below the threshold are skipped without touching their slots
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    for_each_candidate<RUNS>(t, q, thr_score, [&](u64 key) {
        if ((u32)(key >> 32) >= thr_score) {
            u32 slot = atomicAdd(&s_n, 1u);
            if (slot < SEL_SMEM_KEYS) s_keys[slot] = key;
        }
    });
    __syncthreads();
    u32 M = s_n;
    u32 n_valid;
    if (M <= SEL_SMEM_KEYS) {
        u32 n2 = 2;
        while (n2 < M) n2 <<= 1;
        for (u32 i = M + threadIdx.x; i < n2; i += blockDim.x) s_keys[i] = 0ull;
        __syncthreads();
        bitonic_sort_desc_smem(s_keys, n2);
        n_valid = M;
    } else {
        // massive ties around the threshold: radix-select the exact k-th key over all survivors
        if (threadIdx.x == 0) { s_prefix = 0; s_krem = k; }
        __syncthreads();
        for (int shift = 56; shift >= 0; shift -= 8) {
            for (u32 i = threadIdx.x; i < 256; i += blockDim.x) s_hist[i] = 0;
            __syncthreads();
            const u64 prefix = s_prefix;
            for_each_candidate<RUNS>(t, q, thr_score, [&](u64 key) {
                if ((u32)(key >> 32) < thr_score) return;
                bool match = (shift == 56) || ((key >> (shift + 8)) == (prefix >> (shift + 8)));
                if (match) atomicAdd(&s_hist[(key >> shift) & 255], 1u);
            });
            __syncthreads();
            if (threadIdx.x == 0) {
                u32 rem = s_krem;
                int b;
                radix_pick(s_hist, rem, b);
                s_krem = rem;
                s_prefix = prefix | ((u64)b << shift);
            }
            __syncthreads();
        }
        const u64 kth = s_prefix;
        if (threadIdx.x == 0) s_n = 0;
        __syncthreads();
        for_each_candidate<RUNS>(t, q, thr_score, [&](u64 key) {
            if (key >= kth) {
                u32 slot = atomicAdd(&s_n, 1u);
                if (slot < SEL_SMEM_KEYS) s_keys[slot] = key;
            }
        });
        __syncthreads();
        n_valid = min(s_n, (u32)SEL_SMEM_KEYS);
        u32 n2 = 2;
        while (n2 < n_valid) n2 <<= 1;
        for (u32 i = n_valid + threadIdx.x; i < n2; i += blockDim.x) s_keys[i] = 0ull;
        __syncthreads();
        bitonic_sort_desc_smem(s_keys, n2);
    }

    // result keys carry GLOBAL doc ids: score_bits << 32 | (0xFFFFFFFF - global_doc); 0 = empty
    for (u32 i = threadIdx.x; i < k; i += blockDim.x) {
        u64 key = (i < n_valid) ? s_keys[i] : 0ull;
        if (key != 0ull) key -= doc_base;      // (~local) - base == ~(local + base)
        out_keys[(u64)(out_index ? out_index[q] : q) * k + i] = key;
    }
}

// The collapsed top k of query q (collapse_tile_collect's runs, one leader per group and tile): the tile maxima bound
// nothing here (two tiles' best docs may share a group), so every run key takes part.  The keys are walked in
// descending order in windows of SEL_SMEM_KEYS -- each the next keys below the last window's least, from a radix
// select over the 64-bit keys, gathered from the run prefixes (for_each_candidate<true>) and sorted -- and each window
// keeps its leaders (collapse_window) until k groups are taken.  A group's best key over the runs is its global
// leader, so the result is exact.  The hash holds <= k taken codes plus a window's 4,096 (dynamic memory,
// SEL_COLLAPSE_SMEM).  Result keys as topk_select_kernel writes them, 0 past the last leader.
#define SEL_COLLAPSE_HASH_BITS 13
#define SEL_COLLAPSE_SMEM ((2u << SEL_COLLAPSE_HASH_BITS) * sizeof(u32))   // 64 KB
__global__ void __launch_bounds__(SEL_THREADS)
topk_collapse_kernel(TopkCtx t, const u32 *__restrict__ groups, u64 doc_base, u64 *__restrict__ out_keys,
                     u32 *windows) {
    __shared__ u64 s_keys[SEL_SMEM_KEYS];
    __shared__ u32 s_hist[256];
    __shared__ u64 s_prefix;
    __shared__ u32 s_krem, s_n, s_m;
    extern __shared__ u32 s_hash[];
    const u32 q = blockIdx.x, k = t.k;
    u64 *__restrict__ out = out_keys + (u64)q * k;
    u64 hi = ~0ull;                                                  // keys below hi are still to walk
    auto visit = [&](auto f) {
        for_each_candidate<true>(t, q, 1u, [&](u64 key) {
            if (key < hi) f(key);
        });
    };
    collapse_hash_clear(s_hash, SEL_COLLAPSE_HASH_BITS);
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    u32 mine = 0;
    visit([&](u64) { mine++; });
    mine = __reduce_add_sync(0xffffffffu, mine);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(&s_n, mine);
    __syncthreads();
    // CTA-uniform: s_n is written only before the barrier above; each window gathers through its own counter s_m, as
    // collapse_tile_collect does (a shared counter cleared here would race with this read when no radix select runs)
    u32 n = s_n, taken = 0, w = 0;
    while (taken < k && n > 0) {
        const u32 m = min(n, (u32)SEL_SMEM_KEYS);
        const u64 lo = n > m ? radix_kth_largest<u64, 64>(m, s_hist, &s_prefix, &s_krem, visit) : 0ull;
        if (threadIdx.x == 0) s_m = 0;
        __syncthreads();
        for_each_candidate<true>(t, q, max((u32)(lo >> 32), 1u), [&](u64 key) {
            if (key >= lo && key < hi) s_keys[atomicAdd(&s_m, 1u)] = key;
        });
        u32 n2 = 1;
        while (n2 < m) n2 <<= 1;
        __syncthreads();
        for (u32 i = m + threadIdx.x; i < n2; i += blockDim.x) s_keys[i] = 0ull;
        __syncthreads();
        bitonic_sort_desc_smem(s_keys, n2);
        taken = collapse_window<SEL_THREADS, SEL_SMEM_KEYS / SEL_THREADS>(
            s_keys, m, groups, s_hash, SEL_COLLAPSE_HASH_BITS, taken, k,
            [&](u32 r, u64 key) { out[r] = key - doc_base; });      // (~local) - base == ~(local + base)
        n -= m;
        hi = lo;
        w++;
    }
    for (u32 i = taken + threadIdx.x; i < k; i += blockDim.x) out[i] = 0ull;
    if (threadIdx.x == 0 && w > 1) atomicAdd(windows, w - 1);
}

int launch_topk_collapse(sa_index *ix, const TopkCtx &t, u32 n_queries, u64 doc_base, const u32 *groups,
                         u64 *d_out_keys, u32 *d_windows) {
    if (n_queries == 0) return SA_OK;
    SA_CHECK(t.k <= SA_TOPK_DEEP_MAX && t.slots == t.k, "collapse: k = %u, %u slots", t.k, t.slots);
    SA_CUDA(cudaFuncSetAttribute(topk_collapse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)SEL_COLLAPSE_SMEM));
    KernelTimer tm(ix, 1);
    topk_collapse_kernel<<<n_queries, SEL_THREADS, SEL_COLLAPSE_SMEM, ix->stream>>>(t, groups, doc_base, d_out_keys,
                                                                                     d_windows);
    SA_CUDA(cudaGetLastError());
    tm.stop();
    ix->stats.topk_kernel_launches++;
    ix->stats.total_launches++;
    return SA_OK;
}

typedef unsigned __int128 u128;

// The exact top k of a query whose candidates carry a float32 PROXY of a float64 score (collect_tile_f64: classic
// similarity, edismax): the candidate key is proxy_bits << 32 | ~position as usual and tile_d[] holds the float64 score
// bits of the same slot.  The proxy is monotone but not injective, so distinct scores can share it; the tiles kept
// EVERY position at or above their bound (no tie cut), hence every position whose proxy is >= the k-th largest
// proxy P_k is a candidate, and the true top k lies among them (a position below P_k has k better ones).
//   A. thr = k-th largest tile maximum (<= P_k: the maxima belong to distinct positions);
//   B. over the candidates with proxy >= thr, a radix select of the 96-bit key (score bits, ~position) -- exact
//      float64 order, ties to the lower position -- gives the k-th key; the keys >= it are the result, ranked.
// Result: out_keys as topk_select_kernel writes them (ids only) and out_scores the float64 scores; empty = 0 / 0.
__global__ void __launch_bounds__(SEL_THREADS)
topk_select_f64_kernel(TopkCtx t, const u64 *__restrict__ tile_d, u64 doc_base, u64 *__restrict__ out_keys,
                       double *__restrict__ out_scores, const u32 *__restrict__ out_index) {
    __shared__ u32 s_hist[256];
    __shared__ u32 s_krem, s_n;
    __shared__ u32 s_thr;
    __shared__ u128 s_prefix;
    extern __shared__ __align__(16) unsigned char s_dyn[];
    u128 *s_win = reinterpret_cast<u128 *>(s_dyn);                 // [k], launch_topk_select_f64
    const u32 q = blockIdx.x, k = t.k, T = t.n_tiles;
    const u32 *tmax = t.tile_max + (u64)q * T;
    u32 thr = radix_kth_largest<u32, 32>(k, s_hist, &s_thr, &s_krem, [&](auto f) {
        for (u32 tile = threadIdx.x; tile < T; tile += blockDim.x) f(tmax[tile]);
    });
    if (thr == 0) thr = 1;
    const u64 *d = tile_d + (u64)q * T * t.slots;
    const u64 *cand = t.tile_cand + (u64)q * T * t.slots;
    const u32 *cnt = t.tile_cnt + (u64)q * T;
    auto survivors = [&](auto f) {
        for (u32 tile = threadIdx.x; tile < T; tile += blockDim.x) {
            if (tmax[tile] < thr) continue;
            const u64 base = (u64)tile * t.slots;
            for (u32 j = 0; j < cnt[tile]; j++)
                if ((u32)(cand[base + j] >> 32) >= thr) f(((u128)d[base + j] << 32) | (u32)cand[base + j]);
        }
    };
    const u128 kth = radix_kth_largest<u128, 96>(k, s_hist, &s_prefix, &s_krem, survivors);
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    survivors([&](u128 key) {                   // keys are distinct (positions are): at most k reach kth
        if (key >= kth) {
            const u32 slot = atomicAdd(&s_n, 1u);
            if (slot < k) s_win[slot] = key;
        }
    });
    __syncthreads();
    const u32 n = min(s_n, k);
    const u64 row = out_index ? out_index[q] : q;
    for (u32 i = threadIdx.x; i < k; i += blockDim.x) {
        if (i < n) {
            const u128 key = s_win[i];
            u32 rank = 0;
            for (u32 j = 0; j < n; j++) rank += s_win[j] > key;
            out_keys[row * k + rank] = ((u64)1 << 32) | (u64)((u32)key - (u32)doc_base);   // (~local) - base == ~(local + base)
            out_scores[row * k + rank] = __longlong_as_double((long long)(u64)(key >> 32));
        } else {
            out_keys[row * k + i] = 0ull;
            out_scores[row * k + i] = 0.0;
        }
    }
}

int launch_topk_select_f64(sa_index *ix, const TopkCtx &t, const u64 *d_tile_d, u32 n_queries, u64 doc_base,
                           u64 *d_out_keys, double *d_out_scores, const u32 *d_out_index) {
    if (n_queries == 0) return SA_OK;
    KernelTimer tm(ix, 1);
    SA_CHECK(t.k <= SA_TOPK_DEEP_MAX, "k = %u is above %d", t.k, SA_TOPK_DEEP_MAX);
    topk_select_f64_kernel<<<n_queries, SEL_THREADS, (size_t)t.k * sizeof(u128), ix->stream>>>(
        t, d_tile_d, doc_base, d_out_keys, d_out_scores, d_out_index);
    SA_CUDA(cudaGetLastError());
    tm.stop();
    ix->stats.topk_kernel_launches++;
    ix->stats.total_launches++;
    return SA_OK;
}

// Merge per-shard top-k lists after the all-gather: in[r][q][k] -> out[q][k].
__global__ void __launch_bounds__(SEL_THREADS)
topk_merge_kernel(const u64 *__restrict__ in, u64 rank_stride, u32 world, u32 n_queries, u32 k, u64 *__restrict__ out) {
    __shared__ u64 s_keys[SEL_SMEM_KEYS];
    const u32 q = blockIdx.x;
    const u32 n = world * k;
    u32 n2 = 2;
    while (n2 < n) n2 <<= 1;
    for (u32 i = threadIdx.x; i < n2; i += blockDim.x) {
        u64 v = 0ull;
        if (i < n) {
            u32 r = i / k, j = i % k;
            v = in[(u64)r * rank_stride + (u64)q * k + j];
        }
        s_keys[i] = v;
    }
    __syncthreads();
    bitonic_sort_desc_smem(s_keys, n2);
    for (u32 i = threadIdx.x; i < k; i += blockDim.x) out[(u64)q * k + i] = s_keys[i];
}

// topk_merge_kernel for world * k > SEL_SMEM_KEYS (k > SA_TOPK_MAX): every rank's list is sorted descending, 0-padded,
// and its non-zero keys are distinct from every other rank's (the ranks own disjoint doc ranges), so key i of rank r
// lands at i + (keys greater than it in the other lists), found by binary search: a merge without shared memory.
__global__ void __launch_bounds__(SEL_THREADS)
topk_merge_ranked_kernel(const u64 *__restrict__ in, u64 rank_stride, u32 world, u32 k, u64 *__restrict__ out) {
    const u32 q = blockIdx.x;
    for (u32 i = threadIdx.x; i < k; i += blockDim.x) out[(u64)q * k + i] = 0ull;
    __syncthreads();
    for (u32 x = threadIdx.x; x < world * k; x += blockDim.x) {
        const u32 r = x / k, i = x % k;
        const u64 key = in[(u64)r * rank_stride + (u64)q * k + i];
        if (key == 0ull) continue;
        u32 pos = i;
        for (u32 o = 0; o < world && pos < k; o++) {
            if (o == r) continue;
            const u64 *l = in + (u64)o * rank_stride + (u64)q * k;
            u32 lo = 0, hi = k;                                      // first index whose key is below `key`
            while (lo < hi) {
                const u32 mid = (lo + hi) >> 1;
                if (l[mid] > key) lo = mid + 1; else hi = mid;
            }
            pos += lo;
        }
        if (pos < k) out[(u64)q * k + pos] = key;
    }
}

int launch_topk_select(sa_index *ix, const TopkCtx &t, u32 n_queries, u64 doc_base, u64 *d_out_keys,
                       const u32 *d_out_index) {
    if (n_queries == 0) return SA_OK;
    KernelTimer tm(ix, 1);
    if (t.k > SA_TOPK_MAX)
        topk_select_kernel<true><<<n_queries, SEL_THREADS, 0, ix->stream>>>(t, doc_base, d_out_keys, d_out_index);
    else
        topk_select_kernel<false><<<n_queries, SEL_THREADS, 0, ix->stream>>>(t, doc_base, d_out_keys, d_out_index);
    SA_CUDA(cudaGetLastError());
    tm.stop();
    ix->stats.topk_kernel_launches++;
    ix->stats.total_launches++;
    return SA_OK;
}

int launch_topk_merge(sa_index *ix, const u64 *d_in, u64 rank_stride, u32 world, u32 n_queries, u32 k, u64 *d_out) {
    if (n_queries == 0) return SA_OK;
    SA_CHECK(k <= SA_TOPK_DEEP_MAX, "k = %u is above %d for the merge kernel", k, SA_TOPK_DEEP_MAX);
    KernelTimer tm(ix, 1);
    if ((u64)world * k <= SEL_SMEM_KEYS)
        topk_merge_kernel<<<n_queries, SEL_THREADS, 0, ix->stream>>>(d_in, rank_stride, world, n_queries, k, d_out);
    else
        topk_merge_ranked_kernel<<<n_queries, SEL_THREADS, 0, ix->stream>>>(d_in, rank_stride, world, k, d_out);
    SA_CUDA(cudaGetLastError());
    tm.stop();
    ix->stats.topk_kernel_launches++;
    ix->stats.total_launches++;
    return SA_OK;
}

// a tile keeps up to 4 * k docs at or above its bound (four docs per thread on the dense tf-table path) plus ties; a
// deep tile (k > SA_TOPK_MAX) keeps at most k
u32 sa_topk_slots(u32 k) { return k > SA_TOPK_MAX ? k : k <= 16 ? 128u : 256u; }

extern "C" int sa_topk_merge(sa_index *ix, const uint64_t *lists, uint32_t world, uint32_t n_queries, uint32_t k,
                             uint64_t *out) {
    SA_CHECK(ix && (n_queries == 0 || (lists && out)), "NULL argument");
    SA_CHECK(world >= 1 && k >= 1 && k <= SA_TOPK_DEEP_MAX, "world >= 1 and k in [1, %d]", SA_TOPK_DEEP_MAX);
    if (n_queries == 0) return SA_OK;
    std::lock_guard<std::mutex> g(ix->mu);
    SA_CUDA(cudaSetDevice(ix->device));
    const size_t n_in = (size_t)world * n_queries * k, n_out = (size_t)n_queries * k;
    DevBuf buf;
    int rc;
    if ((rc = buf.reserve((n_in + n_out) * sizeof(u64)))) return rc;
    SA_CUDA(cudaMemcpyAsync(buf.p, lists, n_in * sizeof(u64), cudaMemcpyHostToDevice, ix->stream));
    if ((rc = launch_topk_merge(ix, buf.as<u64>(), (u64)n_queries * k, world, n_queries, k, buf.as<u64>() + n_in)))
        return rc;
    SA_CUDA(cudaMemcpyAsync(out, buf.as<u64>() + n_in, n_out * sizeof(u64), cudaMemcpyDeviceToHost, ix->stream));
    SA_CUDA(cudaStreamSynchronize(ix->stream));
    return SA_OK;
}
