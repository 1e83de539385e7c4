// sa_feature.cu -- per-document columns of an index: feature columns (sa_index_set_feature), read by the feature
// and range clauses of the batched boolean queries, and facet columns (sa_index_set_facet), read by their counting
// pass and their In clauses (sa_bool.cu).
//
// A feature column is stored as float[padded n_docs], zero past n_docs, so the tile fold's float4 loads of a whole
// tile need no bounds test.  Beside it, one u32 flag per (slot, tile): whether any value of the tile is > 0.  The fold
// takes a feature clause as present in a tile iff its flag is set, as it takes a term clause present where its list
// has a doc, so min-should-match and MUST pruning skip the tiles where the feature is absent.  And per (slot, tile)
// the min and max of the tile's values > 0: a range clause is present iff the flag is set and [min, max] meets it.
//
// A facet column is stored as uint16[padded n_docs], 0xFFFF for "no value" and past n_docs, so the counting pass
// reads a thread's four docs as one 8-byte load with no bounds test.  Beside it, per tile, the set of codes present
// (1,024 bits): an In clause is present in a tile iff its codes meet that set.
//
// A group column (sa_index_set_group) is stored as u32[padded n_docs], SA_GROUP_NONE for "no group" and past n_docs;
// the collapsed top-k reads it by doc id, for the docs of its windows only.
#include <climits>
#include <cmath>

#include "sa_term.cuh"

// One CTA per tile: flags[tile] = 1 iff any of the tile's values is > 0, and bounds[tile] = (min, max) of those
// values ((+inf, 0) where there is none).  Values are >= 0, so the bits of the positive ones order as the values do.
__global__ void __launch_bounds__(SA_TERM_THREADS) feature_tiles_kernel(const float *__restrict__ values,
                                                                         u32 *__restrict__ flags,
                                                                         float2 *__restrict__ bounds) {
    __shared__ u32 s_lo[SA_TERM_THREADS / 32], s_hi[SA_TERM_THREADS / 32];
    const float4 *v4 = reinterpret_cast<const float4 *>(values + (u64)blockIdx.x * SA_TILE_DOCS);
    u32 lo = 0x7F800000u, hi = 0;          // +inf, +0
#pragma unroll
    for (int j = 0; j < SA_TILE_DOCS / SA_TERM_THREADS / 4; j++) {
        const float4 x = __ldg(v4 + threadIdx.x + j * SA_TERM_THREADS);
        const float xs[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int e = 0; e < 4; e++) {
            if (!(xs[e] > 0.0f)) continue;
            lo = min(lo, __float_as_uint(xs[e]));
            hi = max(hi, __float_as_uint(xs[e]));
        }
    }
    lo = __reduce_min_sync(0xFFFFFFFFu, lo);
    hi = __reduce_max_sync(0xFFFFFFFFu, hi);
    if ((threadIdx.x & 31) == 0) {
        s_lo[threadIdx.x >> 5] = lo;
        s_hi[threadIdx.x >> 5] = hi;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < SA_TERM_THREADS / 32; w++) {
            lo = min(lo, s_lo[w]);
            hi = max(hi, s_hi[w]);
        }
        flags[blockIdx.x] = hi != 0 ? 1u : 0u;
        bounds[blockIdx.x] = make_float2(__uint_as_float(lo), __uint_as_float(hi));
    }
}

// One CTA per tile: sets[tile * SA_FACET_SET_WORDS + w] bit b set iff code 32 w + b is some doc's of the tile.
__global__ void __launch_bounds__(SA_TERM_THREADS) facet_tiles_kernel(const unsigned short *__restrict__ codes,
                                                                       u32 *__restrict__ sets) {
    __shared__ u32 s_set[SA_FACET_SET_WORDS];
    if (threadIdx.x < SA_FACET_SET_WORDS) s_set[threadIdx.x] = 0;
    __syncthreads();
    const ushort4 *c4 = reinterpret_cast<const ushort4 *>(codes + (u64)blockIdx.x * SA_TILE_DOCS);
#pragma unroll
    for (int j = 0; j < SA_TILE_DOCS / SA_TERM_THREADS / 4; j++) {
        const ushort4 c = __ldg(c4 + threadIdx.x + j * SA_TERM_THREADS);
        const unsigned short cs[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
        for (int e = 0; e < 4; e++)
            if (cs[e] != SA_FACET_NONE) atomicOr(s_set + (cs[e] >> 5), 1u << (cs[e] & 31));
    }
    __syncthreads();
    if (threadIdx.x < SA_FACET_SET_WORDS) sets[(u64)blockIdx.x * SA_FACET_SET_WORDS + threadIdx.x] = s_set[threadIdx.x];
}

extern "C" int sa_index_set_feature(sa_index *ix, uint32_t slot, const float *values, uint64_t n_values) {
    SA_CHECK(ix && (values || n_values == 0), "NULL argument");
    SA_CHECK(slot < SA_MAX_FEATURES, "feature slot %u out of range (%d slots)", slot, SA_MAX_FEATURES);
    std::lock_guard<std::mutex> g(ix->mu);
    SA_CHECK(n_values == ix->n_docs, "a feature has one value per doc: %llu values for %llu docs",
             (unsigned long long)n_values, (unsigned long long)ix->n_docs);
    SA_CHECK(ix->n_terms < SA_FEATURE_TERM_BASE, "an index of %u terms reaches the feature term ids", ix->n_terms);
    for (u64 i = 0; i < n_values; i++)
        SA_CHECK(std::isfinite(values[i]) && values[i] >= 0.0f, "feature value %llu is not finite and >= 0",
                 (unsigned long long)i);
    SA_CUDA(cudaSetDevice(ix->device));
    const u32 n_tiles = sa_n_tiles(ix->n_docs);
    const u64 padded = sa_padded_docs(ix->n_docs);
    int rc;
    if (!ix->d_feature_tiles.p) {
        if ((rc = ix->d_feature_tiles.allocate(std::max<size_t>((size_t)SA_MAX_FEATURES * n_tiles * sizeof(u32), 16))))
            return rc;
        SA_CUDA(cudaMemsetAsync(ix->d_feature_tiles.p, 0, ix->d_feature_tiles.cap, ix->stream));
    }
    if (!ix->d_feature_bounds.p) {
        if ((rc = ix->d_feature_bounds.allocate(std::max<size_t>((size_t)SA_MAX_FEATURES * n_tiles * sizeof(float2), 16))))
            return rc;
        SA_CUDA(cudaMemsetAsync(ix->d_feature_bounds.p, 0, ix->d_feature_bounds.cap, ix->stream));
    }
    // into a new buffer, which replaces the slot's once it is filled: a failure leaves the slot as it was
    DevBuf col;
    if ((rc = col.allocate(std::max<size_t>(padded * sizeof(float), 16)))) return rc;
    SA_CUDA(cudaMemsetAsync(col.p, 0, col.cap, ix->stream));
    if (n_values) {
        SA_CUDA(cudaMemcpyAsync(col.p, values, n_values * sizeof(float), cudaMemcpyHostToDevice, ix->stream));
    }
    u32 *flags = ix->d_feature_tiles.as<u32>() + (size_t)slot * n_tiles;
    if (n_tiles) {
        feature_tiles_kernel<<<n_tiles, SA_TERM_THREADS, 0, ix->stream>>>(
            col.as<float>(), flags, ix->d_feature_bounds.as<float2>() + (size_t)slot * n_tiles);
        SA_CUDA(cudaGetLastError());
        ix->stats.total_launches++;
    }
    SA_CUDA(cudaStreamSynchronize(ix->stream));     // `values` is borrowed for the call only
    ix->d_features[slot] = std::move(col);
    ix->feature_set |= 1u << slot;
    return SA_OK;
}

extern "C" int sa_index_set_facet(sa_index *ix, uint32_t slot, const int32_t *codes, uint64_t n_values,
                                  uint32_t n_buckets) {
    SA_CHECK(ix && (codes || n_values == 0), "NULL argument");
    SA_CHECK(slot < SA_MAX_FACETS, "facet slot %u out of range (%d slots)", slot, SA_MAX_FACETS);
    SA_CHECK(n_buckets >= 1 && n_buckets <= SA_FACET_MAX_BUCKETS, "a facet has 1 to %d buckets, not %u",
             SA_FACET_MAX_BUCKETS, n_buckets);
    std::lock_guard<std::mutex> g(ix->mu);
    SA_CHECK(n_values == ix->n_docs, "a facet has one code per doc: %llu codes for %llu docs",
             (unsigned long long)n_values, (unsigned long long)ix->n_docs);
    const u64 padded = sa_padded_docs(ix->n_docs);
    std::vector<uint16_t> col(std::max<u64>(padded, 4), SA_FACET_NONE);
    for (u64 i = 0; i < n_values; i++) {
        SA_CHECK(codes[i] >= -1 && codes[i] < (int32_t)n_buckets, "facet code %llu (%d) is not -1 or in [0, %u)",
                 (unsigned long long)i, codes[i], n_buckets);
        if (codes[i] >= 0) col[i] = (uint16_t)codes[i];
    }
    SA_CUDA(cudaSetDevice(ix->device));
    // into a new buffer, which replaces the slot's once it is filled: a failure leaves the slot as it was
    const u32 n_tiles = sa_n_tiles(ix->n_docs);
    DevBuf d, sets;
    int rc;
    if ((rc = d.allocate(col.size() * sizeof(uint16_t))) ||
        (rc = sets.allocate(std::max<size_t>((size_t)n_tiles * SA_FACET_SET_WORDS * sizeof(u32), 16))))
        return rc;
    SA_CUDA(cudaMemcpyAsync(d.p, col.data(), col.size() * sizeof(uint16_t), cudaMemcpyHostToDevice, ix->stream));
    if (n_tiles) {
        facet_tiles_kernel<<<n_tiles, SA_TERM_THREADS, 0, ix->stream>>>(d.as<unsigned short>(), sets.as<u32>());
        SA_CUDA(cudaGetLastError());
        ix->stats.total_launches++;
    }
    SA_CUDA(cudaStreamSynchronize(ix->stream));     // `col` is a local
    ix->d_facets[slot] = std::move(d);
    ix->d_facet_tiles[slot] = std::move(sets);
    ix->facet_buckets[slot] = n_buckets;
    ix->facet_set |= 1u << slot;
    return SA_OK;
}

extern "C" int sa_index_set_group(sa_index *ix, uint32_t slot, const int32_t *codes, uint64_t n_values) {
    SA_CHECK(ix && (codes || n_values == 0), "NULL argument");
    SA_CHECK(slot < SA_MAX_GROUPS, "group slot %u out of range (%d slots)", slot, SA_MAX_GROUPS);
    std::lock_guard<std::mutex> g(ix->mu);
    SA_CHECK(n_values == ix->n_docs, "a group column has one code per doc: %llu codes for %llu docs",
             (unsigned long long)n_values, (unsigned long long)ix->n_docs);
    std::vector<u32> col(std::max<u64>(sa_padded_docs(ix->n_docs), 4), SA_GROUP_NONE);
    for (u64 i = 0; i < n_values; i++) {
        SA_CHECK(codes[i] >= -1 && codes[i] != INT32_MAX, "group code %llu (%d) is not -1 or in [0, 2^31 - 1)",
                 (unsigned long long)i, codes[i]);
        if (codes[i] >= 0) col[i] = (u32)codes[i];
    }
    SA_CUDA(cudaSetDevice(ix->device));
    // into a new buffer, which replaces the slot's once it is filled: a failure leaves the slot as it was
    DevBuf d;
    int rc;
    if ((rc = d.allocate(col.size() * sizeof(u32)))) return rc;
    SA_CUDA(cudaMemcpyAsync(d.p, col.data(), col.size() * sizeof(u32), cudaMemcpyHostToDevice, ix->stream));
    SA_CUDA(cudaStreamSynchronize(ix->stream));     // `col` is a local
    ix->d_groups[slot] = std::move(d);
    ix->group_set |= 1u << slot;
    return SA_OK;
}
