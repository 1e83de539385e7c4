// sa_feature.cu -- per-document columns of an index: feature columns (sa_index_set_feature), read by the feature
// clauses of the batched boolean queries, and facet columns (sa_index_set_facet), read by their counting pass
// (sa_bool.cu).
//
// A feature column is stored as float[padded n_docs], zero past n_docs, so the tile fold's float4 loads of a whole
// tile need no bounds test.  Beside it, one u32 flag per (slot, tile): whether any value of the tile is > 0.  The fold
// takes a feature clause as present in a tile iff its flag is set, as it takes a term clause present where its list
// has a doc, so min-should-match and MUST pruning skip the tiles where the feature is absent.
//
// A facet column is stored as uint16[padded n_docs], 0xFFFF for "no value" and past n_docs, so the counting pass
// reads a thread's four docs as one 8-byte load with no bounds test.
#include <cmath>

#include "sa_term.cuh"

// One CTA per tile: flags[tile] = 1 iff any of the tile's values is > 0.
__global__ void __launch_bounds__(SA_TERM_THREADS) feature_tiles_kernel(const float *__restrict__ values,
                                                                         u32 *__restrict__ flags) {
    const float4 *v4 = reinterpret_cast<const float4 *>(values + (u64)blockIdx.x * SA_TILE_DOCS);
    bool any = false;
#pragma unroll
    for (int j = 0; j < SA_TILE_DOCS / SA_TERM_THREADS / 4; j++) {
        const float4 x = __ldg(v4 + threadIdx.x + j * SA_TERM_THREADS);
        any = any || x.x > 0.0f || x.y > 0.0f || x.z > 0.0f || x.w > 0.0f;
    }
    const int found = __syncthreads_or(any);
    if (threadIdx.x == 0) flags[blockIdx.x] = found ? 1u : 0u;
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
    // into a new buffer, which replaces the slot's once it is filled: a failure leaves the slot as it was
    DevBuf col;
    if ((rc = col.allocate(std::max<size_t>(padded * sizeof(float), 16)))) return rc;
    SA_CUDA(cudaMemsetAsync(col.p, 0, col.cap, ix->stream));
    if (n_values) {
        SA_CUDA(cudaMemcpyAsync(col.p, values, n_values * sizeof(float), cudaMemcpyHostToDevice, ix->stream));
    }
    u32 *flags = ix->d_feature_tiles.as<u32>() + (size_t)slot * n_tiles;
    if (n_tiles) {
        feature_tiles_kernel<<<n_tiles, SA_TERM_THREADS, 0, ix->stream>>>(col.as<float>(), flags);
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
    DevBuf d;
    int rc;
    if ((rc = d.allocate(col.size() * sizeof(uint16_t)))) return rc;
    SA_CUDA(cudaMemcpyAsync(d.p, col.data(), col.size() * sizeof(uint16_t), cudaMemcpyHostToDevice, ix->stream));
    SA_CUDA(cudaStreamSynchronize(ix->stream));     // `col` is a local
    ix->d_facets[slot] = std::move(d);
    ix->facet_buckets[slot] = n_buckets;
    ix->facet_set |= 1u << slot;
    return SA_OK;
}
