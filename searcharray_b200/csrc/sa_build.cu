// sa_build.cu -- index build on the device (SURVEY.md section 8f-4).
//
// Replaces the numpy half of the reference's index build AFTER tokenisation (which stays on the host: it is a
// Python loop over strings, searcharray/indexing.py:64-98):
//   _invert_docs_terms / _lex_sort     searcharray/indexing.py:101-115   stable sort of the (term, doc, posn) triples by term
//   RoaringishEncoder.encode           searcharray/roaringish/roaringish.py:93-142   header = doc << 36 | (posn // 18) << 18,
//                                      one bit per posn % 18, np.bitwise_or.reduceat over equal headers
//   PosnBitArrayFromFlatBuilder.build  searcharray/phrase/middle_out.py (term boundaries -> ArrayDict slices)
//
// Triples arrive in document order (docs ascending, positions ascending inside a doc), exactly as _gather_tokens
// emits them.  The only sort needed is the STABLE sort by term id: a least-significant-digit radix sort of
// (term id, original index) pairs -- cub::DeviceRadixSort, NVIDIA's library sort shipped with the CUDA toolkit, used
// as a plain library primitive the way a BLAS call would be; everything around it (header / bit construction,
// segmented OR by head flags, compaction, term slices) is this file's kernels.  The head flags are ranked by
// sa_scan.cuh's `scan_flags`, the same device-wide scan the set ops compact with.
#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <vector>

#include "sa_common.cuh"
#include "sa_scan.cuh"

namespace {

__global__ void iota_kernel(u32 *__restrict__ a, u64 n) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[i] = (u32)i;
}

// sorted position i: term = terms_sorted[i], triple = original index order[i].  A position starts a WORD when its
// (term, doc, posn // 18) differs from the previous position's; the head ORs the bits of its run (<= 18 entries:
// distinct positions of one block; repeated positions just OR the same bit again).
__global__ void word_head_kernel(const u32 *__restrict__ terms_sorted, const u32 *__restrict__ order,
                                 const u32 *__restrict__ docs, const u32 *__restrict__ posns, u64 n,
                                 u32 *__restrict__ head) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool h = i == 0;
    if (!h) {
        const u32 a = order[i], b = order[i - 1];
        h = terms_sorted[i] != terms_sorted[i - 1] || docs[a] != docs[b] || posns[a] / SA_LSB_BITS != posns[b] / SA_LSB_BITS;
    }
    head[i] = h ? 1u : 0u;
}

// every head writes its word at its rank; the first word of a term records the term's slice start, and every
// head bumps its term's length
__global__ void word_write_kernel(const u32 *__restrict__ terms_sorted, const u32 *__restrict__ order,
                                  const u32 *__restrict__ docs, const u32 *__restrict__ posns, u64 n,
                                  const u32 *__restrict__ head, const u32 *__restrict__ offs,
                                  u64 *__restrict__ words, u64 *__restrict__ term_off, u64 *__restrict__ term_len) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || !head[i]) return;
    const u32 rank = offs[i];
    const u32 term = terms_sorted[i];
    const u32 a = order[i];
    const u32 doc = docs[a], blk = posns[a] / SA_LSB_BITS;
    u64 bits = 0;
    for (u64 j = i; j < n; j++) {
        if (j > i && head[j]) break;
        bits |= 1ull << (posns[order[j]] % SA_LSB_BITS);
    }
    words[rank] = ((u64)doc << SA_KEY_SHIFT) | ((u64)blk << SA_LSB_BITS) | bits;
    if (i == 0 || terms_sorted[i - 1] != term) term_off[term] = rank;
    atomicAdd((unsigned long long *)&term_len[term], 1ull);
}

}  // namespace

// (term, doc, posn) triples in document order -> the index's upload format: posting words of all terms
// concatenated in term-id order, sorted and header-unique inside a term, plus every term's slice.
// words_out needs room for n_triples words; term_off_out / term_len_out have n_terms entries (absent terms: 0, 0).
extern "C" int sa_op_build_index(const uint32_t *term_ids, const uint32_t *doc_ids, const uint32_t *posns, uint64_t n_triples,
                                 uint32_t n_terms, int device, uint64_t *words_out, uint64_t *n_words_out,
                                 uint64_t *term_off_out, uint64_t *term_len_out) {
    SA_CHECK(n_words_out && (n_terms == 0 || (term_off_out && term_len_out)), "NULL argument");
    *n_words_out = 0;
    for (u32 t = 0; t < n_terms; t++) { term_off_out[t] = 0; term_len_out[t] = 0; }
    if (n_triples == 0) return SA_OK;
    SA_CHECK(term_ids && doc_ids && posns && words_out, "NULL argument");
    // cub's sort counts items in an int
    SA_CHECK(n_triples < (1ull << 31), "too many tokens for one build call (batch them like the reference's batch_size)");
    // every triple must fit the word it lands in: a term slot, a 28-bit doc id, an 18-bit block
    for (u64 i = 0; i < n_triples; i++) {
        SA_CHECK(term_ids[i] < n_terms, "triple %llu: term id %u >= n_terms %u", (unsigned long long)i, term_ids[i], n_terms);
        SA_CHECK(doc_ids[i] < (1u << 28), "triple %llu: doc id %u exceeds the 28-bit key space", (unsigned long long)i,
                 doc_ids[i]);
        SA_CHECK(posns[i] < SA_LSB_BITS * SA_ONE_BLOCK, "triple %llu: position %u exceeds %llu", (unsigned long long)i,
                 posns[i], (unsigned long long)(SA_LSB_BITS * SA_ONE_BLOCK - 1));
    }
    SA_CUDA(cudaSetDevice(device));
    const u64 n = n_triples;
    DevMem m;
    u32 *d_t = m.alloc<u32>(n), *d_ts = m.alloc<u32>(n), *d_i = m.alloc<u32>(n), *d_is = m.alloc<u32>(n);
    u32 *d_doc = m.alloc<u32>(n), *d_pos = m.alloc<u32>(n), *d_head = m.alloc<u32>(n), *d_offs = m.alloc<u32>(n);
    u64 *d_words = m.alloc<u64>(n), *d_toff = m.alloc<u64>(n_terms), *d_tlen = m.alloc<u64>(n_terms);
    if (!(d_t && d_ts && d_i && d_is && d_doc && d_pos && d_head && d_offs && d_words && d_toff && d_tlen)) {
        sa_set_error("device allocation failed");
        return SA_ERR_NOMEM;
    }
    SA_CUDA(cudaMemcpy(d_t, term_ids, n * sizeof(u32), cudaMemcpyHostToDevice));
    SA_CUDA(cudaMemcpy(d_doc, doc_ids, n * sizeof(u32), cudaMemcpyHostToDevice));
    SA_CUDA(cudaMemcpy(d_pos, posns, n * sizeof(u32), cudaMemcpyHostToDevice));
    SA_CUDA(cudaMemset(d_toff, 0, std::max<u32>(n_terms, 1) * sizeof(u64)));
    SA_CUDA(cudaMemset(d_tlen, 0, std::max<u32>(n_terms, 1) * sizeof(u64)));
    const unsigned blocks = (unsigned)((n + 255) / 256);
    iota_kernel<<<blocks, 256>>>(d_i, n);
    // stable LSD radix sort by term id (only the bits a term id can use)
    int end_bit = 1;
    while (end_bit < 32 && (1ull << end_bit) < (u64)std::max<u32>(n_terms, 2)) end_bit++;
    size_t tmp_bytes = 0;
    SA_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, d_t, d_ts, d_i, d_is, (int)n, 0, end_bit));
    void *d_tmp = m.alloc<char>(tmp_bytes);
    if (!d_tmp) { sa_set_error("device allocation failed"); return SA_ERR_NOMEM; }
    SA_CUDA(cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, d_t, d_ts, d_i, d_is, (int)n, 0, end_bit));
    word_head_kernel<<<blocks, 256>>>(d_ts, d_is, d_doc, d_pos, n, d_head);
    u64 total = 0;
    int rc = scan_flags(m, d_head, d_offs, n, &total, 0);
    if (rc) return rc;
    word_write_kernel<<<blocks, 256>>>(d_ts, d_is, d_doc, d_pos, n, d_head, d_offs, d_words, d_toff, d_tlen);
    SA_CUDA(cudaGetLastError());
    SA_CUDA(cudaMemcpy(words_out, d_words, (size_t)total * sizeof(u64), cudaMemcpyDeviceToHost));
    if (n_terms) {
        SA_CUDA(cudaMemcpy(term_off_out, d_toff, n_terms * sizeof(u64), cudaMemcpyDeviceToHost));
        SA_CUDA(cudaMemcpy(term_len_out, d_tlen, n_terms * sizeof(u64), cudaMemcpyDeviceToHost));
    }
    *n_words_out = total;
    return SA_OK;
}
