// sa_filter.cu -- sliced arrays and position filters.
//
// Replaces RoaringishEncoder.slice + payload_slice + FilteredPosns (reference
// searcharray/roaringish/roaringish.py:245-282, roaringish_ops.pyx:46-68, phrase/middle_out.py:291-317):
// the reference materialises, per term, the sub-list of posting words whose doc is among the slice's
// rows and whose block passes the min/max_posn test, then runs the ordinary algorithms on those
// lists.  Same here: an order-preserving compaction kernel writes the filtered lists into scratch,
// the term / phrase / span kernels run on them unchanged, and a gather kernel picks the slice's rows
// out of the dense result (`phrase_freqs[self.term_mat.rows]`, postings.py:702-704).
#include <algorithm>

#include "sa_phrase.cuh"
#include "sa_scan.cuh"
#include "sa_term.cuh"

struct FilterJob { u64 src_off, src_len, dst_off, chunk_off; };   // chunk_off: first entry in the chunk-count table

#define FILT_THREADS 256
#define FILT_ITEMS 8                                  // words per thread per chunk
#define FILT_CHUNK (FILT_THREADS * FILT_ITEMS)

__device__ __forceinline__ bool filter_keep(u64 w, const unsigned char *__restrict__ row_mask, u64 doc_base, u64 n_docs,
                                            u64 pay_lo, u64 pay_hi, int use_payload) {
    bool keep = true;
    if (row_mask) {
        const u64 d = (w >> SA_KEY_SHIFT) - doc_base;
        keep = d < n_docs && row_mask[d];
    }
    if (keep && use_payload) {
        const u64 v = w & SA_MSB_MASK;                  // UNSHIFTED compare, reference roaringish_ops.pyx:55
        keep = v >= pay_lo && v <= pay_hi;
    }
    return keep;
}

// Order-preserving compaction in three steps: per-chunk keep counts, a scan of the chunk counts of
// every list, then the write pass (the keep test is cheap, so it is simply evaluated twice).
template <bool WRITE>
__global__ void __launch_bounds__(FILT_THREADS)
filter_lists_kernel(const u64 *__restrict__ words, const FilterJob *__restrict__ jobs, u64 *__restrict__ dst,
                    u32 *__restrict__ chunk_counts, const unsigned char *__restrict__ row_mask, u64 doc_base, u64 n_docs,
                    u64 pay_lo, u64 pay_hi, int use_payload) {
    __shared__ u32 s_warp[FILT_THREADS / 32];
    const FilterJob job = jobs[blockIdx.y];
    const u64 base = (u64)blockIdx.x * FILT_CHUNK;
    if (base >= job.src_len) return;
    const u64 *__restrict__ src = words + job.src_off;
    const unsigned tid = threadIdx.x;
    // thread t owns words base + t*ITEMS .. +ITEMS-1 (contiguous: the output order is the thread order)
    u64 w[FILT_ITEMS];
    u32 keep_bits = 0;
#pragma unroll
    for (int j = 0; j < FILT_ITEMS; j++) {
        const u64 i = base + (u64)tid * FILT_ITEMS + j;
        w[j] = 0;
        if (i < job.src_len) {
            w[j] = src[i];
            if (filter_keep(w[j], row_mask, doc_base, n_docs, pay_lo, pay_hi, use_payload)) keep_bits |= 1u << j;
        }
    }
    u32 tot;
    const u32 off = block_exclusive_sum<FILT_THREADS>((u32)__popc(keep_bits), s_warp, tot);
    if (!WRITE) {
        if (tid == 0) chunk_counts[job.chunk_off + blockIdx.x] = tot;
        return;
    }
    u64 *__restrict__ out = dst + job.dst_off + chunk_counts[job.chunk_off + blockIdx.x] + off;   // scanned: exclusive offset
#pragma unroll
    for (int j = 0; j < FILT_ITEMS; j++)
        if ((keep_bits >> j) & 1u) *out++ = w[j];
}

// one CTA per list: exclusive scan of its chunk counts (in place); totals[job] = kept words
__global__ void __launch_bounds__(FILT_THREADS)
filter_scan_kernel(const FilterJob *__restrict__ jobs, u32 *__restrict__ chunk_counts, u32 *__restrict__ totals) {
    const FilterJob job = jobs[blockIdx.x];
    cta_exclusive_scan<FILT_THREADS>(chunk_counts + job.chunk_off, (u32)((job.src_len + FILT_CHUNK - 1) / FILT_CHUNK),
                                     totals + blockIdx.x);
}

__global__ void gather_rows_kernel(const float *__restrict__ dense, const u64 *__restrict__ rows, u64 n_rows,
                                   float *__restrict__ out) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_rows) out[i] = dense[rows[i]];
}

__global__ void count_docs_kernel(const u64 *__restrict__ list, u64 n, u32 *__restrict__ out) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    bool head = (i == 0) || ((list[i] >> SA_KEY_SHIFT) != (list[i - 1] >> SA_KEY_SHIFT));
    unsigned m = __ballot_sync(__activemask(), head);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(out, (u32)__popc(m));
}

// Filters the given terms' lists into ix->filt; fills offs/lens (relative to ix->filt) per term.
// d_mask: per-doc keep bytes (NULL = no doc filter).  When d_df_out is given, the number of distinct
// docs of every filtered list is also returned (PosnBitArray.docfreq on FilteredPosns).
int sa_filter_terms_mask(sa_index *ix, const uint32_t *term_ids, uint32_t n_terms, const unsigned char *d_mask,
                         u64 pay_lo, u64 pay_hi, bool use_payload, std::vector<u64> &offs, std::vector<u64> &lens,
                         std::vector<u64> *df_out) {
    std::vector<FilterJob> jobs(n_terms);
    u64 total = 0, chunks_total = 0, max_chunks = 1;
    for (u32 t = 0; t < n_terms; t++) {
        const bool known = term_ids[t] != SA_NO_TERM;
        jobs[t].src_off = known ? ix->h_off[term_ids[t]] : 0;
        jobs[t].src_len = known ? ix->h_len[term_ids[t]] : 0;
        jobs[t].dst_off = total;
        jobs[t].chunk_off = chunks_total;
        const u64 nc = (jobs[t].src_len + FILT_CHUNK - 1) / FILT_CHUNK;
        chunks_total += nc;
        max_chunks = std::max(max_chunks, nc);
        total += jobs[t].src_len + 2;
    }
    int rc;
    if ((rc = ix->filt.reserve((total + 4) * sizeof(u64)))) return rc;
    const size_t jobs_bytes = ((size_t)n_terms * sizeof(FilterJob) + 255) / 256 * 256;
    if ((rc = ix->misc.reserve(jobs_bytes + (chunks_total + 2 * (size_t)n_terms + 8) * sizeof(u32)))) return rc;
    FilterJob *d_jobs = ix->misc.as<FilterJob>();
    u32 *d_chunks = (u32 *)((char *)ix->misc.p + jobs_bytes);
    u32 *d_totals = d_chunks + chunks_total;
    u32 *d_df = d_totals + n_terms;
    SA_CUDA(cudaMemcpyAsync(d_jobs, jobs.data(), n_terms * sizeof(FilterJob), cudaMemcpyHostToDevice, ix->stream));
    dim3 grid((unsigned)max_chunks, n_terms);
    filter_lists_kernel<false><<<grid, FILT_THREADS, 0, ix->stream>>>(ix->d_words.as<u64>(), d_jobs, ix->filt.as<u64>(), d_chunks,
                                                                     d_mask, ix->doc_base, ix->n_docs, pay_lo, pay_hi,
                                                                     use_payload ? 1 : 0);
    SA_CUDA(cudaGetLastError());
    filter_scan_kernel<<<n_terms, FILT_THREADS, 0, ix->stream>>>(d_jobs, d_chunks, d_totals);
    SA_CUDA(cudaGetLastError());
    filter_lists_kernel<true><<<grid, FILT_THREADS, 0, ix->stream>>>(ix->d_words.as<u64>(), d_jobs, ix->filt.as<u64>(), d_chunks,
                                                                    d_mask, ix->doc_base, ix->n_docs, pay_lo, pay_hi,
                                                                    use_payload ? 1 : 0);
    SA_CUDA(cudaGetLastError());
    ix->stats.total_launches += 3;
    std::vector<u32> h_counts(n_terms);
    SA_CUDA(cudaMemcpyAsync(h_counts.data(), d_totals, n_terms * sizeof(u32), cudaMemcpyDeviceToHost, ix->stream));
    SA_CUDA(cudaStreamSynchronize(ix->stream));
    offs.resize(n_terms);
    lens.resize(n_terms);
    for (u32 t = 0; t < n_terms; t++) { offs[t] = jobs[t].dst_off; lens[t] = h_counts[t]; }
    if (df_out) {
        df_out->assign(n_terms, 0);
        SA_CUDA(cudaMemsetAsync(d_df, 0, n_terms * sizeof(u32), ix->stream));
        for (u32 t = 0; t < n_terms; t++) {
            if (lens[t] == 0) continue;
            count_docs_kernel<<<(unsigned)((lens[t] + 255) / 256), 256, 0, ix->stream>>>(ix->filt.as<u64>() + offs[t], lens[t], d_df + t);
            SA_CUDA(cudaGetLastError());
            ix->stats.total_launches++;
        }
        SA_CUDA(cudaMemcpyAsync(h_counts.data(), d_df, n_terms * sizeof(u32), cudaMemcpyDeviceToHost, ix->stream));
        SA_CUDA(cudaStreamSynchronize(ix->stream));
        for (u32 t = 0; t < n_terms; t++) (*df_out)[t] = h_counts[t];
    }
    return SA_OK;
}

int sa_filter_terms(sa_index *ix, const uint32_t *term_ids, uint32_t n_terms, bool use_rows,
                    u64 pay_lo, u64 pay_hi, bool use_payload, std::vector<u64> &offs, std::vector<u64> &lens) {
    return sa_filter_terms_mask(ix, term_ids, n_terms, use_rows ? ix->d_row_mask() : nullptr, pay_lo, pay_hi,
                                use_payload, offs, lens, nullptr);
}

int sa_copy_out_dense(sa_index *ix, float *out_host) {
    if (!ix->rows_active) {
        SA_CUDA(cudaMemcpyAsync(out_host, ix->dense.p, ix->n_docs * sizeof(float), cudaMemcpyDeviceToHost, ix->stream));
        SA_CUDA(cudaStreamSynchronize(ix->stream));
        return SA_OK;
    }
    int rc;
    if ((rc = ix->gather.reserve(ix->n_rows * sizeof(float) + 64))) return rc;
    gather_rows_kernel<<<(unsigned)((ix->n_rows + 255) / 256), 256, 0, ix->stream>>>(ix->dense.as<float>(), ix->d_rows(),
                                                                                   ix->n_rows, ix->gather.as<float>());
    SA_CUDA(cudaGetLastError());
    ix->stats.total_launches++;
    SA_CUDA(cudaMemcpyAsync(out_host, ix->gather.p, ix->n_rows * sizeof(float), cudaMemcpyDeviceToHost, ix->stream));
    SA_CUDA(cudaStreamSynchronize(ix->stream));
    return SA_OK;
}

extern "C" int sa_index_set_rows(sa_index *ix, const uint64_t *rows, uint64_t n_rows) {
    SA_CHECK(ix, "index is NULL");
    std::lock_guard<std::mutex> g(ix->mu);
    SA_CUDA(cudaSetDevice(ix->device));
    if (rows == nullptr) {          // clear the filter
        SA_CHECK(n_rows == 0, "rows is NULL");
        ix->n_rows = 0;
        ix->rows_active = false;
        return SA_OK;
    }
    std::vector<unsigned char> mask(ix->n_docs, 0);
    for (u64 i = 0; i < n_rows; i++) {
        SA_CHECK(rows[i] < ix->n_docs, "row %llu out of range", (unsigned long long)rows[i]);
        mask[rows[i]] = 1;
    }
    // the new filter is built aside and swapped in only once complete: a failed call leaves the previous one installed
    const size_t mask_bytes = ix->row_mask_bytes();
    DevBuf filter;
    int rc;
    if ((rc = filter.allocate(mask_bytes + std::max<u64>(n_rows, 1) * sizeof(u64)))) return rc;
    if (ix->n_docs) SA_CUDA(cudaMemcpyAsync(filter.p, mask.data(), ix->n_docs, cudaMemcpyHostToDevice, ix->stream));
    if (n_rows)
        SA_CUDA(cudaMemcpyAsync(filter.as<char>() + mask_bytes, rows, n_rows * sizeof(u64), cudaMemcpyHostToDevice, ix->stream));
    SA_CUDA(cudaStreamSynchronize(ix->stream));
    ix->row_filter = std::move(filter);
    ix->n_rows = n_rows;
    ix->rows_active = true;
    return SA_OK;
}

// ---- PosnBitArray.docfreq on FilteredPosns (quirk iii: df of the filtered postings) without materialising them.
// df = the distinct docs of the term's list whose row-mask byte is set.  Terms with a tf table have one record per
// (term, doc), so their df is the sum of mask[doc] over the records (4 bytes per doc of the list); the other terms
// count the doc-head words of their posting list that lie in the mask (8 bytes per word).  One CTA per job, integer
// sums only: the result does not depend on the launch geometry.
struct DfJob {
    u64 src_off;        // first record (d_recs) or word (d_words) of the term
    u64 begin, end;     // records: tiles [begin, end); words: list indices [begin, end)
    u64 dir_off;        // record directory of the term (records only)
    u32 slot;           // output index
    u32 recs;           // 1 = records, 0 = posting words
};
#define DF_TILES_PER_JOB 8
#define DF_WORDS_PER_JOB (FILT_THREADS * 16)

__global__ void __launch_bounds__(FILT_THREADS)
docfreq_rows_kernel(const u64 *__restrict__ words, const u32 *__restrict__ recs, const u32 *__restrict__ rec_dir,
                    const DfJob *__restrict__ jobs, const unsigned char *__restrict__ row_mask, u64 doc_base, u64 n_docs,
                    unsigned long long *__restrict__ df) {
    const DfJob job = jobs[blockIdx.x];
    u32 cnt = 0;
    if (job.recs) {
        const u32 *__restrict__ r = recs + job.src_off;
        const u32 *__restrict__ dir = rec_dir + job.dir_off;
        for (u64 tile = job.begin; tile < job.end; tile++) {
            const u32 lo = __ldg(dir + tile), hi = __ldg(dir + tile + 1);
            const unsigned char *__restrict__ m = row_mask + tile * SA_TILE_DOCS;
            for (u32 i = lo + threadIdx.x; i < hi; i += FILT_THREADS) cnt += m[__ldg(r + i) >> SA_REC_TF_BITS];
        }
    } else {
        const u64 *__restrict__ w = words + job.src_off;
        for (u64 i = job.begin + threadIdx.x; i < job.end; i += FILT_THREADS) {
            const u64 doc = __ldg(w + i) >> SA_KEY_SHIFT;
            const bool head = i == 0 || (__ldg(w + i - 1) >> SA_KEY_SHIFT) != doc;
            if (head && doc - doc_base < n_docs) cnt += row_mask[doc - doc_base];
        }
    }
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(df + job.slot, (unsigned long long)cnt);
}

// Caller holds ix->mu; term ids already checked.
static int docfreq_rows_locked(sa_index *ix, const uint32_t *term_ids, uint32_t n_terms, uint64_t *df_out) {
    SA_CUDA(cudaSetDevice(ix->device));
    if (!ix->rows_active) {
        for (u32 i = 0; i < n_terms; i++) df_out[i] = term_ids[i] == SA_NO_TERM ? 0 : ix->h_df[term_ids[i]];
        return SA_OK;
    }
    std::vector<DfJob> jobs;
    const u32 n_tiles = sa_n_tiles(ix->n_docs);
    for (u32 i = 0; i < n_terms; i++) {
        const u32 t = term_ids[i];
        if (t == SA_NO_TERM || ix->h_len[t] == 0) continue;
        DfJob j;
        j.slot = i;
        if (ix->d_recs.p && ix->h_rec_off[t] != SA_NO_DIR && ix->h_dir_off[t] != SA_NO_DIR) {
            j.recs = 1;
            j.src_off = ix->h_rec_off[t];
            j.dir_off = ix->h_dir_off[t];
            for (u64 b = 0; b < n_tiles; b += DF_TILES_PER_JOB) {
                j.begin = b;
                j.end = std::min<u64>(n_tiles, b + DF_TILES_PER_JOB);
                jobs.push_back(j);
            }
        } else {
            j.recs = 0;
            j.src_off = ix->h_off[t];
            j.dir_off = 0;
            for (u64 b = 0; b < ix->h_len[t]; b += DF_WORDS_PER_JOB) {
                j.begin = b;
                j.end = std::min<u64>(ix->h_len[t], b + DF_WORDS_PER_JOB);
                jobs.push_back(j);
            }
        }
    }
    std::vector<u64> h_df(n_terms, 0);
    if (!jobs.empty()) {
        const size_t jobs_bytes = (jobs.size() * sizeof(DfJob) + 255) / 256 * 256;
        int rc;
        if ((rc = ix->misc.reserve(jobs_bytes + (size_t)n_terms * sizeof(u64)))) return rc;
        DfJob *d_jobs = ix->misc.as<DfJob>();
        unsigned long long *d_df = (unsigned long long *)((char *)ix->misc.p + jobs_bytes);
        SA_CUDA(cudaMemcpyAsync(d_jobs, jobs.data(), jobs.size() * sizeof(DfJob), cudaMemcpyHostToDevice, ix->stream));
        SA_CUDA(cudaMemsetAsync(d_df, 0, (size_t)n_terms * sizeof(u64), ix->stream));
        docfreq_rows_kernel<<<(unsigned)jobs.size(), FILT_THREADS, 0, ix->stream>>>(
            ix->d_words.as<u64>(), ix->d_recs.as<u32>(), ix->d_rec_dir.as<u32>(), d_jobs, ix->d_row_mask(),
            ix->doc_base, ix->n_docs, d_df);
        SA_CUDA(cudaGetLastError());
        ix->stats.total_launches++;
        SA_CUDA(cudaMemcpyAsync(h_df.data(), d_df, (size_t)n_terms * sizeof(u64), cudaMemcpyDeviceToHost, ix->stream));
        SA_CUDA(cudaStreamSynchronize(ix->stream));
    }
    memcpy(df_out, h_df.data(), (size_t)n_terms * sizeof(u64));
    return SA_OK;
}

extern "C" int sa_docfreq_rows_batch(sa_index *ix, const uint32_t *term_ids, uint32_t n_terms, uint64_t *df_out) {
    SA_CHECK(ix && (n_terms == 0 || (term_ids && df_out)), "NULL argument");
    int rc = sa_check_term_ids(ix, term_ids, n_terms);
    if (rc) return rc;
    std::lock_guard<std::mutex> g(ix->mu);
    return docfreq_rows_locked(ix, term_ids, n_terms, df_out);
}

extern "C" int sa_docfreq_rows(sa_index *ix, uint32_t term_id, uint64_t *df_out) {
    return sa_docfreq_rows_batch(ix, &term_id, 1, df_out);
}
