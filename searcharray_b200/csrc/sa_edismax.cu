// sa_edismax.cu -- multi-field query combination on the device (SURVEY.md section 8f-1).
//
// Replaces the numpy part of the reference's edismax (searcharray/solr.py:117-355): the per-(term,
// field) BM25 vectors, the per-field phrase vectors and the combined score vector stay in HBM; the
// host only parses the query, computes idf (numpy, like the reference) and reads back the result
// (dense, or just the top-k).
//
//   sa_multi_qf          solr.py:117-178.  One fused term-kernel launch per field writes the field's
//                        BM25 rows; edismax_combine_kernel folds them per doc with the reference's
//                        exact arithmetic: float32 `score * boost`, float64 running sum / maximum,
//                        term = max + (sum - max) * tie, mm on "terms scoring > 0", sum over terms
//                        in order (term-centric); all-float32 per-field sums (field-centric).
//   sa_multi_filter      the phrase phases run on arrays SLICED to qf > 0 (solr.py:326-330): the
//                        posting lists of the query terms are filtered by the match mask
//                        (sa_filter.cu) and their filtered doc frequencies returned (quirk iii).
//   sa_multi_phrases     every pf / pf2 / pf3 phrase of one field in one phrase-kernel launch on the
//                        filtered lists (BM25 applied in the kernel).
//   sa_multi_add_phase   solr.py:335-353: float32 sum of the phase's boosted vectors in list order,
//                        added to qf where qf != 0.
//   sa_multi_topk        exact top-k of the float64 vector (score desc, doc asc): edismax_tile_kernel
//                        ranks each tile by f64_proxy_key and keeps every doc at or above the tile's
//                        bound with its float64 score (collect_tile_f64, as classic_similarity's
//                        search_topk does), topk_select_f64_kernel orders the candidates in float64.
#include <algorithm>
#include <cmath>
#include <functional>

#include "sa_multi.cuh"
#include "sa_phrase.cuh"
#include "sa_term.cuh"

int sa_filter_terms_mask(sa_index *ix, const uint32_t *term_ids, uint32_t n_terms, const unsigned char *d_mask,
                         u64 pay_lo, u64 pay_hi, bool use_payload, std::vector<u64> &offs, std::vector<u64> &lens,
                         std::vector<u64> *df_out);

struct CombineArgs {
    const float *rows[ED_MAX_FIELDS];    // field f: [n_terms[f]][stride]
    u32 n_terms[ED_MAX_FIELDS];
    float boost[ED_MAX_FIELDS];
    u32 has_boost[ED_MAX_FIELDS];
    u32 mm[ED_MAX_FIELDS];
    u32 n_fields;
    double tie;
    u64 n_docs, stride;
    double *qf;
    unsigned char *mask;
    unsigned long long *count;
};

// term-centric (solr.py:117-147)
__global__ void __launch_bounds__(256)
edismax_combine_terms_kernel(const CombineArgs a) {
    const u64 d = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    bool hit = false;
    if (d < a.stride) {
        double total = 0.0;
        u32 matched = 0;
        if (d < a.n_docs) {
            const u32 T = a.n_terms[0];
            for (u32 t = 0; t < T; t++) {
                double run_sum = 0.0, run_max = 0.0;
                for (u32 f = 0; f < a.n_fields; f++) {
                    float s = a.rows[f][(u64)t * a.stride + d];
                    if (a.has_boost[f]) s = __fmul_rn(s, a.boost[f]);
                    run_sum = __dadd_rn(run_sum, (double)s);
                    run_max = fmax(run_max, (double)s);               // np.maximum (no NaNs on this path)
                }
                const double term = __dadd_rn(run_max, __dmul_rn(__dadd_rn(run_sum, -run_max), a.tie));
                if (term > 0.0) matched++;
                total = t == 0 ? term : __dadd_rn(total, term);
            }
            if (matched < a.mm[0]) total = 0.0;
        }
        a.qf[d] = total;
        hit = total > 0.0;
        a.mask[d] = hit ? 1 : 0;
    }
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(a.count, (unsigned long long)__popc(m));
}

// field-centric (solr.py:150-178): everything float32
__global__ void __launch_bounds__(256)
edismax_combine_fields_kernel(const CombineArgs a) {
    const u64 d = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    bool hit = false;
    if (d < a.stride) {
        float result = 0.0f;
        if (d < a.n_docs) {
            float summed = 0.0f, best = 0.0f;
            for (u32 f = 0; f < a.n_fields; f++) {
                float tot = 0.0f;
                u32 matched = 0;
                for (u32 t = 0; t < a.n_terms[f]; t++) {
                    const float s = a.rows[f][(u64)t * a.stride + d];
                    if (s > 0.0f) matched++;
                    tot = t == 0 ? s : __fadd_rn(tot, s);
                }
                if (matched < a.mm[f]) tot = 0.0f;
                if (a.has_boost[f]) tot = __fmul_rn(tot, a.boost[f]);
                summed = f == 0 ? tot : __fadd_rn(summed, tot);
                best = f == 0 ? tot : fmaxf(best, tot);
            }
            // qf + (summed - qf) * tie with a Python-float tie: numpy keeps float32
            result = __fadd_rn(best, __fmul_rn(__fadd_rn(summed, -best), (float)a.tie));
        }
        a.qf[d] = (double)result;
        hit = result > 0.0f;
        a.mask[d] = hit ? 1 : 0;
    }
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(a.count, (unsigned long long)__popc(m));
}

struct PhaseArgs {
    const float *rows[ED_MAX_PHASE_ENTRIES];
    float boost[ED_MAX_PHASE_ENTRIES];
    u32 has_boost[ED_MAX_PHASE_ENTRIES];
    u32 n;
    u64 n_docs;
    double *qf;
    int f32_mode;
};
// a kernel parameter: one phase is one launch (one float32 fold in the reference's order), never split over two
static_assert(sizeof(PhaseArgs) <= 4096, "PhaseArgs must fit the classic kernel parameter limit");

// qf[where qf != 0] += float32 sum of the phase's vectors, in order (solr.py:335-353)
__global__ void __launch_bounds__(256)
edismax_add_phase_kernel(const PhaseArgs a) {
    const u64 d = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (d >= a.n_docs) return;
    const double cur = a.qf[d];
    if (cur == 0.0) return;
    float acc = 0.0f;
    for (u32 i = 0; i < a.n; i++) {
        float s = a.rows[i][d];
        if (a.has_boost[i]) s = __fmul_rn(s, a.boost[i]);
        acc = i == 0 ? s : __fadd_rn(acc, s);
    }
    if (a.f32_mode) a.qf[d] = (double)__fadd_rn((float)cur, acc);
    else a.qf[d] = __dadd_rn(cur, (double)acc);
}

// Top-k candidates of one tile of qf (positions [0, n_docs)), ranked by f64_proxy_key with the float64 scores beside
// them: the collection classic_similarity's search_topk uses (sim_tile_kernel).  The tile is read whole: the combine
// kernels write qf's padding past n_docs with zeros, which never rank.
// DEEP: k > SA_TOPK_MAX, collect_tile_f64's exact tile bound.
template <bool DEEP>
__global__ void __launch_bounds__(SA_TERM_THREADS)
edismax_tile_kernel(const double *__restrict__ qf, u64 n_docs, const TopkCtx t, u64 *__restrict__ tile_d) {
    __shared__ u32 s_top[(SA_TERM_THREADS / 32) * 8];
    __shared__ u32 s_ncand, s_tile_max;
    const u32 tile = blockIdx.x;
    const u64 pos0 = (u64)tile * SA_TILE_DOCS;
    u32 key[SA_TILE_DOCS / SA_TERM_THREADS], my_max = 0;
#pragma unroll
    for (int j = 0; j < SA_TILE_DOCS / SA_TERM_THREADS / 4; j++) {
        const u64 i0 = pos0 + (threadIdx.x + j * SA_TERM_THREADS) * 4;
#pragma unroll
        for (int e = 0; e < 4; e++) {
            key[j * 4 + e] = f64_proxy_key(__ldg(qf + i0 + e));
            my_max = max(my_max, key[j * 4 + e]);
        }
    }
    collect_tile_f64<DEEP>(key, my_max, (u32)min((u64)SA_TILE_DOCS, n_docs - pos0), t, tile_d, 0, tile, s_top, &s_ncand,
                     &s_tile_max, [&](u32 local) { return __ldg(qf + pos0 + local); });
}

// ------------------------------------------------------------------------------ host
extern "C" int sa_multi_create(sa_index *const *fields, uint32_t n_fields, sa_multi **out) {
    SA_CHECK(fields && out && n_fields >= 1 && n_fields <= ED_MAX_FIELDS, "1..%d fields", ED_MAX_FIELDS);
    for (u32 f = 0; f < n_fields; f++) {
        SA_CHECK(fields[f], "field %u is NULL", f);
        SA_CHECK(fields[f]->device == fields[0]->device && fields[f]->n_docs == fields[0]->n_docs &&
                 fields[f]->doc_base == fields[0]->doc_base, "fields must share device, doc range and size");
    }
    std::unique_ptr<sa_multi> m(new sa_multi());
    m->fields.assign(fields, fields + n_fields);
    m->device = fields[0]->device;
    m->n_docs = fields[0]->n_docs;
    m->doc_base = fields[0]->doc_base;
    m->stride = sa_padded_docs(m->n_docs);
    m->filt_offs.resize(n_fields);
    m->filt_lens.resize(n_fields);
    m->phrase_rows.assign(n_fields, 0);
    m->filt_bound.assign(n_fields, 0);
    m->shared.assign(n_fields, 0);
    m->rows.resize(n_fields);
    for (u32 f = 0; f < n_fields; f++)
        for (u32 g = 0; g < n_fields; g++)
            if (g != f && fields[g] == fields[f]) m->shared[f] = 1;
    SA_CUDA(cudaSetDevice(m->device));
    const u64 s = std::max<u64>(m->stride, SA_TILE_DOCS);
    SA_CUDA(cudaStreamCreateWithFlags(&m->stream, cudaStreamNonBlocking));
    int rc;
    if ((rc = m->d_qf.allocate(s * sizeof(double))) || (rc = m->d_mask.allocate(s)) || (rc = m->d_count.allocate(64))) return rc;
    *out = m.release();
    return SA_OK;
}

extern "C" int sa_multi_destroy(sa_multi *m) {
    delete m;
    return SA_OK;
}

extern "C" int sa_multi_qf(sa_multi *m, int field_centric, const uint32_t *n_terms, const uint32_t *term_ids,
                           const float *idf, const float *boost, const uint32_t *has_boost,
                           const float *avg_doc_len, const float *k1, const float *b, const uint32_t *mm,
                           double tie, uint64_t *n_matches) {
    SA_CHECK(m && n_terms && boost && has_boost && avg_doc_len && k1 && b && mm && n_matches, "NULL argument");
    std::lock_guard<std::mutex> g(m->mu);
    SA_CUDA(cudaSetDevice(m->device));
    const u32 F = (u32)m->fields.size();
    CombineArgs a;
    memset(&a, 0, sizeof(a));
    u32 at = 0;
    for (u32 f = 0; f < F; f++) {
        const u32 T = n_terms[f];
        SA_CHECK(T <= SA_MAX_PHRASE_TERMS, "too many query terms");
        SA_CHECK(field_centric || T == n_terms[0], "term-centric needs the same number of terms per field");
        SA_CHECK(T == 0 || (term_ids && idf), "NULL argument");
        sa_index *ix = m->fields[f];
        FieldGuard fg(ix, m->stream);
        int rc;
        if ((rc = (m->shared[f] ? m->rows[f] : ix->dense).reserve(std::max<u64>(T, 1) * m->stride * sizeof(float)))) return rc;
        float *rows = m->field_rows(f);
        a.rows[f] = rows;
        a.n_terms[f] = T;
        a.boost[f] = boost[f];
        a.has_boost[f] = has_boost[f];
        a.mm[f] = mm[f];
        if (T && (avg_doc_len[f] == 0.0f || m->n_docs == 0)) {         // similarity.py:31-32: zeros
            SA_CUDA(cudaMemsetAsync(rows, 0, (size_t)T * m->stride * sizeof(float), m->stream));
        } else if (T) {
            if ((rc = sa_check_term_ids(ix, term_ids + at, T))) return rc;
            std::vector<TermQuery> tqs(T);
            Bm25Params p = make_bm25(1.0f, avg_doc_len[f], k1[f], b[f], ix->doc_lens_nonneg);
            for (u32 t = 0; t < T; t++) {
                tqs[t] = make_term_query(ix, term_ids[at + t], idf[at + t]);
                if (!make_bm25(idf[at + t], avg_doc_len[f], k1[f], b[f], ix->doc_lens_nonneg).sparse_ok) p.sparse_ok = 0;
            }
            if ((rc = ix->queries.reserve(T * sizeof(TermQuery)))) return rc;
            SA_CUDA(cudaMemcpyAsync(ix->queries.p, tqs.data(), T * sizeof(TermQuery), cudaMemcpyHostToDevice, m->stream));
            TopkCtx none;
            memset(&none, 0, sizeof(none));
            TermBatchArgs ta = make_term_args(ix, ix->queries.as<TermQuery>(), p, none);
            ta.out = rows;
            if ((rc = launch_term_batch(ix, ta, T))) return rc;
            SA_CUDA(cudaStreamSynchronize(m->stream));                  // tqs leaves scope
        }
        at += T;
    }
    a.n_fields = F;
    a.tie = tie;
    a.n_docs = m->n_docs;
    a.stride = m->stride;
    a.qf = m->d_qf.as<double>();
    a.mask = m->d_mask.as<unsigned char>();
    a.count = m->d_count.as<unsigned long long>();
    SA_CUDA(cudaMemsetAsync(m->d_count.p, 0, sizeof(unsigned long long), m->stream));
    const unsigned blocks = (unsigned)((std::max<u64>(m->stride, 1) + 255) / 256);
    if (field_centric) edismax_combine_fields_kernel<<<blocks, 256, 0, m->stream>>>(a);
    else edismax_combine_terms_kernel<<<blocks, 256, 0, m->stream>>>(a);
    SA_CUDA(cudaGetLastError());
    unsigned long long cnt = 0;
    SA_CUDA(cudaMemcpyAsync(&cnt, m->d_count.p, sizeof(cnt), cudaMemcpyDeviceToHost, m->stream));
    SA_CUDA(cudaStreamSynchronize(m->stream));
    *n_matches = cnt;
    m->f32_mode = field_centric != 0;
    m->has_qf = true;
    for (u32 f = 0; f < F; f++) { m->filt_offs[f].clear(); m->filt_lens[f].clear(); m->phrase_rows[f] = 0; }
    return SA_OK;
}

extern "C" int sa_multi_filter(sa_multi *m, uint32_t field, const uint32_t *term_ids, uint32_t n_terms,
                               uint64_t *df_out) {
    SA_CHECK(m && term_ids && df_out && field < m->fields.size() && n_terms >= 1, "bad argument");
    SA_CHECK(m->has_qf, "sa_multi_qf has not run");
    std::lock_guard<std::mutex> g(m->mu);
    SA_CUDA(cudaSetDevice(m->device));
    sa_index *ix = m->fields[field];
    int rc = sa_check_term_ids(ix, term_ids, n_terms);
    if (rc) return rc;
    FieldGuard fg(ix, m->stream);
    std::vector<u64> dfs;
    if (m->filt_bound[field] == 0) {
        // one allocation for any query: room for filtered copies of the longest lists a query could name
        std::vector<u64> lens(ix->h_len);
        const size_t top = std::min<size_t>(lens.size(), SA_MAX_PHRASE_TERMS);
        std::partial_sort(lens.begin(), lens.begin() + top, lens.end(), std::greater<u64>());
        u64 bound = 64;
        for (size_t i = 0; i < top; i++) bound += lens[i] + 2;
        m->filt_bound[field] = bound;
    }
    {
        int rc0 = ix->filt.reserve(m->filt_bound[field] * sizeof(u64));
        if (rc0) return rc0;
    }
    if ((rc = sa_filter_terms_mask(ix, term_ids, n_terms, m->d_mask.as<unsigned char>(), 0, SA_ALL_BITS, false,
                                   m->filt_offs[field], m->filt_lens[field], &dfs))) return rc;
    for (u32 t = 0; t < n_terms; t++) df_out[t] = dfs[t];
    return SA_OK;
}

extern "C" int sa_multi_phrases(sa_multi *m, uint32_t field, uint32_t n_phrases, const uint32_t *phrase_starts,
                                const uint32_t *term_slots, const uint32_t *term_ids, const float *idf,
                                float avg_doc_len, float k1, float b) {
    SA_CHECK(m && field < m->fields.size() && n_phrases >= 1 && n_phrases <= ED_MAX_ROWS, "bad argument");
    SA_CHECK(phrase_starts && term_slots && term_ids && idf, "NULL argument");
    std::lock_guard<std::mutex> g(m->mu);
    SA_CUDA(cudaSetDevice(m->device));
    sa_index *ix = m->fields[field];
    const std::vector<u64> &offs = m->filt_offs[field], &lens = m->filt_lens[field];
    SA_CHECK(!offs.empty(), "sa_multi_filter has not run for this field");
    FieldGuard fg(ix, m->stream);
    int rc;
    m->phrase_rows[field] = n_phrases;
    const size_t row_bytes = (size_t)n_phrases * m->stride * sizeof(float);
    if (m->shared[field] && (rc = m->rows[field].reserve(row_bytes))) return rc;
    if (avg_doc_len == 0.0f || m->n_docs == 0) {
        if (!m->shared[field] && (rc = ix->dense.reserve(row_bytes))) return rc;
        SA_CUDA(cudaMemsetAsync(m->field_rows(field), 0, row_bytes, m->stream));
        return SA_OK;
    }
    std::vector<PhraseQuery> pqs(n_phrases);
    const Bm25Params p = make_bm25(1.0f, avg_doc_len, k1, b, ix->doc_lens_nonneg);
    for (u32 i = 0; i < n_phrases; i++) {
        const u32 s0 = phrase_starts[i], nt = phrase_starts[i + 1] - s0;
        SA_CHECK(nt >= 2 && nt <= SA_MAX_PHRASE_TERMS, "phrase %u: 2..%d terms", i, SA_MAX_PHRASE_TERMS);
        SA_CHECK(make_bm25(idf[i], avg_doc_len, k1, b, ix->doc_lens_nonneg).sparse_ok,
                 "edismax phrase phases need ordinary BM25 parameters (k1 > 0, 0 <= b < 1, finite idf >= 0)");
        u64 p_offs[SA_MAX_PHRASE_TERMS], p_lens[SA_MAX_PHRASE_TERMS];
        bool missing = false;
        for (u32 j = 0; j < nt; j++) {
            const u32 slot = term_slots[s0 + j];
            SA_CHECK(slot < offs.size(), "term slot out of range");
            if (term_ids[s0 + j] == SA_NO_TERM || lens[slot] == 0) missing = true;
            p_offs[j] = offs[slot];
            p_lens[j] = lens[slot];
        }
        pqs[i] = make_phrase_query(term_ids + s0, nt, p_offs, p_lens, nullptr, idf[i], missing);
    }
    PhraseDump nodump;
    memset(&nodump, 0, sizeof(nodump));
    if ((rc = sa_phrase_run_sync(ix, pqs, ix->filt.as<u64>(), 1, p, nodump, false))) return rc;
    // the phrase kernel writes ix->dense: a field whose index another field shares keeps its own copy
    if (m->shared[field]) SA_CUDA(cudaMemcpyAsync(m->rows[field].p, ix->dense.p, row_bytes, cudaMemcpyDeviceToDevice, m->stream));
    return SA_OK;
}

extern "C" int sa_multi_add_phase(sa_multi *m, uint32_t n_entries, const uint32_t *entry_field,
                                  const uint32_t *entry_row, const float *entry_boost, const uint32_t *entry_has_boost) {
    SA_CHECK(m && m->has_qf, "sa_multi_qf has not run");
    if (n_entries == 0) return SA_OK;
    SA_CHECK(entry_field && entry_row && entry_boost && entry_has_boost, "NULL argument");
    SA_CHECK(n_entries <= ED_MAX_PHASE_ENTRIES, "%u phase entries: at most %d", n_entries, ED_MAX_PHASE_ENTRIES);
    std::lock_guard<std::mutex> g(m->mu);
    SA_CUDA(cudaSetDevice(m->device));
    PhaseArgs a;
    memset(&a, 0, sizeof(a));
    for (u32 i = 0; i < n_entries; i++) {
        SA_CHECK(entry_field[i] < m->fields.size() && entry_row[i] < m->phrase_rows[entry_field[i]], "entry %u out of range", i);
        a.rows[i] = m->field_rows(entry_field[i]) + (u64)entry_row[i] * m->stride;
        a.boost[i] = entry_boost[i];
        a.has_boost[i] = entry_has_boost[i];
    }
    a.n = n_entries;
    a.n_docs = m->n_docs;
    a.qf = m->d_qf.as<double>();
    a.f32_mode = m->f32_mode ? 1 : 0;
    if (m->n_docs) {
        edismax_add_phase_kernel<<<(unsigned)((m->n_docs + 255) / 256), 256, 0, m->stream>>>(a);
        SA_CUDA(cudaGetLastError());
    }
    SA_CUDA(cudaStreamSynchronize(m->stream));
    return SA_OK;
}

extern "C" int sa_multi_download(sa_multi *m, void *out, int as_float32) {
    SA_CHECK(m && out && m->has_qf, "nothing to download");
    std::lock_guard<std::mutex> g(m->mu);
    SA_CUDA(cudaSetDevice(m->device));
    if (m->n_docs == 0) return SA_OK;
    if (!as_float32) {
        SA_CUDA(cudaMemcpyAsync(out, m->d_qf.as<double>(), m->n_docs * sizeof(double), cudaMemcpyDeviceToHost, m->stream));
        SA_CUDA(cudaStreamSynchronize(m->stream));
        return SA_OK;
    }
    std::vector<double> tmp(m->n_docs);
    SA_CUDA(cudaMemcpyAsync(tmp.data(), m->d_qf.as<double>(), m->n_docs * sizeof(double), cudaMemcpyDeviceToHost, m->stream));
    SA_CUDA(cudaStreamSynchronize(m->stream));
    float *o = (float *)out;
    for (u64 i = 0; i < m->n_docs; i++) o[i] = (float)tmp[i];           // exact: the values are float32
    return SA_OK;
}

extern "C" int sa_multi_is_float32(sa_multi *m, int *out) {
    SA_CHECK(m && out, "NULL argument");
    *out = m->f32_mode ? 1 : 0;
    return SA_OK;
}

extern "C" int sa_multi_topk(sa_multi *m, uint32_t k, uint32_t *out_docs, double *out_scores) {
    SA_CHECK(m && out_docs && out_scores && m->has_qf, "bad argument");
    SA_CHECK(k >= 1 && k <= SA_TOPK_DEEP_MAX, "k must be in [1, %d]", SA_TOPK_DEEP_MAX);
    std::lock_guard<std::mutex> g(m->mu);
    SA_CUDA(cudaSetDevice(m->device));
    for (u32 i = 0; i < k; i++) { out_docs[i] = SA_NO_DOC; out_scores[i] = 0.0; }
    if (m->n_docs == 0) return SA_OK;
    sa_index *ix = m->fields[0];
    FieldGuard fg(ix, m->stream);
    const u32 T = sa_n_tiles(m->n_docs);
    int rc;
    if ((rc = m->keys.reserve((size_t)k * (sizeof(u64) + sizeof(double)) + sizeof(u32)))) return rc;
    u64 *d_keys = m->keys.as<u64>();
    double *d_scores = (double *)(d_keys + k);
    u32 *d_ovf = (u32 *)(d_scores + k);
    std::vector<u64> h(2 * (size_t)k + 1);          // the keys, the scores' bits, the overflow flag
    // a tile with more candidates than slots sends the query once more with a slot per position, which cannot overflow
    for (u32 slots = sa_topk_slots_f64(k, sa_topk_slots(k));; slots = SA_TILE_DOCS) {
        const size_t cb = cand_bytes(T, 1, slots);
        if ((rc = m->cand.reserve(cb + (size_t)T * slots * sizeof(u64)))) return rc;
        u64 *tile_d = (u64 *)((char *)m->cand.p + cb);
        SA_CUDA(cudaMemsetAsync(d_ovf, 0, sizeof(u32), m->stream));
        const TopkCtx t = make_topk_ctx(m->cand.p, T, 1, slots, k, d_ovf);
        {
            KernelTimer tm(ix, 1);
            if (k > SA_TOPK_MAX) {
                edismax_tile_kernel<true><<<T, SA_TERM_THREADS, 0, m->stream>>>(m->d_qf.as<double>(), m->n_docs, t, tile_d);
                ix->stats.deep_tiles += T;
            } else {
                edismax_tile_kernel<false><<<T, SA_TERM_THREADS, 0, m->stream>>>(m->d_qf.as<double>(), m->n_docs, t, tile_d);
            }
            SA_CUDA(cudaGetLastError());
            tm.stop();
            ix->stats.topk_kernel_launches++;
            ix->stats.total_launches++;
        }
        if ((rc = launch_topk_select_f64(ix, t, tile_d, 1, m->doc_base, d_keys, d_scores, nullptr))) return rc;
        SA_CUDA(cudaMemcpyAsync(h.data(), d_keys, (size_t)k * (sizeof(u64) + sizeof(double)) + sizeof(u32),
                                cudaMemcpyDeviceToHost, m->stream));
        SA_CUDA(cudaStreamSynchronize(m->stream));
        if (!(u32)h[2 * k] || slots == SA_TILE_DOCS) break;
    }
    for (u32 i = 0; i < k; i++) {
        if (h[i] == 0) continue;
        out_docs[i] = 0xFFFFFFFFu - (u32)h[i];                           // the select added doc_base
        memcpy(&out_scores[i], &h[k + i], sizeof(double));
    }
    return SA_OK;
}
