// sa_view.cu -- the batched top-k path on a sliced array (a view: SearchArray.search_topk on arr[key]).
//
// The result of a query is the top k of what SearchArray.score returns on the view (reference postings.py:652-680
// on FilteredPosns, middle_out.py:291-317): per-doc counts of the FILTERED postings, BM25 over the view's positions
// with the view's doc lengths and the parent's avgdl, and an idf the caller derived from the view's document
// frequencies (sa_docfreq_rows_batch).  Ids are positions in the view.  Per chunk of queries:
//   1. per-doc counts in DOC space, one row per query in ix->dense:
//        phrase / slop queries: the chunk's phrase terms are filtered once (sa_filter_terms_mask), then every query
//          takes the raw-count route phrase_common takes for a view (sa_phrase_run_sync / sa_span_run) into row 0,
//          which step 2 consumes before the next query overwrites it;
//        term queries: the term kernel in tf mode on the index's own lists, rows [0, n_term) (see the call);
//   2. view_tile_kernel: one CTA per (8,192 view positions, query) gathers count = row[rows[i]] and evaluates
//      bm25_one(count, view_doc_lens[i]) for EVERY position, as bm25_dense_kernel does for .score, so exotic
//      k1 / b and zero counts give the same bits; the tile is staged in shared memory and flush_tile_collect writes
//      the view-space row and the tile's top-k candidates;
//   3. launch_topk_select over the view's tiles (doc_base 0: the keys carry view positions).
// A query whose candidate slots overflowed is re-run alone with a slot per position of the tile, as redo_query
// does for the unsliced batch.
// HBM traffic of a term query: the term scan's own bytes + 4*N (its doc-space row) + 20 per view position (8 row
// index, 4 doc length, 4 gathered count, 4 view-space row).
#include <algorithm>

#include "sa_phrase.cuh"
#include "sa_span.cuh"
#include "sa_term.cuh"

struct ViewState {
    DevBuf d_dl;           // float [padded n_rows]: the doc lengths the view's BM25 uses
    DevBuf d_vrows;        // float [chunk][padded n_rows]: view-space score rows
    DevBuf d_tq;           // TermQuery [chunk]
    DevBuf d_idf;          // float [n_queries], row order
    DevBuf d_row_query;    // u32 [n_queries]: row -> query
    DevBuf d_ovf;          // u32 [n_queries], row order: candidate slots overflowed
    DevBuf d_keys;         // u64 [n_queries * k]: the result keys
};

void sa_free_view(sa_index *ix) {
    if (!ix->view) return;
    ViewState &V = *ix->view;
    V.d_dl.release();
    V.d_vrows.release();
    V.d_tq.release();
    V.d_idf.release();
    V.d_row_query.release();
    V.d_ovf.release();
    V.d_keys.release();
    delete ix->view;
    ix->view = nullptr;
}

// grid = (view tiles, queries).  row = row0 + blockIdx.y indexes the view-space rows, the candidate slots and the
// overflow flags; doc_rows + blockIdx.y * doc_stride is the query's doc-space count row, idf[blockIdx.y] its idf.
__global__ void __launch_bounds__(SA_TERM_THREADS)
view_tile_kernel(const float *__restrict__ doc_rows, u64 doc_stride, const u64 *__restrict__ rows,
                 const float *__restrict__ view_dl, u64 n_rows, Bm25Params p, const float *__restrict__ idf,
                 float *__restrict__ view_rows, u64 view_stride, u32 row0, const TopkCtx t) {
    __shared__ __align__(16) float s_out[SA_TILE_DOCS];
    __shared__ u32 s_top[(SA_TERM_THREADS / 32) * 8];
    __shared__ u32 s_ncand, s_tile_max;
    const u32 tile = blockIdx.x, row = row0 + blockIdx.y;
    const u64 pos0 = (u64)tile * SA_TILE_DOCS;
    const float *__restrict__ counts = doc_rows + (u64)blockIdx.y * doc_stride;
    p.idf = idf[blockIdx.y];
    u32 my_max = 0;
    // thread tid owns positions 4g .. 4g+3 of the tile for g = tid + j * SA_TERM_THREADS: the float4 layout
    // flush_tile_collect reads, so every thread reads back only what it wrote
#pragma unroll
    for (int j = 0; j < SA_TILE_DOCS / SA_TERM_THREADS / 4; j++) {
        const unsigned g = threadIdx.x + j * SA_TERM_THREADS;
        float v[4];
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const u64 i = pos0 + g * 4 + e;
            v[e] = 0.0f;
            if (i < n_rows) {
                v[e] = bm25_one(__ldg(counts + __ldg(rows + i)), __ldg(view_dl + i), p);
                if (v[e] > 0.0f) my_max = max(my_max, __float_as_uint(v[e]));   // NaN and <= 0 never rank
            }
        }
        reinterpret_cast<float4 *>(s_out)[g] = make_float4(v[0], v[1], v[2], v[3]);
    }
    const u32 n_items = (u32)min((u64)SA_TILE_DOCS, n_rows - pos0);
    flush_tile_collect(s_out, view_rows + (u64)row * view_stride + pos0, t, row, tile, my_max, n_items,
                       min((u32)SA_TERM_THREADS, (n_items + 3) / 4), s_top, &s_ncand, &s_tile_max);
}

static int launch_view_tiles(sa_index *ix, const float *doc_rows, u64 doc_stride, const float *d_idf, u32 n_queries,
                             u32 row0, const Bm25Params &p, const TopkCtx &t) {
    ViewState &V = *ix->view;
    if (n_queries == 0 || t.n_tiles == 0) return SA_OK;
    KernelTimer tm(ix, 1);
    view_tile_kernel<<<dim3(t.n_tiles, n_queries), SA_TERM_THREADS, 0, ix->stream>>>(
        doc_rows, doc_stride, ix->d_rows, V.d_dl.as<float>(), ix->n_rows, p, d_idf, V.d_vrows.as<float>(),
        sa_padded_docs(ix->n_rows), row0, t);
    SA_CUDA(cudaGetLastError());
    tm.stop();
    ix->stats.topk_kernel_launches++;
    ix->stats.total_launches++;
    return SA_OK;
}

// tf of n term queries into ix->dense rows [0, n), on the index's own lists (tf-table fast path, no top-k)
static int view_term_counts(sa_index *ix, const TermQuery *h_tq, u32 n) {
    ViewState &V = *ix->view;
    int rc;
    if ((rc = ix->dense.reserve((size_t)n * sa_padded_docs(ix->n_docs) * sizeof(float)))) return rc;
    SA_CUDA(cudaMemcpyAsync(V.d_tq.p, h_tq, n * sizeof(TermQuery), cudaMemcpyHostToDevice, ix->stream));
    TopkCtx none;
    memset(&none, 0, sizeof(none));
    TermBatchArgs a = make_term_args(ix, V.d_tq.as<TermQuery>(), make_bm25(0, 1, 1, 0, ix->doc_lens_nonneg), none);
    a.mode = TERM_MODE_TF;
    return launch_term_batch(ix, a, n);
}

// Raw counts of one phrase / slop query on the view's filtered lists into ix->dense row 0: what phrase_common
// computes for sa_phrase_freqs on a sliced array.  f_offs / f_lens: the query's filtered lists in ix->filt.
static int view_phrase_counts(sa_index *ix, const u32 *tids, u32 nt, u32 slop, bool missing, const u64 *f_offs,
                              const u64 *f_lens) {
    const u64 stride = sa_padded_docs(ix->n_docs);
    int rc;
    if (missing) {                                   // an unknown term: zeros (postings.py:705-708)
        if ((rc = ix->dense.reserve(stride * sizeof(float)))) return rc;
        SA_CUDA(cudaMemsetAsync(ix->dense.p, 0, stride * sizeof(float), ix->stream));
        return SA_OK;
    }
    u64 offs[SA_MAX_PHRASE_TERMS], lens[SA_MAX_PHRASE_TERMS], dirs[SA_MAX_PHRASE_TERMS];
    for (u32 i = 0; i < nt; i++) { offs[i] = f_offs[i]; lens[i] = f_lens[i]; dirs[i] = SA_NO_DIR; }
    const u64 *d_lists = ix->filt.as<u64>();
    if (slop > 0) {
        bool literal;
        if ((rc = sa_span_is_literal(ix, d_lists, offs, lens, nt, &literal))) return rc;
        return sa_span_run(ix, d_lists, offs, lens, dirs, nt, slop, literal, nullptr);
    }
    std::vector<PhraseQuery> pqs(1, make_phrase_query(tids, nt, offs, lens, dirs, 0.0f, false));
    PhraseDump nodump;
    memset(&nodump, 0, sizeof(nodump));
    return sa_phrase_run_sync(ix, pqs, d_lists, 0, make_bm25(0, 1, 1, 0, ix->doc_lens_nonneg), nodump, true);
}

static bool query_missing(const sa_index *ix, const u32 *tids, u32 nt) {
    for (u32 i = 0; i < nt; i++)
        if (tids[i] == SA_NO_TERM || ix->h_len[tids[i]] == 0) return true;
    return false;
}

// keys (and the overflow flags) to the host in one copy and one synchronise
static int view_download(sa_index *ix, u32 nq, u32 k, uint32_t *out_pos, float *out_scores, std::vector<u32> *ovf) {
    ViewState &V = *ix->view;
    const size_t nk = (size_t)nq * k, ovf_bytes = ovf ? (size_t)nq * sizeof(u32) : 0;
    int rc;
    if ((rc = sa_pinned_reserve(ix, nk * sizeof(u64) + ovf_bytes))) return rc;
    SA_CUDA(cudaMemcpyAsync(ix->h_pinned, V.d_keys.p, nk * sizeof(u64), cudaMemcpyDeviceToHost, ix->stream));
    if (ovf)
        SA_CUDA(cudaMemcpyAsync((u64 *)ix->h_pinned + nk, V.d_ovf.p, ovf_bytes, cudaMemcpyDeviceToHost, ix->stream));
    SA_CUDA(cudaStreamSynchronize(ix->stream));
    sa_unpack_keys((const u64 *)ix->h_pinned, nk, out_pos, out_scores);
    if (ovf) ovf->assign((const u32 *)((u64 *)ix->h_pinned + nk), (const u32 *)((u64 *)ix->h_pinned + nk) + nq);
    return SA_OK;
}

extern "C" int sa_score_batch_topk_rows(sa_index *ix, const uint32_t *terms, const uint32_t *term_starts,
                                        const float *idf, uint32_t n_queries, uint32_t slop,
                                        const float *view_doc_lens, float avg_doc_len, float k1, float b, uint32_t k,
                                        uint32_t *out_pos, float *out_scores) {
    SA_CHECK(ix, "index is NULL");
    SA_CHECK(n_queries == 0 || (terms && term_starts && idf && out_pos && out_scores), "NULL argument");
    SA_CHECK(k >= 1 && k <= SA_TOPK_MAX, "k must be in [1, %d]", SA_TOPK_MAX);
    int rc;
    for (u32 q = 0; q < n_queries; q++) {
        const u32 nt = term_starts[q + 1] - term_starts[q];
        SA_CHECK(nt >= 1 && nt <= SA_MAX_PHRASE_TERMS, "query %u: bad number of terms", q);
        if ((rc = sa_check_term_ids(ix, terms + term_starts[q], nt))) return rc;
    }
    std::lock_guard<std::mutex> g(ix->mu);
    SA_CHECK(ix->rows_active, "no row filter installed (sa_index_set_rows)");
    const u64 n_rows = ix->n_rows;
    SA_CHECK(n_rows < 0xFFFFFFFFull, "a view must have fewer than 2^32 - 1 rows");
    SA_CHECK(n_rows == 0 || view_doc_lens, "view_doc_lens is NULL");
    SA_CUDA(cudaSetDevice(ix->device));
    const size_t nk = (size_t)n_queries * k;
    if (n_queries == 0 || n_rows == 0 || avg_doc_len == 0.0f) {     // .score is all zeros: nothing ranks
        for (size_t i = 0; i < nk; i++) { out_pos[i] = SA_NO_DOC; out_scores[i] = 0.0f; }
        return SA_OK;
    }
    if (!ix->view) ix->view = new ViewState();
    ViewState &V = *ix->view;
    const u64 stride = sa_padded_docs(ix->n_docs), vstride = sa_padded_docs(n_rows);
    const u32 n_vtiles = sa_n_tiles(n_rows), slots = sa_topk_slots(k);
    // chunk so the doc-space and view-space rows of one chunk stay within ~4 GB of HBM
    const u32 chunk = (u32)std::min<u64>(65535, std::max<u64>(1, std::min<u64>(n_queries,
                                         (4ull << 30) / ((stride + vstride) * sizeof(float)))));
    // Every buffer is reserved before the first write: DevBuf::reserve does not keep the contents.  ix->dense is the
    // exception -- each step reserves it and consumes what it wrote before the next reserve.
    if ((rc = V.d_dl.reserve(vstride * sizeof(float)))) return rc;
    if ((rc = V.d_vrows.reserve((size_t)chunk * vstride * sizeof(float)))) return rc;
    if ((rc = V.d_tq.reserve((size_t)chunk * sizeof(TermQuery)))) return rc;
    if ((rc = V.d_idf.reserve((size_t)n_queries * sizeof(float)))) return rc;
    if ((rc = V.d_row_query.reserve((size_t)n_queries * sizeof(u32)))) return rc;
    if ((rc = V.d_ovf.reserve((size_t)n_queries * sizeof(u32)))) return rc;
    if ((rc = V.d_keys.reserve(nk * sizeof(u64)))) return rc;
    if ((rc = ix->cand.reserve(cand_bytes(n_vtiles, chunk, slots)))) return rc;

    // rows: chunk by chunk, the term queries first, then the phrase queries
    struct Chunk { u32 row0, n_term, n_phrase; };
    std::vector<Chunk> chunks;
    std::vector<u32> row_query;
    std::vector<float> row_idf;
    row_query.reserve(n_queries);
    row_idf.reserve(n_queries);
    for (u32 q0 = 0; q0 < n_queries; q0 += chunk) {
        const u32 q1 = std::min(n_queries, q0 + chunk);
        Chunk C{(u32)row_query.size(), 0, 0};
        for (int pass = 0; pass < 2; pass++)
            for (u32 q = q0; q < q1; q++) {
                const bool term = term_starts[q + 1] - term_starts[q] == 1;
                if (term != (pass == 0)) continue;
                row_query.push_back(q);
                row_idf.push_back(idf[q]);
                (term ? C.n_term : C.n_phrase)++;
            }
        chunks.push_back(C);
    }
    SA_CUDA(cudaMemcpyAsync(V.d_dl.p, view_doc_lens, n_rows * sizeof(float), cudaMemcpyHostToDevice, ix->stream));
    SA_CUDA(cudaMemcpyAsync(V.d_idf.p, row_idf.data(), n_queries * sizeof(float), cudaMemcpyHostToDevice, ix->stream));
    SA_CUDA(cudaMemcpyAsync(V.d_row_query.p, row_query.data(), n_queries * sizeof(u32), cudaMemcpyHostToDevice, ix->stream));
    SA_CUDA(cudaMemsetAsync(V.d_ovf.p, 0, n_queries * sizeof(u32), ix->stream));
    // BM25 exactly as ops.bm25_score -> sa_op_bm25_score sets it up (idf per row, in the kernel)
    const Bm25Params p = make_bm25(0.0f, avg_doc_len, k1, b, false);
    const float *d_idf = V.d_idf.as<float>();

    for (const Chunk &C : chunks) {
        const u32 Q = C.n_term + C.n_phrase;
        TopkCtx t = make_topk_ctx(ix->cand.p, n_vtiles, Q, slots, k, V.d_ovf.as<u32>() + C.row0);
        if (C.n_phrase) {
            // one filter pass over every list of the chunk's phrases (a phrase with a missing term has none)
            std::vector<u32> ftids, fstart;
            std::vector<unsigned char> missing;
            for (u32 j = 0; j < C.n_phrase; j++) {
                const u32 q = row_query[C.row0 + C.n_term + j];
                const u32 *tids = terms + term_starts[q];
                const u32 nt = term_starts[q + 1] - term_starts[q];
                fstart.push_back((u32)ftids.size());
                missing.push_back(query_missing(ix, tids, nt));
                if (!missing.back()) ftids.insert(ftids.end(), tids, tids + nt);
            }
            std::vector<u64> f_offs, f_lens;
            if (!ftids.empty() && (rc = sa_filter_terms_mask(ix, ftids.data(), (u32)ftids.size(), ix->d_row_mask, 0,
                                                             SA_ALL_BITS, false, f_offs, f_lens, nullptr))) return rc;
            for (u32 j = 0; j < C.n_phrase; j++) {
                const u32 q = row_query[C.row0 + C.n_term + j];
                const u32 *tids = terms + term_starts[q];
                const u32 nt = term_starts[q + 1] - term_starts[q];
                const u64 *fo = missing[j] ? nullptr : f_offs.data() + fstart[j];
                const u64 *fl = missing[j] ? nullptr : f_lens.data() + fstart[j];
                if ((rc = view_phrase_counts(ix, tids, nt, slop, missing[j], fo, fl))) return rc;
                if ((rc = launch_view_tiles(ix, ix->dense.as<float>(), stride, d_idf + C.row0 + C.n_term + j, 1,
                                            C.n_term + j, p, t))) return rc;
            }
        }
        if (C.n_term) {
            // A view keeps or drops WHOLE docs (no position filter here), so a doc of the view has the same tf in the
            // filtered list as in the index's own list: the term kernel runs on the own lists, with the tf table, and
            // no compaction.  Docs outside the view get counts too; view_tile_kernel never gathers them.
            std::vector<TermQuery> tqs(C.n_term);
            for (u32 j = 0; j < C.n_term; j++) tqs[j] = make_term_query(ix, terms[term_starts[row_query[C.row0 + j]]], 0.0f);
            if ((rc = view_term_counts(ix, tqs.data(), C.n_term))) return rc;
            if ((rc = launch_view_tiles(ix, ix->dense.as<float>(), stride, d_idf + C.row0, C.n_term, 0, p, t))) return rc;
        }
        if ((rc = launch_topk_select(ix, t, Q, 0, V.d_keys.as<u64>(), V.d_row_query.as<u32>() + C.row0))) return rc;
    }
    std::vector<u32> ovf;
    if ((rc = view_download(ix, n_queries, k, out_pos, out_scores, &ovf))) return rc;
    bool redone = false;
    for (u32 r = 0; r < n_queries; r++) {
        if (!ovf[r]) continue;
        // exact re-run of one query: a candidate slot per position of the tile cannot overflow
        const u32 q = row_query[r];
        const u32 *tids = terms + term_starts[q];
        const u32 nt = term_starts[q + 1] - term_starts[q];
        if (nt == 1) {
            TermQuery tq = make_term_query(ix, tids[0], 0.0f);
            if ((rc = view_term_counts(ix, &tq, 1))) return rc;
        } else {
            const bool miss = query_missing(ix, tids, nt);
            std::vector<u64> f_offs, f_lens;
            if (!miss && (rc = sa_filter_terms_mask(ix, tids, nt, ix->d_row_mask, 0, SA_ALL_BITS, false, f_offs, f_lens,
                                                    nullptr))) return rc;
            if ((rc = view_phrase_counts(ix, tids, nt, slop, miss, f_offs.data(), f_lens.data()))) return rc;
        }
        if ((rc = ix->cand.reserve(cand_bytes(n_vtiles, 1, SA_TILE_DOCS)))) return rc;
        SA_CUDA(cudaMemsetAsync(V.d_ovf.as<u32>() + r, 0, sizeof(u32), ix->stream));
        TopkCtx t = make_topk_ctx(ix->cand.p, n_vtiles, 1, SA_TILE_DOCS, k, V.d_ovf.as<u32>() + r);
        if ((rc = launch_view_tiles(ix, ix->dense.as<float>(), stride, d_idf + r, 1, 0, p, t))) return rc;
        if ((rc = launch_topk_select(ix, t, 1, 0, V.d_keys.as<u64>(), V.d_row_query.as<u32>() + r))) return rc;
        redone = true;
    }
    if (!redone) return SA_OK;
    return view_download(ix, n_queries, k, out_pos, out_scores, nullptr);
}
