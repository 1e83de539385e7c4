// sa_view.cu -- sa_score_batch_topk_sim: SearchArray.search_topk on a sliced array (a view: arr[key]) under every
// similarity, and on the unsliced array under bm25_impact, bm25_legacy_similarity and classic_similarity.
//
// The result of a query is the top k of SearchArray.score(q, similarity=sim, slop=slop) on the same array or view
// (reference postings.py:652-680 on FilteredPosns, middle_out.py:291-317): per-doc counts of the (on a view:
// filtered) postings, the similarity's formula over the positions, and an idf the caller derived from the document
// frequencies (a view's from sa_docfreq_rows_batch).  Ids are positions in the view, or doc ids on an unsliced
// array.  Per chunk of queries (sa_plan_rows, the chunks and row order of the unsliced BM25 batch):
//   1. per-doc counts in DOC space, one row per query in ix->dense:
//        phrase / slop queries: on a view the chunk's phrase terms are filtered once (sa_filter_terms_mask), then
//          every query takes sa_phrase_row, the raw-count route of sa_phrase_freqs, into row 0, which step 2
//          consumes before the next query overwrites it;
//        term queries: the term kernel in tf mode on the index's own lists, rows [0, n_term) (see term_tiles);
//   2. sim_tile_kernel: one CTA per (8,192 positions, query) gathers each position's count, scores it and collects
//      the tile's top-k candidates;
//   3. launch_topk_select (launch_topk_select_f64 for classic) over the tiles.
// A query whose candidate slots overflowed is re-run alone with a slot per position of the tile, as redo_query
// does for the unsliced batch.  Step 2 (launch_sim_tiles) is also the BM25 scoring of redo_query's phrase and span
// re-runs, over the raw counts in row 0 of the unsliced array.
// HBM traffic of a term query: the term scan's own bytes + 4*N (its doc-space row), then per position 4 (gathered
// count) and 8 (row index, views only), and 4 (doc length) per position whose count is > 0.
#include <algorithm>
#include <cmath>
#include <type_traits>

#include "sa_phrase.cuh"
#include "sa_sim.cuh"
#include "sa_span.cuh"
#include "sa_term.cuh"

struct ViewState {
    DevBuf d_dl;           // float [n_rows]: the doc lengths BM25 uses on the view
    DevBuf d_tq;           // TermQuery [chunk]
    DevBuf d_idf;          // double [n_queries], row order
    DevBuf d_row_query;    // u32 [n_queries]: row -> query
    DevBuf d_ovf;          // u32 [n_queries], row order: candidate slots overflowed
    DevBuf d_keys;         // u64 [n_queries * k]: the result keys
    DevBuf d_cand_d;       // u64 [chunk][tiles][slots]: float64 score bits of the classic candidates
    DevBuf d_scores;       // double [n_queries * k]: the classic result scores
    DevBuf d_where;        // the WhereMask rows of a masked sa_score_batch_topk_sim
};

void ViewStateDelete::operator()(ViewState *v) const { delete v; }

template <int KIND> using TileParams = std::conditional_t<KIND == SA_SIM_BM25, Bm25Params, SimParams>;

// grid = (tiles of positions, queries).  row = row0 + blockIdx.y indexes the candidate slots and the overflow flags;
// doc_rows + blockIdx.y * doc_stride is the query's doc-space count row, idf[blockIdx.y] its idf.  Position i reads
// its count at doc = rows[i] on a view (rows == NULL: the unsliced array, doc = i) and its doc length at
//   SA_SIM_BM25: doc_lens[i], the lengths the view's BM25 uses (the stepped-slice quirk of bm25_score), or the
//                index's own on the unsliced array;
//   the others:  doc_lens[doc], SearchArray.doclengths().
// A zero count never scores > 0 under any of the formulas (0 / x, 0 * l and sqrt(0) give +-0 or NaN, and the idf
// cannot turn them positive), so the doc length is loaded only where the count is > 0.  What the tile ranks by, and
// how:
//   BM25:    the float32 score bm25_one(count, dl, p), with the row's idf narrowed back to the float32 the caller
//            rounded it from; flush_tile_collect and topk_select_kernel apply unchanged.
//   impact:  the float32 score itself, as BM25.
//   legacy:  score = fl64(idf * (double)sat), sat the float32 saturation, idf finite.  For idf > 0 it is strictly
//            increasing in sat: two distinct float32 sats differ by a relative 2^-24 at least, the double product
//            of each is exact to a relative 2^-53 -- their order survives the rounding (and both the float32 and
//            float64 ranges are wide enough that nothing overflows or underflows).  So sat is an EXACT key with the
//            same ties, and the existing collector and select are exact; for idf < 0 the key is -sat (the score
//            is > 0 only where sat < 0), for idf == 0 nothing ranks.  The score is formed on the host for the k
//            winners only: |idf| * key, the same rounding as idf * sat.
//   classic: score = fl64(fl64(idf * sqrt_tf) * inv_sqrt_dl) has no exact float32 key.  The tile ranks by
//            f64_proxy_key(score) and collects with collect_tile_f64 (every position at or above the bound, the
//            float64 scores in tile_d, overflow -> the exact re-run); topk_select_f64_kernel ranks in float64.
// WHERE (sim_where_tile_kernel): position i scores only where its bit of the mask row of query
// row_query[blockIdx.y] is set; the others are +0, as a position without the term, before the tile's bound is taken.
// DEEP: k > SA_TOPK_MAX, the tile's candidates from deep_tile_collect (classic: collect_tile_f64's deep bound).
template <int KIND, bool WHERE, bool DEEP>
__device__ __forceinline__ void sim_tile(const float *__restrict__ doc_rows, u64 doc_stride, const u64 *__restrict__ rows,
                                         const float *__restrict__ doc_lens, u64 n_pos, TileParams<KIND> p,
                                         const double *__restrict__ idf, u32 row0, const TopkCtx &t,
                                         u64 *__restrict__ tile_d, const WhereMask &wh, const u32 *__restrict__ row_query) {
    constexpr int PER_THREAD = SA_TILE_DOCS / SA_TERM_THREADS;
    __shared__ __align__(16) float s_out[KIND == SA_SIM_CLASSIC ? 4 : SA_TILE_DOCS];
    __shared__ u32 s_top[(SA_TERM_THREADS / 32) * 8];
    __shared__ u32 s_ncand, s_tile_max;
    const unsigned tid = threadIdx.x;
    const u32 tile = blockIdx.x, row = row0 + blockIdx.y;
    const u64 pos0 = (u64)tile * SA_TILE_DOCS;
    const float *__restrict__ counts = doc_rows + (u64)blockIdx.y * doc_stride;
    const double q_idf = idf[blockIdx.y];
    if constexpr (KIND == SA_SIM_BM25) p.idf = (float)q_idf;
    u32 my_max = 0;
    u32 key[PER_THREAD];          // classic: the proxy bits of the thread's positions
    u32 allow = ~0u;              // bit 4 j + e: position 4 g + e may rank
    if (WHERE) allow = where_word(wh, __ldg(row_query + blockIdx.y), tile);
    // thread tid owns positions 4g .. 4g+3 of the tile for g = tid + j * SA_TERM_THREADS (flush_tile_collect's layout)
#pragma unroll
    for (int j = 0; j < PER_THREAD / 4; j++) {
        const unsigned g = tid + j * SA_TERM_THREADS;
        float v[4];
#pragma unroll
        for (int e = 0; e < 4; e++) {
            const u64 i = pos0 + g * 4 + e;
            v[e] = 0.0f;
            if (i < n_pos && ((allow >> (j * 4 + e)) & 1u)) {
                const u64 doc = rows ? __ldg(rows + i) : i;
                const float tf = __ldg(counts + doc);
                if (tf > 0.0f) {
                    const float dl = __ldg(doc_lens + (KIND == SA_SIM_BM25 ? i : doc));
                    if constexpr (KIND == SA_SIM_BM25) {
                        v[e] = bm25_one(tf, dl, p);
                    } else if constexpr (KIND == SA_SIM_BM25_IMPACT) {
                        v[e] = sim_impact(tf, dl, p);
                    } else if constexpr (KIND == SA_SIM_BM25_LEGACY) {
                        const float sat = sim_legacy_sat(tf, dl, p);
                        v[e] = q_idf > 0.0 ? sat : (q_idf < 0.0 ? -sat : 0.0f);
                    } else {
                        v[e] = __uint_as_float(f64_proxy_key(sim_classic(q_idf, tf, dl)));
                    }
                    if (v[e] > 0.0f) my_max = max(my_max, __float_as_uint(v[e]));   // NaN and <= 0 never rank
                }
            }
            key[j * 4 + e] = v[e] > 0.0f ? __float_as_uint(v[e]) : 0u;
        }
        if (KIND != SA_SIM_CLASSIC) reinterpret_cast<float4 *>(s_out)[g] = make_float4(v[0], v[1], v[2], v[3]);
    }
    const u32 n_items = (u32)min((u64)SA_TILE_DOCS, n_pos - pos0);
    if constexpr (KIND == SA_SIM_CLASSIC) {
        collect_tile_f64<DEEP>(key, my_max, n_items, t, tile_d, row, tile, s_top, &s_ncand, &s_tile_max, [&](u32 local) {
            // the float64 score again, for the few candidates (cheaper than holding 32 doubles per thread)
            const u64 doc = rows ? __ldg(rows + pos0 + local) : pos0 + local;
            return sim_classic(q_idf, __ldg(counts + doc), __ldg(doc_lens + doc));
        });
    } else {
        // nothing reads the scores outside the tile: collect the candidates without storing the row
        flush_tile_collect<false, DEEP>(s_out, nullptr, t, row, tile, my_max, n_items,
                                  min((u32)SA_TERM_THREADS, (n_items + 3) / 4), s_top, &s_ncand, &s_tile_max);
    }
}

template <int KIND, bool DEEP>
__global__ void __launch_bounds__(SA_TERM_THREADS)
sim_tile_kernel(const float *__restrict__ doc_rows, u64 doc_stride, const u64 *__restrict__ rows,
                const float *__restrict__ doc_lens, u64 n_pos, TileParams<KIND> p, const double *__restrict__ idf,
                u32 row0, const TopkCtx t, u64 *__restrict__ tile_d) {
    sim_tile<KIND, false, DEEP>(doc_rows, doc_stride, rows, doc_lens, n_pos, p, idf, row0, t, tile_d, WhereMask{nullptr, 0},
                          nullptr);
}

// sa_score_batch_topk_sim with where_bits: sim_tile_kernel with a document mask over the positions.
template <int KIND, bool DEEP>
__global__ void __launch_bounds__(SA_TERM_THREADS)
sim_where_tile_kernel(const float *__restrict__ doc_rows, u64 doc_stride, const u64 *__restrict__ rows,
                      const float *__restrict__ doc_lens, u64 n_pos, TileParams<KIND> p, const double *__restrict__ idf,
                      u32 row0, const TopkCtx t, u64 *__restrict__ tile_d, const WhereMask wh,
                      const u32 *__restrict__ row_query) {
    sim_tile<KIND, true, DEEP>(doc_rows, doc_stride, rows, doc_lens, n_pos, p, idf, row0, t, tile_d, wh, row_query);
}

// One call's queries and scoring.
struct SimRun {
    int kind;                 // SA_SIM_*
    Bm25Params bm25;          // SA_SIM_BM25 (the idf is set per row, in the kernel)
    SimParams sim;            // the other kinds
    const u32 *terms, *term_starts;
    u32 slop;
    WhereMask where;          // bits NULL: no mask
    const u32 *tids(u32 q) const { return terms + term_starts[q]; }
    u32 n_terms(u32 q) const { return term_starts[q + 1] - term_starts[q]; }
};

int launch_sim_tiles(sa_index *ix, int kind, const float *counts, const u64 *rows, const float *doc_lens, u64 n_pos,
                     const Bm25Params &bm25, const SimParams &sim, const double *d_idf, u32 n, u32 row0,
                     const TopkCtx &t, u64 *tile_d, const WhereMask &wh, const u32 *d_row_query) {
    if (n == 0 || t.n_tiles == 0) return SA_OK;
    const u64 stride = sa_padded_docs(ix->n_docs);
    const dim3 grid(t.n_tiles, n);
    KernelTimer tm(ix, 1);
#define SA_SIM_TILES(KIND, P, DEEP)                                                                                 \
    if (wh.bits)                                                                                                    \
        sim_where_tile_kernel<KIND, DEEP><<<grid, SA_TERM_THREADS, 0, ix->stream>>>(counts, stride, rows, doc_lens, \
                                                                                    n_pos, P, d_idf, row0, t,       \
                                                                                    tile_d, wh, d_row_query);       \
    else                                                                                                            \
        sim_tile_kernel<KIND, DEEP><<<grid, SA_TERM_THREADS, 0, ix->stream>>>(counts, stride, rows, doc_lens, n_pos, \
                                                                              P, d_idf, row0, t, tile_d)
    const bool deep = t.k > SA_TOPK_MAX;
    if (kind == SA_SIM_BM25) {
        if (deep) { SA_SIM_TILES(SA_SIM_BM25, bm25, true); } else { SA_SIM_TILES(SA_SIM_BM25, bm25, false); }
    } else if (kind == SA_SIM_BM25_IMPACT) {
        if (deep) { SA_SIM_TILES(SA_SIM_BM25_IMPACT, sim, true); } else { SA_SIM_TILES(SA_SIM_BM25_IMPACT, sim, false); }
    } else if (kind == SA_SIM_BM25_LEGACY) {
        if (deep) { SA_SIM_TILES(SA_SIM_BM25_LEGACY, sim, true); } else { SA_SIM_TILES(SA_SIM_BM25_LEGACY, sim, false); }
    } else {
        if (deep) { SA_SIM_TILES(SA_SIM_CLASSIC, sim, true); } else { SA_SIM_TILES(SA_SIM_CLASSIC, sim, false); }
    }
#undef SA_SIM_TILES
    SA_CUDA(cudaGetLastError());
    tm.stop();
    ix->stats.topk_kernel_launches++;
    ix->stats.total_launches++;
    ix->stats.sim_instances |= 1ull << (2 * kind + (wh.bits ? 1 : 0));
    if (deep) ix->stats.deep_tiles += (u64)n * t.n_tiles;
    return SA_OK;
}

// The tile pass over ix->dense rows [0, n): row j holds the counts of call row call_row + j (its idf
// V.d_idf[call_row + j], its query V.d_row_query[call_row + j]), collected into row row0 + j of t.
static int launch_tiles(sa_index *ix, const SimRun &R, u32 call_row, u32 n, u32 row0, const TopkCtx &t) {
    ViewState &V = *ix->view;
    const bool view = ix->rows_active;
    return launch_sim_tiles(ix, R.kind, ix->dense.as<float>(), view ? ix->d_rows() : nullptr,
                            R.kind == SA_SIM_BM25 ? V.d_dl.as<float>() : ix->d_doc_lens.as<float>(),
                            view ? ix->n_rows : ix->n_docs, R.bm25, R.sim, V.d_idf.as<double>() + call_row, n, row0,
                            t, V.d_cand_d.as<u64>(), R.where, V.d_row_query.as<u32>() + call_row);
}

static int launch_select(sa_index *ix, int kind, const TopkCtx &t, u32 n_queries, const u32 *d_out_index) {
    ViewState &V = *ix->view;
    const u64 doc_base = ix->rows_active ? 0 : ix->doc_base;    // a view returns positions, an array doc ids
    if (kind == SA_SIM_CLASSIC)
        return launch_topk_select_f64(ix, t, V.d_cand_d.as<u64>(), n_queries, doc_base, V.d_keys.as<u64>(),
                                      V.d_scores.as<double>(), d_out_index);
    return launch_topk_select(ix, t, n_queries, doc_base, V.d_keys.as<u64>(), d_out_index);
}

// Term queries qs[0, n): their tf into ix->dense rows [0, n), then their tile pass (rows row0 + j of t, call
// rows call_row + j).  A view keeps or drops WHOLE docs (no position filter here), so a doc of the view has the same tf in the
// filtered list as in the index's own list: the term kernel runs on the own lists, with the tf table, and no
// compaction.  Docs outside the view get counts too; the tile pass never gathers them.
static int term_tiles(sa_index *ix, const SimRun &R, const u32 *qs, u32 n, u32 call_row, u32 row0,
                      const TopkCtx &t) {
    ViewState &V = *ix->view;
    if (n == 0) return SA_OK;
    std::vector<TermQuery> tqs(n);
    for (u32 j = 0; j < n; j++) tqs[j] = make_term_query(ix, R.tids(qs[j])[0], 0.0f);
    int rc;
    if ((rc = ix->dense.reserve((size_t)n * sa_padded_docs(ix->n_docs) * sizeof(float)))) return rc;
    SA_CUDA(cudaMemcpyAsync(V.d_tq.p, tqs.data(), n * sizeof(TermQuery), cudaMemcpyHostToDevice, ix->stream));
    TopkCtx none;
    memset(&none, 0, sizeof(none));
    TermBatchArgs a = make_term_args(ix, V.d_tq.as<TermQuery>(), make_bm25(0, 1, 1, 0, ix->doc_lens_nonneg), none);
    a.mode = TERM_MODE_TF;
    if ((rc = launch_term_batch(ix, a, n))) return rc;
    return launch_tiles(ix, R, call_row, n, row0, t);
}

// Phrase / slop queries qs[0, n), one at a time: raw counts into ix->dense row 0 (sa_phrase_row), then the query's
// tile pass (row row0 + j of t, call row call_row + j).  On a view, one filter pass over every list of the n queries comes
// first; a missing query has no filtered lists, and sa_phrase_row reads none for it.
static int phrase_tiles(sa_index *ix, const SimRun &R, const u32 *qs, u32 n, u32 call_row, u32 row0,
                        const TopkCtx &t) {
    const bool view = ix->rows_active;
    std::vector<u32> ftids, fstart;
    std::vector<u64> f_offs, f_lens;
    int rc;
    for (u32 j = 0; j < n && view; j++) {
        const u32 *tids = R.tids(qs[j]);
        const u32 nt = R.n_terms(qs[j]);
        u64 offs[SA_MAX_PHRASE_TERMS], lens[SA_MAX_PHRASE_TERMS], dirs[SA_MAX_PHRASE_TERMS];
        bool missing, literal;
        if ((rc = sa_resolve_terms(ix, tids, nt, offs, lens, dirs, &missing, &literal))) return rc;
        fstart.push_back((u32)ftids.size());
        if (!missing) ftids.insert(ftids.end(), tids, tids + nt);
    }
    if (!ftids.empty() && (rc = sa_filter_terms_mask(ix, ftids.data(), (u32)ftids.size(), ix->d_row_mask(), 0,
                                                     SA_ALL_BITS, false, f_offs, f_lens, nullptr))) return rc;
    for (u32 j = 0; j < n; j++) {
        bool scored;
        if ((rc = sa_phrase_row(ix, R.tids(qs[j]), R.n_terms(qs[j]), R.slop, view ? f_offs.data() + fstart[j] : nullptr,
                                view ? f_lens.data() + fstart[j] : nullptr, nullptr, &scored)) ||
            (rc = launch_tiles(ix, R, call_row + j, 1, row0 + j, t))) return rc;
    }
    return SA_OK;
}

// keys (the classic scores, the overflow flags) to the host in one copy each and one synchronise
static int download(sa_index *ix, bool classic, u32 nq, u32 k, std::vector<u64> &keys, std::vector<double> &scores,
                    std::vector<u32> *ovf) {
    ViewState &V = *ix->view;
    const size_t nk = (size_t)nq * k;
    int rc;
    if ((rc = ix->h_pinned.reserve(nk * (sizeof(u64) + sizeof(double)) + (size_t)nq * sizeof(u32)))) return rc;
    u64 *h_keys = ix->h_pinned.as<u64>();
    double *h_scores = (double *)(h_keys + nk);
    u32 *h_ovf = (u32 *)(h_scores + nk);
    SA_CUDA(cudaMemcpyAsync(h_keys, V.d_keys.p, nk * sizeof(u64), cudaMemcpyDeviceToHost, ix->stream));
    if (classic)
        SA_CUDA(cudaMemcpyAsync(h_scores, V.d_scores.p, nk * sizeof(double), cudaMemcpyDeviceToHost, ix->stream));
    if (ovf) SA_CUDA(cudaMemcpyAsync(h_ovf, V.d_ovf.p, nq * sizeof(u32), cudaMemcpyDeviceToHost, ix->stream));
    SA_CUDA(cudaStreamSynchronize(ix->stream));
    keys.assign(h_keys, h_keys + nk);
    if (classic) scores.assign(h_scores, h_scores + nk);
    if (ovf) ovf->assign(h_ovf, h_ovf + nq);
    return SA_OK;
}

int sa_where_check(const uint32_t *where_bits, uint64_t where_n, uint64_t where_stride, u64 n) {
    if (!where_bits) return SA_OK;
    SA_CHECK(where_n == n, "the mask covers %llu docs, the call ranks %llu", (unsigned long long)where_n,
             (unsigned long long)n);
    SA_CHECK(where_stride == 0 || where_stride == SA_WHERE_WORDS(n),
             "where_stride must be 0 (one mask) or %llu words (a mask per query), not %llu",
             (unsigned long long)SA_WHERE_WORDS(n), (unsigned long long)where_stride);
    return SA_OK;
}

int sa_where_upload(sa_index *ix, DevBuf &buf, const uint32_t *where_bits, u64 n, uint64_t where_stride, u32 n_queries,
                    WhereMask *out) {
    *out = WhereMask{nullptr, where_stride};
    if (!where_bits) return SA_OK;
    const size_t bytes = (where_stride ? (size_t)n_queries : 1) * SA_WHERE_WORDS(n) * sizeof(u32);
    int rc;
    if ((rc = buf.reserve(std::max<size_t>(bytes, 4)))) return rc;
    SA_CUDA(cudaMemcpyAsync(buf.p, where_bits, bytes, cudaMemcpyHostToDevice, ix->stream));
    out->bits = buf.as<u32>();
    return SA_OK;
}

extern "C" int sa_score_batch_topk_sim(sa_index *ix, int kind, const uint32_t *terms, const uint32_t *term_starts,
                                       const double *idf, uint32_t n_queries, uint32_t slop,
                                       const float *view_doc_lens, double avg_doc_len, double k1, double b,
                                       uint32_t k, const uint32_t *where_bits, uint64_t where_n,
                                       uint64_t where_stride, uint32_t *out_ids, double *out_scores) {
    SA_CHECK(ix, "index is NULL");
    SA_CHECK(n_queries == 0 || (terms && term_starts && idf && out_ids && out_scores), "NULL argument");
    SA_CHECK(kind == SA_SIM_BM25 || kind == SA_SIM_BM25_IMPACT || kind == SA_SIM_BM25_LEGACY || kind == SA_SIM_CLASSIC,
             "unknown similarity %d", kind);
    SA_CHECK(k >= 1 && k <= SA_TOPK_DEEP_MAX, "k must be in [1, %d]", SA_TOPK_DEEP_MAX);
    const bool classic = kind == SA_SIM_CLASSIC;
    int rc;
    for (u32 q = 0; q < n_queries; q++) {
        const u32 nt = term_starts[q + 1] - term_starts[q];
        SA_CHECK(nt >= 1 && nt <= SA_MAX_PHRASE_TERMS, "query %u: bad number of terms", q);
        if ((rc = sa_check_term_ids(ix, terms + term_starts[q], nt))) return rc;
        SA_CHECK((kind != SA_SIM_BM25_LEGACY && !classic) || std::isfinite(idf[q]), "query %u: idf is not finite", q);
    }
    std::lock_guard<std::mutex> g(ix->mu);
    const bool view = ix->rows_active;
    SA_CHECK(view || kind != SA_SIM_BM25, "no row filter installed (sa_index_set_rows)");
    const u64 n_pos = view ? ix->n_rows : ix->n_docs;
    SA_CHECK(n_pos < 0xFFFFFFFFull, "the array must have fewer than 2^32 - 1 rows");
    SA_CHECK(kind != SA_SIM_BM25 || n_pos == 0 || view_doc_lens, "view_doc_lens is NULL");
    if ((rc = sa_where_check(where_bits, where_n, where_stride, n_pos))) return rc;
    SA_CUDA(cudaSetDevice(ix->device));
    const size_t nk = (size_t)n_queries * k;
    for (size_t i = 0; i < nk; i++) { out_ids[i] = SA_NO_DOC; out_scores[i] = 0.0; }
    // BM25 (its float32 avgdl, as it runs), impact and legacy score zeros at avgdl == 0 (similarity.py:49-50, 66-67);
    // classic has no such branch
    const bool zero_avgdl = kind == SA_SIM_BM25 ? (float)avg_doc_len == 0.0f : avg_doc_len == 0.0;
    if (n_queries == 0 || n_pos == 0 || (!classic && zero_avgdl)) return SA_OK;
    if (!ix->view) ix->view.reset(new ViewState());
    ViewState &V = *ix->view;
    // BM25 exactly as ops.bm25_score -> sa_op_bm25_score sets it up: float32 parameters, `1 - b` in float32
    SimRun R{kind, make_bm25(0.0f, (float)avg_doc_len, (float)k1, (float)b, false),
             make_sim_params(avg_doc_len, k1, b), terms, term_starts, slop, WhereMask{nullptr, 0}};
    const u32 n_tiles = sa_n_tiles(n_pos), slots = classic ? sa_topk_slots_f64(k, 256u) : sa_topk_slots(k);
    const RowPlan plan = sa_plan_rows(ix->n_docs, term_starts, n_queries);
    const u32 chunk = plan.chunk;
    const std::vector<u32> &row_query = plan.row_query;
    // Every buffer is reserved before the first write: DevBuf::reserve does not keep the contents.  ix->dense is the
    // exception -- each step reserves it and consumes what it wrote before the next reserve.
    if (kind == SA_SIM_BM25 && (rc = V.d_dl.reserve(n_pos * sizeof(float)))) return rc;
    if ((rc = V.d_tq.reserve((size_t)chunk * sizeof(TermQuery)))) return rc;
    if ((rc = V.d_idf.reserve((size_t)n_queries * sizeof(double)))) return rc;
    if ((rc = V.d_row_query.reserve((size_t)n_queries * sizeof(u32)))) return rc;
    if ((rc = V.d_ovf.reserve((size_t)n_queries * sizeof(u32)))) return rc;
    if ((rc = V.d_keys.reserve(nk * sizeof(u64)))) return rc;
    if ((rc = ix->cand.reserve(cand_bytes(n_tiles, chunk, slots)))) return rc;
    if (classic && (rc = V.d_scores.reserve(nk * sizeof(double)))) return rc;
    if (classic && (rc = V.d_cand_d.reserve((size_t)chunk * n_tiles * slots * sizeof(u64)))) return rc;
    if ((rc = sa_where_upload(ix, V.d_where, where_bits, n_pos, where_stride, n_queries, &R.where))) return rc;

    std::vector<double> row_idf(n_queries);
    for (u32 r = 0; r < n_queries; r++) row_idf[r] = idf[row_query[r]];
    if (kind == SA_SIM_BM25)
        SA_CUDA(cudaMemcpyAsync(V.d_dl.p, view_doc_lens, n_pos * sizeof(float), cudaMemcpyHostToDevice, ix->stream));
    SA_CUDA(cudaMemcpyAsync(V.d_idf.p, row_idf.data(), n_queries * sizeof(double), cudaMemcpyHostToDevice, ix->stream));
    SA_CUDA(cudaMemcpyAsync(V.d_row_query.p, row_query.data(), n_queries * sizeof(u32), cudaMemcpyHostToDevice, ix->stream));
    SA_CUDA(cudaMemsetAsync(V.d_ovf.p, 0, n_queries * sizeof(u32), ix->stream));

    for (const RowChunk &C : plan.chunks) {
        const u32 Q = C.n_term + C.n_phrase;
        const u32 *qs = row_query.data() + C.row0;
        TopkCtx t = make_topk_ctx(ix->cand.p, n_tiles, Q, slots, k, V.d_ovf.as<u32>() + C.row0);
        if ((rc = phrase_tiles(ix, R, qs + C.n_term, C.n_phrase, C.row0 + C.n_term, C.n_term, t))) return rc;
        if ((rc = term_tiles(ix, R, qs, C.n_term, C.row0, 0, t))) return rc;
        if ((rc = launch_select(ix, kind, t, Q, V.d_row_query.as<u32>() + C.row0))) return rc;
    }
    std::vector<u64> keys;
    std::vector<double> scores;
    std::vector<u32> ovf;
    if ((rc = download(ix, classic, n_queries, k, keys, scores, &ovf))) return rc;
    bool redone = false;
    for (u32 r = 0; r < n_queries; r++) {
        if (!ovf[r]) continue;
        // exact re-run of one query: a candidate slot per position of the tile cannot overflow
        if ((rc = ix->cand.reserve(cand_bytes(n_tiles, 1, SA_TILE_DOCS)))) return rc;
        if (classic && (rc = V.d_cand_d.reserve((size_t)n_tiles * SA_TILE_DOCS * sizeof(u64)))) return rc;
        SA_CUDA(cudaMemsetAsync(V.d_ovf.as<u32>() + r, 0, sizeof(u32), ix->stream));
        TopkCtx t = make_topk_ctx(ix->cand.p, n_tiles, 1, SA_TILE_DOCS, k, V.d_ovf.as<u32>() + r);
        const bool term = R.n_terms(row_query[r]) == 1;
        if ((rc = (term ? term_tiles : phrase_tiles)(ix, R, &row_query[r], 1, r, 0, t))) return rc;
        if ((rc = launch_select(ix, kind, t, 1, V.d_row_query.as<u32>() + r))) return rc;
        redone = true;
    }
    if (redone && (rc = download(ix, classic, n_queries, k, keys, scores, nullptr))) return rc;
    for (u32 q = 0; q < n_queries; q++)
        for (u32 i = 0; i < k; i++) {
            const size_t j = (size_t)q * k + i;
            const u64 key = keys[j];
            if (key == 0) continue;
            out_ids[j] = 0xFFFFFFFFu - (u32)key;
            float f;
            const u32 bits = (u32)(key >> 32);
            memcpy(&f, &bits, sizeof(f));
            if (kind == SA_SIM_BM25_LEGACY) out_scores[j] = std::fabs(idf[q]) * (double)f;   // f = sign(idf) * sat
            else if (classic) out_scores[j] = scores[j];
            else out_scores[j] = f;                                                      // BM25 and impact
        }
    return SA_OK;
}
