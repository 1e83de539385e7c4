// sa_span.cuh -- declarations for the slop > 0 ("span search") path.
#pragma once
#include "sa_common.cuh"

// One span query against one shard.  All offsets index the batch-wide scratch arenas.
struct SpanQuery {
    u32 n_terms;
    u32 slop;
    u32 shortest;                       // index of the shortest list (candidate generator)
    u32 literal;                        // 1 = the reference's header-0 underflow corner (replayed literally)
    float idf;
    u32 n_ctas;                         // generator CTAs of this query (ceil(len[shortest] / 256))
    u64 rec_off;                        // generator records: rec[rec_off + gen * n_terms + t]
    u64 cta_off;                        // per-(term, generator CTA) compaction records
    u64 off[SA_MAX_PHRASE_TERMS];       // term lists in `words`
    u64 len[SA_MAX_PHRASE_TERMS];
    u64 dir_off[SA_MAX_PHRASE_TERMS];   // tile directory of the list, or SA_NO_DIR
    u64 s_off[SA_MAX_PHRASE_TERMS];     // sliced-list region of term t in the word arena
    u64 g_off[SA_MAX_PHRASE_TERMS];     // group-start region of term t in the u32 arena
    u64 s_cap[SA_MAX_PHRASE_TERMS];
    u64 m_off;                          // match records (one per phase-2 iteration) of this query
    u64 cand_off;                       // candidate-doc bitmap of this query in the u32 bitmap arena, or SA_NO_DIR
};

struct SpanCounts {                      // written by phase 1, read by phase 2
    u32 n_sliced[SA_MAX_PHRASE_TERMS];
    u32 n_groups[SA_MAX_PHRASE_TERMS];
    u32 overflow;
    u32 unsorted;                        // the match records are not in doc order (misaligned doc groups)
    u32 undefined;                       // span-table overflows the reference leaves undefined
};

// Host-side plan of a batch of span queries: descriptors + scratch layout.
struct SpanPlan {
    std::vector<SpanQuery> qs;
    u64 words_total = 0, groups_total = 0, rec_total = 0, cta_total = 0, match_total = 0;
    u32 max_ctas = 0;
    u64 max_shortest = 0;
    bool any_literal = false;
    // conjunction prefilter (balanced lists): queries whose candidate-doc bitmap is built before phase 1
    std::vector<u32> conj;
    u64 cand_total = 0;                 // u32 words of bitmap arena
};

// Appends one query.  dir_offs may be NULL (no tile directories, e.g. filtered lists).
// n_docs != 0 and every list has a directory: balanced queries get the conjunction prefilter.
void sa_span_plan_add(SpanPlan &plan, const u64 *offs, const u64 *lens, const u64 *dir_offs, u32 n_terms,
                      u32 slop, float idf, bool literal, u64 n_docs = 0);
size_t sa_span_scratch_bytes(const SpanPlan &plan);
// Enqueues the whole plan.  d_qs: device copy of plan.qs; d_counts: SpanCounts[Q] (zeroed here).
// topk != NULL (batched path): nothing is pre-zeroed; the matches become per-query records and one
// tile pass writes the dense rows (zeros + BM25-scored matches, sa_ensure_norm must have run) and
// collects the top-k candidates (rows topk_row0 + q).  topk == NULL: raw counts are ADDED into the
// rows, which are zeroed here.
int sa_span_enqueue(sa_index *ix, const u64 *d_lists, const SpanPlan &plan, const SpanQuery *d_qs,
                    SpanCounts *d_counts, void *d_scratch, float *dense_rows, u64 stride,
                    const struct TopkCtx *topk = nullptr, u32 topk_row0 = 0);
// One query, synchronously, into ix->dense row 0 (raw counts).  sa_phrase_row runs it for a query given by term ids;
// the batch re-run calls it with a stored descriptor.
int sa_span_run(sa_index *ix, const u64 *d_lists, const u64 *offs, const u64 *lens, const u64 *dir_offs,
                uint32_t n_terms, uint32_t slop, bool literal);
// "Every list starts with a word at (doc 0, block 0)" for lists that live in d_lists (device check, one synchronise
// per list): the literal flag of filtered lists, for sa_phrase_row.
int sa_span_is_literal(sa_index *ix, const u64 *d_lists, const u64 *offs, const u64 *lens, u32 n_terms, bool *out);
