// sa_phrase.cuh -- declarations for the phrase (slop == 0) path.
#pragma once
#include "sa_common.cuh"
#include "sa_term.cuh"

#define SA_PHRASE_THREADS 256
#define SA_PHRASE_MODE_LR 0      // left-to-right chain  (reference middle_out.py:96-122)
#define SA_PHRASE_MODE_RL 1      // right-to-left chain  (reference middle_out.py:125-151)
#define SA_PHRASE_MODE_MID 2     // middle-out: LR on [0,split), RL on [split,n), then and/min (:163-168)

// One phrase query against one shard.
struct PhraseQuery {
    u32 n_terms;
    u32 mode;
    u32 split;            // SA_PHRASE_MODE_MID only
    u32 same_guess;       // bit s set => step s is speculated to take the "same term" branch
    u64 off[SA_MAX_PHRASE_TERMS];   // word offset of each term's list (relative to `words`)
    u64 len[SA_MAX_PHRASE_TERMS];
    u64 dir_plus1[SA_MAX_PHRASE_TERMS];   // 1 + offset of the list's tile directory in d_tile_dir; 0 = none
    float idf;
    u32 use_conj;         // batches: 1 = the conjunction regime runs it (sa_phrase_use_conjunction); the kernels ignore it
};

struct PhraseStats {      // per query, accumulated over all chunks (global atomics)
    u32 n_inner[SA_MAX_PHRASE_TERMS];   // equal-header pairs seen at step s
    u32 n_diff[SA_MAX_PHRASE_TERMS];    // ... of which lhs word != rhs word
    u32 overflow;                        // 1: scratch arena exhausted; 2: conjunction regime gave up (dense candidates) -> search regime
    u32 n_match;                         // docs with a non-zero phrase count (M of SURVEY 8d's B_phrase)
    unsigned long long n_cont;           // continuation words written over all steps (sum of C_s)
};

// Optional dump of one CTA's final lists (per-op parity export; needs n_chunks == 1).
struct PhraseDump {
    u64 *cont;        // continuation words of the last step
    u64 *n_cont;
    u64 *docs;        // doc << 32 | count of the last step (BEFORE and/min with earlier steps)
    u64 *n_docs;
};

struct PhraseArgs {
    const u64 *words;           // lists live at words + off
    const float *doc_lens;
    u64 n_docs, doc_base;
    const PhraseQuery *queries;
    PhraseStats *stats;
    float *out;                 // [Q][out_stride], pre-zeroed
    u64 out_stride;
    u32 n_chunks;               // doc-range chunks per query (grid.x)
    u64 docs_per_chunk;
    u64 *arena;                 // scratch bump arena (u64 words)
    unsigned long long *arena_used;
    u64 arena_cap;
    Bm25Params bm25;
    int score;                  // 0: write phrase freqs, 1: BM25 (sparse)
    PhraseDump dump;
    // Every CTA writes the dense tiles of its doc range itself (zeros + matches) -- no separate
    // zero-fill pass -- and, when topk.k != 0, collects their top-k candidates on the way.
    // docs_per_chunk is a multiple of SA_TILE_DOCS.  topk.overflow / tile arrays are indexed by
    // row = topk_row0 + query.
    TopkCtx topk;
    u32 topk_row0;
    const u32 *tile_dir;        // word tile directories (sa_index::d_tile_dir) or NULL (filtered lists)
    const u32 *qsel;            // launch only these queries (indices into `queries`); NULL = all, in order
};

// Which queries of a batch run in which regime (device index lists into the PhraseQuery array)
struct PhraseSplit {
    const u32 *d_search;
    u32 n_search;
    const u32 *d_conj;
    u32 n_conj;
};

// Doc ranges of a phrase or span launch: n_chunks per query, each docs_per_chunk docs (whole tiles) long.
struct DocChunks {
    u32 n_chunks;
    u64 docs_per_chunk;
};

int launch_phrase(sa_index *ix, const PhraseArgs &a, u32 n_queries);
void sa_phrase_plan(PhraseQuery &pq, const u32 *term_ids);
// A planned descriptor.  missing: some term matches nothing -- every length is zeroed (the rows stay zero).
// dirs: tile directory offsets (SA_NO_DIR = none), or NULL for lists outside the index.
PhraseQuery make_phrase_query(const u32 *term_ids, u32 n, const u64 *offs, const u64 *lens, const u64 *dirs,
                              float idf, bool missing);
bool sa_phrase_guess_ok(PhraseQuery &pq, const PhraseStats &st);
u64 sa_phrase_arena_words(const PhraseQuery &pq, u32 n_chunks);
int sa_phrase_enqueue(sa_index *ix, const PhraseQuery *d_pqs, PhraseStats *d_stats, u32 Q,
                      float *dense_rows, u64 stride, DocChunks chunks, u64 *d_arena,
                      unsigned long long *d_arena_used, u64 arena_words, int score, const Bm25Params &p,
                      const TopkCtx *topk, u32 topk_row0, const PhraseSplit *split);
DocChunks phrase_doc_chunks(const sa_index *ix, u32 n_queries, u32 ctas_per_sm);
bool sa_phrase_use_conjunction(const PhraseQuery &pq, u64 n_docs);
int sa_phrase_run_sync(sa_index *ix, std::vector<PhraseQuery> &pqs, const u64 *d_words,
                       int score, const Bm25Params &p, PhraseDump dump, bool allow_conj);
// One phrase (slop 0) or span (slop > 0) query's per-doc counts into ix->dense row 0, synchronously.  The caller
// holds ix->mu and has checked n_terms and the term ids.  Lists: the index's own (f_offs == NULL), or the filtered
// copies in ix->filt at f_offs / f_lens (sa_filter_terms / sa_filter_terms_mask).  A missing query (sa_resolve_terms)
// gets a zero row without a launch and reads no f_offs.  bm25: NULL for raw counts; otherwise, where bm25->sparse_ok,
// a slop-0 query is scored in the phrase kernels under *bm25 (its idf included).  *scored: the row holds BM25 scores
// (that case, or a missing query's zero row under sparse_ok parameters) rather than counts.
int sa_phrase_row(sa_index *ix, const u32 *term_ids, u32 n_terms, u32 slop, const u64 *f_offs, const u64 *f_lens,
                  const Bm25Params *bm25, bool *scored);
