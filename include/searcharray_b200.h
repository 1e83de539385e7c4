/*
 * searcharray_b200.h -- C ABI of libsearcharray_b200.so (sm_90a CUDA kernels, H100).
 *
 * Drop-in boundary for SearchArray's scoring hot path (SURVEY.md section 8b).  The
 * reference (softwaredoug/searcharray, paths below relative to its repo root) has no C
 * ABI of its own: its "operator interface" is a set of Cython `def`s taking host numpy
 * arrays.  Replacing those one-for-one would bounce every intermediate over PCIe, so
 * the boundary sits one level up, at what SearchArray.score / .termfreqs call on
 * `self.posns` and `similarity` (searcharray/postings.py:607-708).
 *
 * Conventions: every function returns 0 on success, non-zero on error (text via
 * sa_last_error(), thread-local).  Host pointers are borrowed for the duration of the
 * call only.  Plain pointers and sizes -- no torch / numpy types.  A handle may be used
 * from several host threads (calls on one handle serialise on an internal mutex, the
 * reference's tests fire .score from 3 threads: test/test_tmdb.py:285-312).
 *
 * Posting word layout (searcharray/roaringish/roaringish.py:30-35):
 *     bits 63..36 doc id (28 b) | 35..18 block = posn / 18 (18 b) | 17..0 bitmap of posn % 18
 * Words of one term are sorted ascending and header-unique (header = bits 63..18).
 */
#ifndef SEARCHARRAY_B200_H
#define SEARCHARRAY_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct sa_index sa_index;

#define SA_OK 0
#define SA_ERR_CUDA 1
#define SA_ERR_ARG 2
#define SA_ERR_NOMEM 3
#define SA_ERR_NCCL 4

#define SA_NO_TERM 0xFFFFFFFFu      /* "token not in the term dictionary" (TermMissingError) */
#define SA_NO_DOC 0xFFFFFFFFu       /* empty top-k slot */
/* The largest k of the batched top-k entry points: sa_score_batch_topk, sa_batch_upload, the boolean ones,
 * sa_score_batch_topk_sim (every kind), sa_multi_topk and sa_score_batch_topk_allgather take 1 <= k <=
 * SA_TOPK_DEEP_MAX. */
#define SA_TOPK_DEEP_MAX 1024
#define SA_MAX_PHRASE_TERMS 16
#define SA_ALL_BITS 0xFFFFFFFFFFFFFFFFull

/* ----------------------------------------------------------------------- misc */
const char *sa_last_error(void);
int sa_device_count(int *n_out);
/* Pinned host memory for result vectors (D2H of a dense float32[N] at full PCIe rate). */
int sa_host_alloc(void **ptr_out, uint64_t bytes);
int sa_host_free(void *ptr);
/* Device buffers the library holds right now in this process, and their bytes (every index, multi-field handle and
 * in-flight call).  Returns to its earlier value once everything created since is destroyed. */
int sa_device_allocations(uint64_t *live_buffers, uint64_t *live_bytes);

/* ---------------------------------------------------------------------- index
 * Uploads one shard of the inverted index into HBM.  Replaces the host-side state the
 * hot path reads: ArrayDict.data / .metadata (searcharray/phrase/memmap_arrays.py:15-53),
 * SearchArray.doc_lens (postings.py:293-299) and the docfreq cache
 * (searcharray/phrase/middle_out.py:511-528, warm() :337-342: per-term df is computed on
 * the device at upload).
 *   words        all terms' posting words, concatenated          [n_words]
 *   term_offsets / term_lengths   slice of `words` per term id    [n_terms]
 *   doc_lens     float32 length of every doc in the shard         [n_docs]
 *   doc_base     global id of the shard's first doc; the shard owns [doc_base, doc_base+n_docs)
 *                and every word's doc id must lie in that range (doc-range sharding, sec. 8e)
 * A word whose block ((w >> 18) & 0x3FFFF) exceeds MAX_POSN / 18 = 14,563 (MAX_POSN = 2^18 - 1, the reference's
 * per-doc position limit, roaringish.py:86) is SA_ERR_ARG: a doc's term frequency must fit the index's 19-bit counts.
 */
int sa_index_create(const uint64_t *words, uint64_t n_words,
                    const uint64_t *term_offsets, const uint64_t *term_lengths, uint32_t n_terms,
                    const float *doc_lens, uint64_t n_docs, uint64_t doc_base,
                    int device, sa_index **index_out);
int sa_index_destroy(sa_index *index);
/* How sa_index_create moved the posting words to HBM (SURVEY 8f-2): 0 = plain copy (small indexes), 1 = the host
 * range -- e.g. the np.memmap of the reference's MemoryMappedArrays .dat file (phrase/memmap_arrays.py:145-208) --
 * was page-locked in place with cudaHostRegister and DMA'd at PCIe rate, 2 = pipelined through pinned bounce
 * buffers because the range could not be registered. */
int sa_index_upload_mode(const sa_index *index, int *mode_out);
/* 1 when a batch of sa_batch_upload / sa_score_batch_topk has written its term queries' dense rows to compressible
 * device memory.  The L2 then compresses their all-zero lines on the way to DRAM, and the term scan walks those rows
 * in small query groups.  0 when no batch has had term queries yet, or when every row is in plain
 * cudaMalloc memory: the device has no compression support, the driver does not grant it, or the process started
 * with SA_DENSE_PLAIN=1.  The results are the same bits either way. */
int sa_index_dense_compressible(const sa_index *index, int *compressible_out);
int sa_index_info(const sa_index *index, uint64_t *n_docs, uint64_t *n_words,
                  uint32_t *n_terms, uint64_t *device_bytes);

/* PosnBitArray.docfreq (middle_out.py:521-528): distinct docs of the term in this shard. */
int sa_docfreq(sa_index *index, uint32_t term_id, uint64_t *df_out);

/* Restricts subsequent queries to a subset of the shard's docs -- the sliced-array
 * semantics of SearchArray.__getitem__ / FilteredPosns (postings.py:344-358,
 * middle_out.py:291-317).  `rows` = sorted local doc indices (0-based in the shard);
 * results then have n_rows entries, in `rows` order.  rows == NULL clears the filter. */
int sa_index_set_rows(sa_index *index, const uint64_t *rows, uint64_t n_rows);
/* docfreq on the filtered postings (reference quirk iii: df is taken on the slice). */
int sa_docfreq_rows(sa_index *index, uint32_t term_id, uint64_t *df_out);
/* The same for n_terms terms in one device pass (what SearchArray.docfreq returns on the slice for each of them;
 * PosnBitArray.docfreq on FilteredPosns, middle_out.py:521-528 and 291-317).  SA_NO_TERM -> 0; no row filter
 * installed -> the shard's df.  Counts the docs of every list that lie in the filter; writes no filtered list. */
int sa_docfreq_rows_batch(sa_index *index, const uint32_t *term_ids, uint32_t n_terms, uint64_t *df_out);

/* ------------------------------------------------------------------ term path
 * SearchArray.termfreqs(token) (postings.py:607-638): popcount64_reduce + as_dense fused;
 * out = float32[n_docs] on the host (or [n_rows] when a row filter is set).
 * min_payload/max_payload: RoaringishEncoder.slice's block filter exactly as the reference
 * applies it (roaringish.py:267-282 + roaringish_ops.pyx:46-68: compares the UNSHIFTED
 * masked word with min_posn/18 and max_posn/18); pass 0 and SA_ALL_BITS for "no filter". */
int sa_termfreqs(sa_index *index, uint32_t term_id,
                 uint64_t min_payload, uint64_t max_payload, float *out_host);

/* SearchArray.score(token, similarity=bm25_similarity(k1, b)) (postings.py:652-680 +
 * similarity.py:24-38 + bm25/bm25.pyx:11-41): termfreqs + BM25 fused in one kernel.
 * idf is computed by the host exactly as compute_idf does (similarity.py:19-21, float64 ->
 * C float); avg_doc_len, k1, b as the reference passes them to bm25_score. */
int sa_score_term(sa_index *index, uint32_t term_id, float idf, float avg_doc_len,
                  float k1, float b, uint64_t min_payload, uint64_t max_payload,
                  float *out_host);

/* ---------------------------------------------------------------- phrase path
 * SearchArray._phrase_freq / PosnBitArray.phrase_freqs (postings.py:689-708,
 * middle_out.py:418-446): slop == 0 -> compute_phrase_freqs (middle-out bigram chain,
 * phrase/bigram_freqs.py); slop > 0 -> span_search (phrase/spans.py, roaringish/spans.pyx).
 * Any term id == SA_NO_TERM -> zeros.  n_terms >= 2. */
int sa_phrase_freqs(sa_index *index, const uint32_t *term_ids, uint32_t n_terms, uint32_t slop,
                    uint64_t min_payload, uint64_t max_payload, float *out_host);
int sa_score_phrase(sa_index *index, const uint32_t *term_ids, uint32_t n_terms, uint32_t slop,
                    float idf, float avg_doc_len, float k1, float b,
                    uint64_t min_payload, uint64_t max_payload, float *out_host);

/* ------------------------------------------------------- batched, HBM-resident
 * The queries/sec path: scores stay in HBM, only the top-k leaves the device.
 * Query q = terms[term_starts[q] .. term_starts[q+1]) (1 term = BM25 term query, >= 2 =
 * phrase with `slop`), idf[q] as above.  For every query the dense float32[n_docs] score
 * vector is produced in HBM exactly as sa_score_term / sa_score_phrase would, then reduced
 * to the k best (score desc, doc id asc; only score > 0; empty slots = SA_NO_DOC / 0).
 * out_docs[q*k + i] are GLOBAL doc ids (doc_base added).  The reference idiom this
 * replaces is np.argpartition(scores, -N) (searcharray/utils/sort.py:24). */
int sa_score_batch_topk(sa_index *index, const uint32_t *terms, const uint32_t *term_starts,
                        const float *idf, uint32_t n_queries, uint32_t slop,
                        float avg_doc_len, float k1, float b, uint32_t k,
                        uint32_t *out_docs, float *out_scores);
/* The batched top-k on a sliced array, and under the other similarities (kind = SA_SIM_*, below): the top k of
 * SearchArray.score(q, similarity=...) on the view the installed row filter selects (sa_index_set_rows;
 * postings.py:652-680 on FilteredPosns, middle_out.py:291-317) or, with no filter, on the whole array.  Counts as
 * SearchArray.termfreqs (the filtered postings on a view); avg_doc_len the parent's.
 *   SA_SIM_BM25 (on a view only; the unsliced array takes sa_score_batch_topk): BM25 as sa_score_term computes it,
 *     idf[q] the float32 idf of the slice's document frequencies (sa_docfreq_rows_batch), widened;
 *     view_doc_lens = float32[n_rows], the lengths the view's BM25 uses (bm25/bm25.pyx:28-41); avg_doc_len, k1 and b
 *     are rounded to float32.
 *   The others: sa_op_similarity over the query's counts; doc lengths the index's own (gathered through the row
 *     filter: SearchArray.doclengths()), view_doc_lens is ignored; idf[q] the similarity's own float64 idf (must be
 *     finite for SA_SIM_BM25_LEGACY and SA_SIM_CLASSIC; unused by SA_SIM_BM25_IMPACT); avg_doc_len, k1, b the
 *     Python values (numpy's float32 promotion is applied here).
 * avg_doc_len == 0 -> nothing ranks, except under SA_SIM_CLASSIC.  out_scores are float64 (the float32 BM25 and
 * impact scores widened).  Only scores > 0 rank (+inf does, NaN never); order score desc, then id asc
 * (np.argpartition as above); empty slots SA_NO_DOC / 0.  Ids: positions in the view, or GLOBAL doc ids (doc_base
 * added) on an unsliced array; fewer than 2^32 - 1 of them.  where_bits / where_n / where_stride: a document mask
 * over the positions it ranks (a view's, or the array's docs), as below; where_bits NULL: no mask. */
int sa_score_batch_topk_sim(sa_index *index, int kind, const uint32_t *terms, const uint32_t *term_starts,
                            const double *idf, uint32_t n_queries, uint32_t slop, const float *view_doc_lens,
                            double avg_doc_len, double k1, double b, uint32_t k, const uint32_t *where_bits,
                            uint64_t where_n, uint64_t where_stride, uint32_t *out_ids, double *out_scores);
/* A document mask for the batched top-k (sa_score_batch_topk_sim and the boolean entry points below): the result is
 * the top k of where(mask_q, S_q, 0), S_q being the scores the call without a mask ranks for query q, under the same
 * selection rule.  The mask never changes a score -- idf, document frequencies, avgdl and doc lengths stay the
 * unmasked call's -- it only removes docs from the ranking.  where_bits: u32 words, one row of SA_WHERE_WORDS(where_n)
 * words covering where_n docs (the index's docs, or a view's positions under sa_score_batch_topk_sim), for the whole
 * batch (where_stride == 0) or one row per query (where_stride == that row length; row q is query q's).  Within a row
 * the bits are in the tile kernels' owner order, not doc order: word t * 256 + i holds, at bit 4 j + e, doc
 * t * 8192 + 4 (i + 256 j) + e (t: the 8,192-doc tile, i: the owning thread, j < 8, e < 4); bits past where_n are 0.
 * where_n must equal the doc (position) count the call ranks; anything else is SA_ERR_ARG before any device work.
 * where_bits NULL: no mask (where_n and where_stride are then ignored). */
#define SA_WHERE_WORDS(n) ((((uint64_t)(n) + 8191u) / 8192u) * 256u)
/* Batched boolean queries, one entry point for every form; the nullable per-clause arrays select it.  Each layer below
 * adds to the one before, and a batch that does not use a layer's arrays scores as the layer before, bit for bit.
 *
 * Or / And (clause_weight, clause_occur, clause_group, clause_tie and clause_node NULL; n_nodes == n_queries): OR /
 * AND / min-should-match over term and phrase clauses (the reference's composition in test/test_search.py:126-226).
 * Query q = clauses [node_clause_starts[q], node_clause_starts[q+1]) (1 to SA_BOOL_MAX_CLAUSES of them;
 * node_clause_starts[0] == 0); clause c = clause_terms[clause_term_starts[c] .. clause_term_starts[c+1]) (1 term, or a
 * phrase with `slop`), scored exactly as sa_score_term / sa_score_phrase with idf clause_idf[c].  Per query,
 * s = score(c0) + score(c1) + ... folded left in float32; a doc ranks iff s > 0 and at least mm[q] (<= its clauses)
 * clauses score > 0 there.  Result: the top k by (score desc, doc id asc; as np.argpartition,
 * searcharray/utils/sort.py:24), GLOBAL doc ids (doc_base added), empty slots SA_NO_DOC / 0.  Phrase clauses need
 * ordinary BM25 parameters (k1 > 0, 0 <= b < 1).  *n_redone (nullable): queries re-run exactly because a tile had more
 * candidates than slots.
 *
 * Roles and weights (clause_weight and clause_occur given, both or neither): Lucene's MUST / SHOULD / FILTER /
 * MUST_NOT, per clause clause_weight[c] (finite, >= 0) and clause_occur[c] (one of SA_OCCUR_*).  Per query, over its
 * MUST and SHOULD clauses in clause order, s = w0 * score(c0), then s = s + w1 * score(c1), ..., every product and sum
 * rounded to float32 (no fused multiply-add).  A doc ranks iff s > 0, at least mm[q] (<= its SHOULD clauses) SHOULD
 * clauses score > 0 there (unweighted: a weight of 0 still matches), every MUST and FILTER clause scores > 0 there,
 * and no MUST_NOT clause does.  FILTER and MUST_NOT clauses add nothing to s.  Every clause, whatever its role, is
 * scored as above, with its own idf.  With every clause SHOULD and weight 1 the result equals Or / And's, bit for bit.
 *
 * Disjunction-max groups (clause_group and clause_tie given, both or neither, and only with clause_occur): Lucene's
 * DisjunctionMaxQuery, edismax's per-term qf.  clause_group[c] is the batch-wide index of the first clause of c's
 * group (c itself for a plain clause), and clause_tie[c] is read at a group's first clause (finite, in [0, 1]; checked
 * at every group's first clause).  A group is a run of consecutive clauses of one query with one occur, and is one
 * clause of its query: with v_j = w_j * score(c_j) over its members, m = max_j v_j, t = v_0 + v_1 + ... (left fold),
 * it contributes d = m + (t - m) * tie (every step rounded to float32, no fused multiply-add) with weight 1 to s under
 * its occur, and it matches a doc where any member scores > 0 (unweighted).  mm[q] counts SHOULD groups (<= their
 * number).  Members of a group of two or more clauses need ordinary BM25 parameters (k1 > 0, 0 <= b < 1, finite
 * idf >= 0), so that every v >= +0; a group of one is a plain clause.
 *
 * Nested queries (clause_node given, only with the group arrays): an Or / And / Bool used as a clause of another.
 * Nodes 0 .. n_queries-1 are the queries whose top k is returned; nodes n_queries .. n_nodes-1 are nested queries.
 * Node n owns clauses [node_clause_starts[n], node_clause_starts[n+1]), with the per-clause arrays, groups and mm[n]
 * above, checked per node.  clause_node[c] == SA_NO_NODE: a leaf, its terms clause_terms[clause_term_starts[c] ..).
 * Otherwise c is nested node clause_node[c]: it has no terms, the node's index is above that of the node holding c,
 * no other clause references it, and c is not a DisMax member; every nested node is referenced.  A nested node N
 * scores r_N(d) = the score N ranks doc d with as a query of its own (s_N(d) where all its conditions hold and
 * s_N(d) > 0, +0 elsewhere), and matches where r_N(d) > 0: it adds w * r_N under MUST / SHOULD (rounded, then added),
 * counts once towards its holder's mm, and under FILTER / MUST_NOT plays a leaf's role.  Without clause_node,
 * n_nodes == n_queries.
 *
 * Document mask (where_bits, where_n, where_stride; SA_WHERE_WORDS): over the index's n_docs docs.  Per query the
 * result is the top k of the unmasked call's scores where the query's mask is set; every score equals the unmasked
 * one bit for bit.
 *
 * Feature clauses (Lucene's FeatureField, Elasticsearch's rank_feature): a one-term leaf whose term id is
 * SA_FEATURE_TERM(fn, slot) scores the index's feature column `slot` (sa_index_set_feature; on the clause's field in
 * the multi-field call) through function fn, with its parameter in clause_idf[c].  With x the doc's value, v = +0
 * where x is 0, and otherwise:
 *   SA_FEATURE_LINEAR      v = x                                             (clause_idf[c] must be 0)
 *   SA_FEATURE_SATURATION  v = x / (x + pivot), each step rounded to float32  (pivot = clause_idf[c], finite, > 0)
 *   SA_FEATURE_LOG         v = float32(log(double(s) + double(x)))             (s = clause_idf[c], finite, >= 1)
 * The clause matches where v > 0 and is otherwise a leaf like a term: counted once towards mm, w * v added under MUST
 * / SHOULD, a leaf's role under FILTER / MUST_NOT.  It is not a DisMax member of a group of two or more.  An Or / And
 * batch holding one runs as the roles layer with every clause SHOULD and weight 1 (the same result).  A reserved id
 * naming an unknown function or a slot not set on the index, a reserved id inside a phrase, and a parameter out of
 * range are SA_ERR_ARG before any device work.  Only the boolean entry points read reserved ids; every other entry
 * point takes them as the out-of-range term ids they are.
 *
 * Range and In clauses (Elasticsearch's range and terms filters, Lucene's point range and TermInSetQuery): leaves
 * scored as a constant, v = 1.0f where the clause matches and +0 elsewhere, otherwise as a feature clause (counted
 * once towards mm, w * v added under MUST / SHOULD, a leaf's role under FILTER / MUST_NOT, not a DisMax member of a
 * group of two or more); clause_idf[c] must be 0.  A range clause has exactly three entries: SA_RANGE_TERM(slot),
 * then the float32 bit patterns of lo and hi; it matches where the value x of feature column `slot` has x > 0 and
 * lo <= x <= hi (NaN bits are refused; -inf / +inf leave a side open).  An In clause is SA_IN_TERM(slot) followed by
 * one or more codes of facet column `slot` (sa_index_set_facet), each below the facet's n_buckets, duplicates
 * allowed; it matches where the doc's code is one of them (a doc without a value never does).  A range whose
 * column's tile bounds miss [lo, hi], or an In whose codes are not in the tile, is absent from the tile, and under
 * MUST / FILTER the tile is published empty before any list is read (sa_stats.filter_tiles).  A wrong entry count,
 * NaN bits, a code out of range, a slot not set and a non-zero parameter are SA_ERR_ARG before any device work.
 *
 * Hit and facet counts (n_facets, facet_field, facet_slot, out_total and out_facet_counts, the last arguments; out_total
 * non-NULL): Lucene's totalHits and Elasticsearch's terms aggregations, counted where the fold decides which docs
 * rank.  out_total[q] is the number of docs query q ranks (the docs whose score the top k is taken from: s > 0 and
 * every condition above, mask included), over all of them, not only the top k.  With
 * n_facets (<= SA_BOOL_MAX_FACETS) facets, facet i is the facet column facet_slot[i] (sa_index_set_facet) of the index
 * of field facet_field[i] (0 on the single-index entry point; a field slot of the multi on the multi-field one), with
 * B_i buckets, and out_facet_counts[q * (B_0 + ... + B_{n-1}) + B_0 + ... + B_{i-1} + b] is the number of docs query q
 * ranks whose code in facet i is b (docs without a value are in no bucket).  The counts cover the index's own docs
 * (a shard's, on a shard).  A slot not set, more than SA_BOOL_MAX_FACETS facets, a field out of range or
 * out_facet_counts NULL with n_facets > 0 is SA_ERR_ARG before any device work.  The ranking is the same as without
 * counting, bit for bit; an Or / And batch then runs as the roles layer with every clause SHOULD and weight 1.
 * out_total NULL: no counting (n_facets, facet_field, facet_slot and out_facet_counts are ignored).
 *
 * Arrays given in a pairing other than those above (weights without occurs, groups without ties or without occurs,
 * clause_node without groups, n_nodes != n_queries without clause_node) are SA_ERR_ARG before any device work. */
#define SA_BOOL_MAX_CLAUSES 64
#define SA_BOOL_MAX_FACETS 4
#define SA_OCCUR_SHOULD 0
#define SA_OCCUR_MUST 1
#define SA_OCCUR_FILTER 2
#define SA_OCCUR_MUST_NOT 3
#define SA_NO_NODE 0xFFFFFFFFu
/* Per-document feature columns of an index (popularity, votes, a quality score), read by the feature and range
 * clauses above.  sa_index_set_feature copies values[0 .. n_values) (n_values == the index's n_docs; each finite and
 * >= 0, 0 meaning the doc lacks the feature) into slot `slot` (< SA_MAX_FEATURES), replacing what the slot held, and
 * records per 8,192-doc tile whether any value is > 0 and the min and max of those values.  The index owns the copy and frees it with itself.  A bad argument, or an
 * index whose n_terms reaches SA_FEATURE_TERM_BASE, is SA_ERR_ARG and leaves the index as it was. */
#define SA_MAX_FEATURES 16
#define SA_FEATURE_TERM_BASE 0xFF000000u
#define SA_FEATURE_LINEAR 0
#define SA_FEATURE_SATURATION 1
#define SA_FEATURE_LOG 2
#define SA_FEATURE_TERM(fn, slot) (SA_FEATURE_TERM_BASE | ((uint32_t)(fn) << 8) | (uint32_t)(slot))
#define SA_FEATURE_RANGE 0x10
#define SA_FEATURE_IN 0x11
#define SA_RANGE_TERM(slot) SA_FEATURE_TERM(SA_FEATURE_RANGE, slot)   /* a feature slot */
#define SA_IN_TERM(slot) SA_FEATURE_TERM(SA_FEATURE_IN, slot)         /* a facet slot */
int sa_index_set_feature(sa_index *index, uint32_t slot, const float *values, uint64_t n_values);
/* Per-document facet columns of an index (a language, a decade, a category), counted by the facet counts above.
 * sa_index_set_facet copies codes[0 .. n_values) (n_values == the index's n_docs) into slot `slot`
 * (< SA_MAX_FACETS), replacing what the slot held: a code in [0, n_buckets) is the doc's bucket, -1 means the doc has
 * no value.  1 <= n_buckets <= SA_FACET_MAX_BUCKETS.  The index owns the copy (uint16 per doc) and, per 8,192-doc
 * tile, a 1,024-bit set of the codes present (read by In clauses), and frees them with itself.  A bad argument is SA_ERR_ARG and leaves the index as it was. */
#define SA_MAX_FACETS 8
#define SA_FACET_MAX_BUCKETS 1024
int sa_index_set_facet(sa_index *index, uint32_t slot, const int32_t *codes, uint64_t n_values, uint32_t n_buckets);
int sa_score_batch_topk_bool(sa_index *index, uint32_t n_nodes, const uint32_t *node_clause_starts,
                             const uint32_t *clause_node, const uint32_t *clause_terms,
                             const uint32_t *clause_term_starts, const float *clause_idf, const float *clause_weight,
                             const uint8_t *clause_occur, const uint32_t *clause_group, const float *clause_tie,
                             const uint32_t *mm, uint32_t n_queries, uint32_t slop, float avg_doc_len, float k1,
                             float b, uint32_t k, const uint32_t *where_bits, uint64_t where_n, uint64_t where_stride,
                             uint32_t *out_docs, float *out_scores, uint32_t *n_redone, uint32_t n_facets,
                             const uint32_t *facet_field, const uint32_t *facet_slot, uint32_t *out_total,
                             uint32_t *out_facet_counts);
/* Per-document group columns of an index (a franchise, a parent SKU, a site), read by the collapsed top-k below.
 * sa_index_set_group copies codes[0 .. n_values) (n_values == the index's n_docs) into slot `slot` (< SA_MAX_GROUPS),
 * replacing what the slot held: a code in [0, 2^31 - 1) is the doc's group, -1 means the doc belongs to no group.  The
 * index owns the copy (uint32 per doc, SA_GROUP_NONE for -1 and past n_docs) and frees it with itself.  A bad
 * argument is SA_ERR_ARG and leaves the index as it was. */
#define SA_MAX_GROUPS 4
#define SA_GROUP_NONE 0xFFFFFFFFu
int sa_index_set_group(sa_index *index, uint32_t slot, const int32_t *codes, uint64_t n_values);
/* Collapsed top-k (Elasticsearch's collapse, Solr's collapsing query parser with nullPolicy=expand): one result per
 * group of group column `group_slot` (sa_index_set_group).  The arguments after group_slot are
 * sa_score_batch_topk_bool's, in its order and under its refusals.  Per query let S_q be the dense vector
 * sa_score_batch_topk_bool ranks from (mask applied).  The ranked docs are those with S_q > 0; a group's leader is its
 * ranked doc with the highest S_q, ties to the lower doc id; a ranked doc whose code is SA_GROUP_NONE is a group of its
 * own.  Result: the k best leaders by (score desc, doc id asc), with the ids and float32 scores the call without
 * collapsing returns for those docs, empty slots SA_NO_DOC / 0.  So a column of distinct codes, or one of SA_GROUP_NONE
 * only, returns sa_score_batch_topk_bool's result bit for bit, and the first k' results at k are the result at k'.
 * The hit and facet counts count documents, not groups: they equal sa_score_batch_topk_bool's.  Each (query, tile)
 * keeps its exact k best leaders (a group's global leader is among the k best leaders of its tile whenever the group
 * is in the global top k), so nothing overflows and *n_redone is always 0.  On a shard the groups are collapsed over
 * the shard's own docs.  A slot not set is SA_ERR_ARG before any device work. */
int sa_score_batch_topk_bool_collapse(sa_index *index, uint32_t group_slot, uint32_t n_nodes,
                                      const uint32_t *node_clause_starts, const uint32_t *clause_node,
                                      const uint32_t *clause_terms, const uint32_t *clause_term_starts,
                                      const float *clause_idf, const float *clause_weight, const uint8_t *clause_occur,
                                      const uint32_t *clause_group, const float *clause_tie, const uint32_t *mm,
                                      uint32_t n_queries, uint32_t slop, float avg_doc_len, float k1, float b,
                                      uint32_t k, const uint32_t *where_bits, uint64_t where_n, uint64_t where_stride,
                                      uint32_t *out_docs, float *out_scores, uint32_t *n_redone, uint32_t n_facets,
                                      const uint32_t *facet_field, const uint32_t *facet_slot, uint32_t *out_total,
                                      uint32_t *out_facet_counts);
/* Scoring at given documents, the second stage after a batched top-k (reranker features, window rescoring): replaces
 * the reference's `arr.score(q)[docs[q]]` (postings.py:652 `score`, indexed at the candidates) without a dense row.
 * The descriptor arguments are sa_score_batch_topk_bool's, in its order and under its refusals; in place of k, the
 * mask, the top-k outputs and the counts it takes docs[n_queries * n_per_query] and fills
 * out_scores[n_queries * n_per_query]: out_scores[q * K + j] (K = n_per_query) is the value at doc docs[q * K + j] of
 * the dense vector S_q the top-k entry point ranks from -- the fold's float32 s where the doc ranks (s > 0, mm met,
 * every MUST / FILTER clause matching and no MUST_NOT clause, for top-level and nested nodes alike) and +0.0
 * elsewhere.  Ids are global (doc_base added), as the top-k returns them; SA_NO_DOC gives 0.0; duplicates and any
 * order are allowed.  Called on the docs of a top-k call with the same descriptors it returns that call's scores bit
 * for bit.  Any other id outside [doc_base, doc_base + n_docs), n_queries * n_per_query >= 2^31, and a query with
 * more than 64 nested nodes are SA_ERR_ARG before any device work.  Term, feature, DisMax and nested clauses are
 * evaluated at each doc from the index's lists (one thread per (query, doc)); only phrase clauses write their count
 * rows, as in the top-k. */
int sa_score_docs_bool(sa_index *index, uint32_t n_nodes, const uint32_t *node_clause_starts,
                       const uint32_t *clause_node, const uint32_t *clause_terms, const uint32_t *clause_term_starts,
                       const float *clause_idf, const float *clause_weight, const uint8_t *clause_occur,
                       const uint32_t *clause_group, const float *clause_tie, const uint32_t *mm,
                       uint32_t n_queries, uint32_t slop, float avg_doc_len, float k1, float b,
                       const uint32_t *docs, uint32_t n_per_query, float *out_scores);

/* The same batch in three stages, so a serving loop (or the benchmark) can keep the query
 * descriptors resident and time the device work alone: upload (H2D of descriptors), execute
 * (enqueue kernels only, asynchronous), download (sync, overflow repair, D2H of the top-k;
 * *n_overflow = queries whose candidate list overflowed and were re-run exactly). */
int sa_batch_upload(sa_index *index, const uint32_t *terms, const uint32_t *term_starts,
                    const float *idf, uint32_t n_queries, uint32_t slop,
                    float avg_doc_len, float k1, float b, uint32_t k);
int sa_batch_execute(sa_index *index);
int sa_batch_download(sa_index *index, uint32_t *out_docs, float *out_scores, uint32_t *n_overflow);
/* CUDA-event timer on the library's own stream (the stream the kernels are launched on). */
int sa_timer_start(sa_index *index);
int sa_timer_stop(sa_index *index, double *ms_out);

/* Kernel-time accounting for roofline reporting (CUDA events on the library's stream):
 * milliseconds spent in, and launches of, the dominant kernels since the last reset. */
typedef struct {
    double term_kernel_ms;
    uint64_t term_kernel_launches;
    uint64_t term_kernel_queries;     /* queries covered by those launches */
    double topk_kernel_ms;
    uint64_t topk_kernel_launches;
    double phrase_kernel_ms;
    uint64_t phrase_kernel_launches;
    uint64_t total_launches;          /* every kernel launched by the library */
    /* phrase (slop 0) batches, summed over the queries of every sa_batch_download since the reset:
     * continuation words written (sum of C_s) and docs with a non-zero phrase count (M) -- the
     * data-dependent terms of SURVEY 8d's B_phrase = 8*sum(W) + 16*sum(C_s) + 4*N + 4*M */
    uint64_t phrase_cont_words;
    uint64_t phrase_matched_docs;
    /* launches of the conjunction regime's phrase_tile_kernel (also counted in phrase_kernel_launches): 0 = the
     * search regime alone ran, phrase_kernel_launches > phrase_tile_launches after one = a re-run in the search regime */
    uint64_t phrase_tile_launches;
    /* the bool_tile_kernel instances launched (sa_bool.cu, bool_kernel): bit variant * 10 + form * 2 + masked, with
     * form 0 Or / And, 1 roles and weights, 2 fields, 3 DisMax, 4 nested and variant 0 plain, 1 FEATURE, 2 COUNT,
     * 3 COLLAPSE */
    uint64_t bool_instances;
    /* the sim_tile_kernel / sim_where_tile_kernel instances launched (sa_view.cu, launch_sim_tiles): bit
     * 2 * kind + masked, kind the SA_SIM_* value (0 impact, 1 legacy, 2 classic, 3 BM25, also the BM25 batch's phrase
     * and span re-runs) and masked 1 for sim_where_tile_kernel */
    uint64_t sim_instances;
    /* query groups the term launches walked (sa_term.cu): ceil(queries / G) per launch of group width G, so one per
     * launch that walks every query as one group */
    uint64_t term_kernel_groups;
    /* (query, tile) pairs whose candidates the deep collector took (k > 32: the tile's exact top k, sorted), over
     * every batched top-k entry point */
    uint64_t deep_tiles;
    /* (node, tile) pairs of the boolean entry points' first passes published empty because a MUST / FILTER range or
     * In clause was absent from the tile (its column's tile bounds or code set miss the clause) */
    uint64_t filter_tiles;
    /* (query, tile) pairs whose leaders the collapse collector took (sa_score_batch_topk_bool_collapse and its
     * multi-field twin) */
    uint64_t collapse_tiles;
    /* windows the collapse walk took past the first, in the tiles and in the per-query select: a tile or a query
     * whose best ranked docs crowd into few groups walks its docs in several windows */
    uint64_t collapse_windows;
} sa_stats;
int sa_stats_reset(sa_index *index);
int sa_stats_get(sa_index *index, sa_stats *out);
int sa_set_profiling(sa_index *index, int enabled);   /* per-kernel CUDA events on/off */

/* -------------------------------------------------------------- multi-GPU (8e)
 * One process per GPU, each owning a contiguous doc-id range.  The only exchange on the
 * scoring path is one all-gather of per-shard top-k per query batch.
 * sa_comm_unique_id fills a 128-byte NCCL unique id on rank 0 (the caller broadcasts it
 * with whatever bootstrap it has); sa_comm_init joins the clique. */
int sa_comm_unique_id(void *id128_out);
int sa_comm_init(sa_index *index, const void *id128, int rank, int world_size);
int sa_comm_destroy(sa_index *index);
/* Harness plumbing over the same communicator: barrier, and max-over-ranks of a double
 * (bench.py uses these for the barrier + max-over-ranks timing rule). */
int sa_comm_barrier(sa_index *index);
int sa_comm_allreduce_max(sa_index *index, double *inout);
int sa_comm_allreduce_sum_u64(sa_index *index, uint64_t *inout, uint64_t n);
int sa_batch_execute_allgather(sa_index *index);
int sa_batch_download_allgather(sa_index *index, uint32_t *out_docs, float *out_scores,
                                uint32_t *n_overflow);
/* Like sa_score_batch_topk on every rank's shard, then ncclAllGather of the per-shard
 * (doc, score) lists and a k-way merge on the device; every rank receives the global top-k. */
int sa_score_batch_topk_allgather(sa_index *index, const uint32_t *terms, const uint32_t *term_starts,
                                  const float *idf, uint32_t n_queries, uint32_t slop,
                                  float avg_doc_len, float k1, float b, uint32_t k,
                                  uint32_t *out_docs, float *out_scores);
/* The merge step of sa_score_batch_topk_allgather on lists the caller holds: lists[r][q][i], world per-rank lists of
 * k keys (score_bits << 32 | ~doc, as the batched top-k keeps them) per query, each sorted descending and 0-padded,
 * the ranks' doc ranges disjoint; out[q][i] = the k largest keys of query q over the ranks, descending, 0-padded.
 * Runs the device merge the all-gather uses (topk_merge_kernel, or topk_merge_ranked_kernel for world * k > 4,096)
 * on the index's device; 1 <= k <= SA_TOPK_DEEP_MAX. */
int sa_topk_merge(sa_index *index, const uint64_t *lists, uint32_t world, uint32_t n_queries, uint32_t k,
                  uint64_t *out);

/* ------------------------------------------------------ multi-field edismax (8f-1)
 * Replaces the numpy half of searcharray/solr.py:117-355 (edismax): the per-(term, field) BM25
 * vectors, the phrase-phase vectors and the combined score vector stay in HBM.  The host mirror
 * (searcharray_b200/solr.py) parses the query like solr.py:77-114, computes idf like
 * similarity.py:19-21 and drives these calls.  All fields index the same documents.
 *   sa_multi_qf       solr.py:117-178.  field f has n_terms[f] query terms; term_ids / idf are the
 *                     per-field lists concatenated.  has_boost[f] == 0 <=> "field" without ^boost.
 *                     mm[f]: clauses that must score > 0 (term-centric: mm[0] over term positions;
 *                     field-centric: per field, already clamped to its term count).  The combined
 *                     vector is float64 (term-centric) or float32 (field-centric), as in numpy.
 *   sa_multi_filter   solr.py:326-330: restrict field `field`'s posting lists of `term_ids` to the docs
 *                     with qf > 0 (FilteredPosns, middle_out.py:291-317); df_out = doc frequencies of
 *                     the filtered lists (what SearchArray.docfreq reports on the sliced array).
 *   sa_multi_phrases  phrase i = filtered lists term_slots[phrase_starts[i] .. phrase_starts[i+1])
 *                     (slots index the last sa_multi_filter's term list; term_ids: the same terms' ids);
 *                     BM25 with idf[i].  Row i of the field holds the result (solr.py:181-244).
 *   sa_multi_add_phase  float32 sum, in order, of rows (entry_field[i], entry_row[i]) * entry_boost[i],
 *                     added to the combined vector where it is non-zero (solr.py:335-353).
 *   sa_multi_download / sa_multi_topk   the dense vector (float64, or float32 when as_float32), or its
 *                     exact top-k (score desc, doc asc; absolute doc ids; empty slots SA_NO_DOC / 0). */
typedef struct sa_multi sa_multi;
int sa_multi_create(sa_index *const *fields, uint32_t n_fields, sa_multi **multi_out);
int sa_multi_destroy(sa_multi *multi);
int sa_multi_qf(sa_multi *multi, int field_centric, const uint32_t *n_terms, const uint32_t *term_ids,
                const float *idf, const float *boost, const uint32_t *has_boost,
                const float *avg_doc_len, const float *k1, const float *b, const uint32_t *mm,
                double tie, uint64_t *n_matches);
int sa_multi_filter(sa_multi *multi, uint32_t field, const uint32_t *term_ids, uint32_t n_terms,
                    uint64_t *df_out);
int sa_multi_phrases(sa_multi *multi, uint32_t field, uint32_t n_phrases, const uint32_t *phrase_starts,
                     const uint32_t *term_slots, const uint32_t *term_ids, const float *idf,
                     float avg_doc_len, float k1, float b);
int sa_multi_add_phase(sa_multi *multi, uint32_t n_entries, const uint32_t *entry_field,
                       const uint32_t *entry_row, const float *entry_boost, const uint32_t *entry_has_boost);
int sa_multi_download(sa_multi *multi, void *out, int as_float32);
int sa_multi_is_float32(sa_multi *multi, int *out);
int sa_multi_topk(sa_multi *multi, uint32_t k, uint32_t *out_docs, double *out_scores);
/* Boolean queries over several fields of one document set (Elasticsearch's `+title:star overview:war`): the arguments
 * and layers of sa_score_batch_topk_bool, with clause c on field clause_field[c] (< the multi's fields; read for leaves
 * only) and its term ids that field's.  clause_weight and clause_occur are required (Or / And take every clause
 * SHOULD with weight 1); clause_group / clause_tie and clause_node are optional as there, and the mask is over the
 * fields' n_docs docs.  Field f of the multi is scored with avg_doc_len[f], k1[f] and b[f]; each clause's idf is the
 * caller's, from its own field.  Per query the result is sa_score_batch_topk_bool's composition with
 * score(c) = .score of the clause on its field; a field whose avg_doc_len is 0 scores 0 at every doc (a MUST / FILTER
 * clause on it ranks nothing, a MUST_NOT clause on it vetoes nothing).  A DisMax group's members may sit on different
 * fields, each scored on its own: Elasticsearch's best_fields, and per-term groups inside an Or with mm for edismax's
 * term-centric qf.  Fields that share one sa_index must share (avg_doc_len, k1, b): the index caches one norm table.
 * The hit and facet counts are sa_score_batch_topk_bool's, facet_field[i] being a field slot of the multi.
 * Result ids are global doc ids (doc_base added). */
int sa_multi_score_batch_topk_bool(sa_multi *multi, uint32_t n_nodes, const uint32_t *node_clause_starts,
                                   const uint32_t *clause_node, const uint32_t *clause_field,
                                   const uint32_t *clause_terms, const uint32_t *clause_term_starts,
                                   const float *clause_idf, const float *clause_weight, const uint8_t *clause_occur,
                                   const uint32_t *clause_group, const float *clause_tie, const uint32_t *mm,
                                   uint32_t n_queries, uint32_t slop, const float *avg_doc_len, const float *k1,
                                   const float *b, uint32_t k, const uint32_t *where_bits, uint64_t where_n,
                                   uint64_t where_stride, uint32_t *out_docs, float *out_scores, uint32_t *n_redone,
                                   uint32_t n_facets, const uint32_t *facet_field, const uint32_t *facet_slot,
                                   uint32_t *out_total, uint32_t *out_facet_counts);
/* sa_score_batch_topk_bool_collapse over the fields of a multi: group column group_slot of field group_field's index
 * (a field slot of the multi), then sa_multi_score_batch_topk_bool's arguments in its order.  A field out of range or a
 * slot not set on its index is SA_ERR_ARG before any device work. */
int sa_multi_score_batch_topk_bool_collapse(sa_multi *multi, uint32_t group_field, uint32_t group_slot,
                                            uint32_t n_nodes, const uint32_t *node_clause_starts,
                                            const uint32_t *clause_node, const uint32_t *clause_field,
                                            const uint32_t *clause_terms, const uint32_t *clause_term_starts,
                                            const float *clause_idf, const float *clause_weight,
                                            const uint8_t *clause_occur, const uint32_t *clause_group,
                                            const float *clause_tie, const uint32_t *mm, uint32_t n_queries,
                                            uint32_t slop, const float *avg_doc_len, const float *k1, const float *b,
                                            uint32_t k, const uint32_t *where_bits, uint64_t where_n,
                                            uint64_t where_stride, uint32_t *out_docs, float *out_scores,
                                            uint32_t *n_redone, uint32_t n_facets, const uint32_t *facet_field,
                                            const uint32_t *facet_slot, uint32_t *out_total,
                                            uint32_t *out_facet_counts);
/* sa_score_docs_bool over the fields of a multi: sa_multi_score_batch_topk_bool's descriptor arguments up to b, then
 * the docs (global ids of the fields' document set), n_per_query and out_scores, under sa_score_docs_bool's contract
 * with sa_multi_score_batch_topk_bool as the top-k it matches. */
int sa_multi_score_docs_bool(sa_multi *multi, uint32_t n_nodes, const uint32_t *node_clause_starts,
                             const uint32_t *clause_node, const uint32_t *clause_field, const uint32_t *clause_terms,
                             const uint32_t *clause_term_starts, const float *clause_idf, const float *clause_weight,
                             const uint8_t *clause_occur, const uint32_t *clause_group, const float *clause_tie,
                             const uint32_t *mm, uint32_t n_queries, uint32_t slop, const float *avg_doc_len,
                             const float *k1, const float *b, const uint32_t *docs, uint32_t n_per_query,
                             float *out_scores);

/* ------------------------------------------------- per-op exports (parity tests)
 * Device implementations of the reference's native ops on raw arrays (host in, host out),
 * for kernel-level parity tests against the Cython originals (SURVEY.md section 8b). */
/* popcount64_reduce (roaringish/popcount.pyx:212-237): returns groups in *n_out; exact sums rounded once to float32,
 * docs whose words carry no bits kept with count 0 */
int sa_op_popcount64_reduce(const uint64_t *words, uint64_t n, int device,
                            uint64_t *keys_out, float *counts_out, uint64_t *n_out);
/* bm25_score (bm25/bm25.pyx:28-41): in place over all n */
int sa_op_bm25_score(float *tf_inout, const float *doc_lens, uint64_t n, float avg_doc_len,
                     float idf, float k1, float b, int device);
/* The reference's other similarities (searcharray/similarity.py:41-89) evaluated on the device:
 * SA_SIM_BM25_IMPACT -> float32[n] `tf / (tf + k1 * (1 - b + b * dl / avgdl))` (bm25_impact, :41-54; idf unused);
 * SA_SIM_BM25_LEGACY -> float64[n] `idf * (tf * (k1 + 1)) / (...)` (bm25_legacy_similarity, :57-72);
 * SA_SIM_CLASSIC     -> float64[n] `idf * sqrt(tf) * (1 / sqrt(dl))` (classic_similarity, :75-89; k1, b, avgdl unused).
 * idf is the float64 scalar the caller computed the way the reference does; numpy's dtype promotion is reproduced. */
#define SA_SIM_BM25_IMPACT 0
#define SA_SIM_BM25_LEGACY 1
#define SA_SIM_CLASSIC 2
/* BM25 on a view, for sa_score_batch_topk_sim only (sa_op_similarity rejects it) */
#define SA_SIM_BM25 3
int sa_op_similarity(int kind, const float *term_freqs, const float *doc_lens, uint64_t n,
                     double avg_doc_len, double idf, double k1, double b, int device, void *out);
/* bigram_freqs (phrase/bigram_freqs.py:213-307): cont_rhs=1 -> Continuation.RHS else LHS.
 * ids/counts: per-doc matches (zero-count docs kept, quirk iv); next: continuation words.
 * Capacities: ids/counts >= min(n_lhs,n_rhs)*2, next >= 2*min(n_lhs, n_rhs)+2. */
int sa_op_bigram_freqs(const uint64_t *lhs, uint64_t n_lhs, const uint64_t *rhs, uint64_t n_rhs,
                       int cont_rhs, int device,
                       uint64_t *ids_out, float *counts_out, uint64_t *n_ids_out,
                       uint64_t *next_out, uint64_t *n_next_out);

/* The reference's sorted-set ops on raw arrays (sa_setops.cu), one export per Cython op, returning what the
 * op returns (index arrays, not values, for the intersect family).  Inputs sorted by (x & mask) as every
 * reference caller passes them; output capacities: intersect family min(n_lhs, n_rhs) per array (keep mode:
 * n_lhs / n_rhs), merge n_lhs + n_rhs, the grouped ops and unique / payload_slice n.
 *   sa_op_intersect                searcharray/roaringish/intersect.pyx:278-320 (drop_duplicates as there;
 *                                  mask == 0 -> SA_ERR_ARG, the reference raises ValueError)
 *   sa_op_adjacent                 :323-343   pairs with (lhs & mask) + lowbit(mask) == (rhs & mask)
 *   sa_op_intersect_with_adjacents :346-390   both in one call
 *   sa_op_merge                    searcharray/roaringish/merge.pyx:137-158
 *   sa_op_sort_merge_counts        merge.pyx:211-232
 *   sa_op_unique                   searcharray/roaringish/unique.pyx:139-145
 *   sa_op_popcount64 / sa_op_popcount_reduce_at / sa_op_key_sum_over   popcount.pyx:120-122, 150-165, 195-204
 *   sa_op_payload_slice / sa_op_as_dense   roaringish_ops.pyx:46-68, 84-98
 * Inside a run of equal values, merge / sort_merge_counts pair the k-th lhs copy with the k-th rhs copy, as the
 * reference's two-pointer loop does (drop_duplicates drops the paired rhs copies; counts add over pairs).
 * sa_op_last_staged_ctas: how many CTAs of the calling thread's last intersect-family call took the
 * TMA-staged shared-memory path: a test hook.
 * sa_op_last_path_ctas: the same call's CTAs by path, out[0] staged, out[1] searched global memory, out[2] had an
 * empty rhs range (no partner possible); summed over the partner passes of the call (keep mode and
 * intersect_with_adjacents run two). */
int sa_op_intersect(const uint64_t *lhs, uint64_t n_lhs, const uint64_t *rhs, uint64_t n_rhs,
                    uint64_t mask, int drop_duplicates, int device,
                    uint64_t *lhs_idx_out, uint64_t *rhs_idx_out, uint64_t *n_lhs_out, uint64_t *n_rhs_out);
int sa_op_adjacent(const uint64_t *lhs, uint64_t n_lhs, const uint64_t *rhs, uint64_t n_rhs,
                   uint64_t mask, int device, uint64_t *lhs_idx_out, uint64_t *rhs_idx_out, uint64_t *n_out);
int sa_op_intersect_with_adjacents(const uint64_t *lhs, uint64_t n_lhs, const uint64_t *rhs, uint64_t n_rhs,
                                   uint64_t mask, int device,
                                   uint64_t *lhs_idx_out, uint64_t *rhs_idx_out, uint64_t *n_out,
                                   uint64_t *adj_lhs_idx_out, uint64_t *adj_rhs_idx_out, uint64_t *n_adj_out);
int sa_op_merge(const uint64_t *lhs, uint64_t n_lhs, const uint64_t *rhs, uint64_t n_rhs,
                int drop_duplicates, int device, uint64_t *out, uint64_t *n_out);
int sa_op_sort_merge_counts(const uint64_t *lhs_ids, const float *lhs_counts, uint64_t n_lhs,
                            const uint64_t *rhs_ids, const float *rhs_counts, uint64_t n_rhs,
                            int device, uint64_t *ids_out, float *counts_out, uint64_t *n_out);
int sa_op_unique(const uint64_t *arr, uint64_t n, uint64_t rshift, int device, uint64_t *out, uint64_t *n_out);
int sa_op_popcount64(const uint64_t *arr, uint64_t n, int device, uint64_t *out);
int sa_op_popcount_reduce_at(const uint64_t *ids, const uint64_t *payload, uint64_t n, int device,
                             uint64_t *ids_out, float *counts_out, uint64_t *n_out);
int sa_op_key_sum_over(const uint64_t *ids, const uint64_t *counts, uint64_t n, int device,
                       uint64_t *ids_out, float *counts_out, uint64_t *n_out);
int sa_op_payload_slice(const uint64_t *arr, uint64_t n, uint64_t msb_mask, uint64_t min_payload,
                        uint64_t max_payload, int device, uint64_t *out, uint64_t *n_out);
int sa_op_as_dense(const uint64_t *indices, const float *values, uint64_t n, uint64_t size, int device, float *out);
uint64_t sa_op_last_staged_ctas(void);
void sa_op_last_path_ctas(uint64_t out[3]);

/* ------------------------------------------------------------ index build (8f-4)
 * The numpy half of the reference's index build after tokenisation (searcharray/indexing.py:101-145:
 * stable sort of the (term, doc, posn) triples by term; searcharray/roaringish/roaringish.py:93-142: encode) on
 * the device.  Triples in document order as _gather_tokens emits them (indexing.py:64-98).
 * words_out: room for n_triples words; term_off_out / term_len_out: every term's slice of words_out (terms without
 * triples: 0, 0).  SA_ERR_ARG before any device work for n_triples >= 2^31, a term id >= n_terms, a doc id >= 2^28
 * or a position > 18 * 2^18 - 1 (the word's 18-bit block). */
int sa_op_build_index(const uint32_t *term_ids, const uint32_t *doc_ids, const uint32_t *posns, uint64_t n_triples,
                      uint32_t n_terms, int device, uint64_t *words_out, uint64_t *n_words_out,
                      uint64_t *term_off_out, uint64_t *term_len_out);

#ifdef __cplusplus
}
#endif
#endif /* SEARCHARRAY_B200_H */
