// sa_phrase.cu -- exact phrase matching (slop == 0) on roaringish posting words.
//
// Replaces (reference paths relative to softwaredoug/searcharray):
//   compute_phrase_freqs + L->R / R->L drivers + _intersect_bigram_matches  phrase/middle_out.py:73-168
//   bigram_freqs, _inner_bigram_freqs, _inner_bigram_same_term, _adj_to_phrase_freq,
//   _adjacent_bigram_freqs, _set_adjbit_at_header                          phrase/bigram_freqs.py:48-307
//   intersect_with_adjacents / intersect / merge / sort_merge_counts /
//   popcount_reduce_at / key_sum_over                                       roaringish/*.pyx
//   PosnBitArray.phrase_freqs dense scatter                                 phrase/middle_out.py:418-446
//
// Design.  Phrase matching never crosses a document, and every term's words are sorted by doc
// id, so the doc-id space is cut into chunks and ONE CTA RUNS THE WHOLE n-TERM PIPELINE FOR ONE
// (query, doc-range chunk): it locates each term's slice for its doc range (warp-cooperative
// 32-ary search), then for every bigram step walks the shorter "driver" list one element per
// thread, binary-searches the other list for the equal header and the adjacent header (the
// reference's galloping intersect has plain set semantics on header-unique lists, SURVEY 8a row
// 10), does the 18-bit shift/AND/popcount, emits the continuation words in order through a block
// scan, and reduces the per-doc counts with a segmented sum.  The running min over steps is a
// search into the previous step's (doc, count) list.  Matches are scattered into the pre-zeroed
// dense vector, optionally through BM25.
//
// The reference's "same term" branch (bigram_freqs.py:139) depends on a GLOBAL property
// (all equal-header pairs identical).  Each launch runs with a speculated flag per step and
// counts (pairs, differing pairs) per step; the host verifies and re-launches on a mis-guess
// (only adversarial inputs ever do).
#include <algorithm>

#include "sa_phrase.cuh"
#include "sa_scan.cuh"
#include "sa_span.cuh"
#include "sa_term.cuh"

#define PT SA_PHRASE_THREADS
#define PW_SUB_DOCS (SA_TILE_DOCS / (SA_PHRASE_THREADS / 32))   // docs of a tile that one warp of the conjunction regime owns (1,024)

struct Elem {
    u64 w0, w1;
    u32 n_emit, cnt, doc;
    bool entry, inner, diff;
};

__device__ __forceinline__ u64 lower_bound_hdr(const u64 *__restrict__ a, u64 n, u64 target) {
    u64 lo = 0, hi = n;
    while (lo < hi) {
        u64 mid = (lo + hi) >> 1;
        if ((a[mid] & SA_HDR_MASK) < target) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// One equal-header pair (bigram_freqs.py:104-155 normal branch, :65-101 same-term branch).
__device__ __forceinline__ void inner_calc(u64 l, u64 r, bool same, bool cont_rhs, u32 &cnt, u64 &word) {
    if (!same) {
        u64 ov = (l & SA_LSB_MASK) & ((r & SA_LSB_MASK) >> 1);
        cnt = (u32)__popcll(ov);
        word = cont_rhs ? (((ov << 1) & SA_LSB_MASK) | (r & SA_HDR_MASK)) : (ov | (l & SA_HDR_MASK));
    } else {
        u64 full = l & (r << 1);
        u32 adj = (u32)__popcll(full & SA_LSB_MASK);
        u32 runs = (u32)__popcll((full & (full << 1)) & SA_LSB_MASK);
        cnt = adj - ((runs + 1) >> 1);                        // _adj_to_phrase_freq: - ceil(runs/2)
        word = cont_rhs ? ((((r << 1) & r) & SA_LSB_MASK) | (l & ~SA_LSB_MASK))
                        : ((l & ~SA_LSB_MASK) | ((l & (l >> 1)) & SA_LSB_MASK));   // `>> 1` leak kept
    }
}

// What driver element i contributes.  D = driver list, O = the other list.
template <bool CONT_RHS, bool DRIVER_LHS>
__device__ __forceinline__ Elem compute_elem(const u64 *__restrict__ D, u64 nD, u64 i,
                                             const u64 *__restrict__ O, u64 nO, bool same) {
    Elem e;
    e.w0 = e.w1 = 0;
    e.n_emit = 0;
    e.cnt = 0;
    e.entry = e.inner = e.diff = false;
    const u64 x = D[i];
    const u64 h = x & SA_HDR_MASK;
    e.doc = (u32)(x >> SA_KEY_SHIFT);
    if (DRIVER_LHS) {
        // x is an lhs word: partners are rhs words at header h (inner) and h + 1 block (adjacent)
        u64 pos = lower_bound_hdr(O, nO, h);
        bool inner = pos < nO && (O[pos] & SA_HDR_MASK) == h;
        u64 r = inner ? O[pos] : 0;
        u64 pos2 = pos + (inner ? 1 : 0);
        bool has_adj = pos2 < nO && (O[pos2] & SA_HDR_MASK) == h + SA_ONE_BLOCK;
        u64 r2 = has_adj ? O[pos2] : 0;
        bool am = has_adj && (x & SA_BIT17) && (r2 & 1ull);
        if (inner) {
            u32 c;
            u64 word;
            inner_calc(x, r, same, CONT_RHS, c, word);
            e.cnt += c;
            if (CONT_RHS) {
                // the rhs word at h may also end a cross-word match that started in lhs[i-1]
                if (i > 0) {
                    u64 lp = D[i - 1];
                    if ((lp & SA_HDR_MASK) + SA_ONE_BLOCK == h && (lp & SA_BIT17) && (r & 1ull)) word |= 1ull;
                }
            } else if (am) {
                word |= SA_BIT17;
            }
            e.w0 = word;
            e.n_emit = 1;
            e.inner = true;
            e.diff = (x != r);
        }
        if (am) {
            e.cnt += 1;
            if (CONT_RHS) {
                // adjacent-only continuation, unless lhs[i+1] pairs with that rhs word itself
                bool next_handles = (i + 1 < nD) && ((D[i + 1] & SA_HDR_MASK) == h + SA_ONE_BLOCK);
                if (!next_handles) {
                    u64 w = (r2 & SA_HDR_MASK) | 1ull;
                    if (e.n_emit == 0) e.w0 = w; else e.w1 = w;
                    e.n_emit++;
                }
            } else if (!inner) {
                e.w0 = h | SA_BIT17;
                e.n_emit = 1;
            }
        }
        e.entry = inner || am;
    } else {
        // x is an rhs word: partners are lhs words at header h - 1 block (adjacent) and h (inner)
        const bool can_adj = h >= SA_ONE_BLOCK;
        u64 pos = lower_bound_hdr(O, nO, can_adj ? h - SA_ONE_BLOCK : h);
        bool has_adj = can_adj && pos < nO && (O[pos] & SA_HDR_MASK) == h - SA_ONE_BLOCK;
        u64 lp = has_adj ? O[pos] : 0;
        u64 posl = pos + (has_adj ? 1 : 0);
        bool inner = posl < nO && (O[posl] & SA_HDR_MASK) == h;
        u64 l = inner ? O[posl] : 0;
        bool am = has_adj && (lp & SA_BIT17) && (x & 1ull);
        if (!CONT_RHS && am) {
            // adjacent-only continuation on the lhs side, unless rhs[i-1] pairs with lp itself
            bool prev_handles = (i > 0) && ((D[i - 1] & SA_HDR_MASK) == h - SA_ONE_BLOCK);
            if (!prev_handles) {
                e.w0 = (lp & SA_HDR_MASK) | SA_BIT17;
                e.n_emit = 1;
            }
        }
        if (inner) {
            u32 c;
            u64 word;
            inner_calc(l, x, same, CONT_RHS, c, word);
            e.cnt += c;
            if (CONT_RHS) {
                if (am) word |= 1ull;
            } else if (i + 1 < nD) {
                u64 rn = D[i + 1];
                if ((rn & SA_HDR_MASK) == h + SA_ONE_BLOCK && (l & SA_BIT17) && (rn & 1ull)) word |= SA_BIT17;
            }
            if (e.n_emit == 0) e.w0 = word; else e.w1 = word;
            e.n_emit++;
            e.inner = true;
            e.diff = (l != x);
            e.doc = (u32)(l >> SA_KEY_SHIFT);
        } else if (am) {
            if (CONT_RHS) {
                e.w0 = h | 1ull;
                e.n_emit = 1;
            }
            e.doc = (u32)(lp >> SA_KEY_SHIFT);
        }
        if (am) e.cnt += 1;
        e.entry = inner || am;
    }
    return e;
}

#include "sa_phrase_warp.cuh"

struct StepShared {
    u32 warp_sums[PT / 32];
    u32 edoc[PT];
    u32 ecnt[PT];
    u32 carry_doc, carry_cnt, carry_valid;
    u32 st_inner, st_diff;
    u64 n_cont, n_docs;
};

// One bigram step over this CTA's chunk.  Writes the continuation list (sorted) to cont_out and
// the per-doc counts (doc << 32 | count, sorted by doc, zero counts kept) to docs_out.
template <bool CONT_RHS, bool DRIVER_LHS>
__device__ void bigram_step(const u64 *__restrict__ D, u64 nD, const u64 *__restrict__ O, u64 nO, bool same,
                            u64 *__restrict__ cont_out, u64 *__restrict__ docs_out, StepShared &S) {
    const unsigned tid = threadIdx.x;
    if (tid == 0) {
        S.n_cont = 0;
        S.n_docs = 0;
        S.carry_valid = 0;
        S.st_inner = 0;
        S.st_diff = 0;
    }
    __syncthreads();
    for (u64 t0 = 0; t0 < nD; t0 += PT) {
        const u64 i = t0 + tid;
        Elem e;
        e.n_emit = 0;
        e.entry = e.inner = e.diff = false;
        e.cnt = 0;
        e.doc = 0;
        e.w0 = e.w1 = 0;
        if (i < nD) e = compute_elem<CONT_RHS, DRIVER_LHS>(D, nD, i, O, nO, same);
        // speculation bookkeeping
        unsigned mi = __ballot_sync(0xffffffffu, e.inner), md = __ballot_sync(0xffffffffu, e.diff);
        if ((tid & 31) == 0 && mi) {
            atomicAdd(&S.st_inner, (u32)__popc(mi));
            if (md) atomicAdd(&S.st_diff, (u32)__popc(md));
        }
        // continuation words, in order
        u32 total;
        u32 off = block_exclusive_sum<PT>(e.n_emit, S.warp_sums, total);
        const u64 cbase = S.n_cont;
        if (e.n_emit >= 1) cont_out[cbase + off] = e.w0;
        if (e.n_emit == 2) cont_out[cbase + off + 1] = e.w1;
        // (doc, count) entries of this tile, compacted into shared memory
        u32 etotal;
        u32 eoff = block_exclusive_sum<PT>(e.entry ? 1u : 0u, S.warp_sums, etotal);
        if (e.entry) {
            S.edoc[eoff] = e.doc;
            S.ecnt[eoff] = e.cnt;
        }
        __syncthreads();
        if (tid == 0) S.n_cont = cbase + total;
        if (etotal) {     // block-uniform
            const bool flush = S.carry_valid && S.edoc[0] != S.carry_doc;
            const bool merge = S.carry_valid && S.edoc[0] == S.carry_doc;
            const u32 c_doc = S.carry_doc, c_cnt = S.carry_cnt;
            const u64 dbase = S.n_docs;
            // segmented sum: the head of each run adds up its run
            bool emit = false, is_last = false;
            u32 sum = 0, doc = 0;
            if (tid < etotal) {
                doc = S.edoc[tid];
                bool head = (tid == 0) || (S.edoc[tid - 1] != doc);
                if (head) {
                    u32 k = tid;
                    while (k < etotal && S.edoc[k] == doc) sum += S.ecnt[k++];
                    if (tid == 0 && merge) sum += c_cnt;
                    is_last = (k == etotal);
                    emit = !is_last;
                }
            }
            u32 htotal;
            u32 hoff = block_exclusive_sum<PT>(emit ? 1u : 0u, S.warp_sums, htotal);
            const u64 obase = dbase + (flush ? 1 : 0);
            if (emit) docs_out[obase + hoff] = ((u64)doc << 32) | sum;
            if (tid == 0 && flush) docs_out[dbase] = ((u64)c_doc << 32) | c_cnt;
            __syncthreads();
            if (is_last) {            // exactly one thread: the head of the tile's last run
                S.carry_doc = doc;
                S.carry_cnt = sum;
                S.carry_valid = 1;
                S.n_docs = obase + htotal;
            }
        }
        __syncthreads();
    }
    if (tid == 0 && S.carry_valid) {
        docs_out[S.n_docs] = ((u64)S.carry_doc << 32) | S.carry_cnt;
        S.n_docs += 1;
        S.carry_valid = 0;
    }
    __syncthreads();
}

// cur[i].count = min(cur[i].count, prev[doc].count) (0 if the doc is not in prev)
// == _intersect_bigram_matches (middle_out.py:73-93) on nested / sorted doc lists.
__device__ void and_min(u64 *__restrict__ cur, u64 n_cur, const u64 *__restrict__ prev, u64 n_prev) {
    for (u64 i = threadIdx.x; i < n_cur; i += PT) {
        u64 e = cur[i];
        u64 doc = e >> 32;
        u64 lo = 0, hi = n_prev;
        while (lo < hi) {
            u64 mid = (lo + hi) >> 1;
            if ((prev[mid] >> 32) < doc) lo = mid + 1; else hi = mid;
        }
        u32 c = 0;
        if (lo < n_prev && (prev[lo] >> 32) == doc) c = min((u32)(prev[lo] & 0xFFFFFFFFull), (u32)(e & 0xFFFFFFFFull));
        cur[i] = (doc << 32) | c;
    }
    __syncthreads();
}

struct ChainResult { u64 *docs; u64 n_docs; u64 *cont; u64 n_cont; };

// ---------------------------------------------------------------------------------------------------------------
// The SEARCH regime (|shortest list| << |the others|): one CTA per (query, doc-range chunk) runs the whole chain once
// over its chunk; a step's driver elements binary-search the other list in global memory, which skips most of it.
// DEEP (here and in phrase_tile_kernel): k > SA_TOPK_MAX, collected by deep_tile_collect.
template <bool DEEP>
__global__ void __launch_bounds__(PT, 4)
phrase_kernel(const PhraseArgs a) {
    __shared__ StepShared S;
    __shared__ u64 s_lo[SA_MAX_PHRASE_TERMS], s_n[SA_MAX_PHRASE_TERMS];
    __shared__ u64 s_slab;
    __shared__ int s_ok;
    __shared__ __align__(16) float s_tile[SA_TILE_DOCS];
    __shared__ u32 s_top[(PT / 32) * 8];
    __shared__ u32 s_ncand, s_tile_max;

    // grid = (queries, chunks): neighbouring CTAs belong to different queries (see term_tile_kernel)
    const u32 q = a.qsel ? a.qsel[blockIdx.x] : blockIdx.x;
    const u32 chunk = blockIdx.y;
    const PhraseQuery &pq = a.queries[q];
    const u32 n_terms = pq.n_terms;
    const unsigned tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const u64 d0 = a.doc_base + (u64)chunk * a.docs_per_chunk;
    const u64 dend = a.doc_base + a.n_docs;
    if (d0 >= dend) return;                    // (grid is sized so this does not happen)
    const u64 d1 = min(d0 + a.docs_per_chunk, dend);
    ChainResult fin;
    fin.docs = nullptr; fin.n_docs = 0; fin.cont = nullptr; fin.n_cont = 0;
    bool run = true;

    // 1. every term's slice for this doc range
    for (u32 t = warp; t < n_terms; t += PT / 32) {
        const u64 *lst = a.words + pq.off[t];
        u64 lo, hi;
        if (pq.dir_plus1[t] && a.tile_dir) {               // chunks are whole tiles: the list's tile directory has the slice
            const u32 *dir = a.tile_dir + (pq.dir_plus1[t] - 1);
            lo = __ldg(dir + (u32)(((u64)chunk * a.docs_per_chunk) / SA_TILE_DOCS));
            hi = __ldg(dir + (u32)((d1 - a.doc_base + SA_TILE_DOCS - 1) / SA_TILE_DOCS));
        } else {
            lo = warp_lower_bound_shifted(lst, 0, pq.len[t], d0, SA_KEY_SHIFT);
            hi = warp_lower_bound_shifted(lst, lo, pq.len[t], d1, SA_KEY_SHIFT);
        }
        if (lane == 0) { s_lo[t] = lo; s_n[t] = hi - lo; }
    }
    __syncthreads();
    u64 cap = 0, widest = 0;
    for (u32 t = 0; t < n_terms; t++) {
        cap = max(cap, s_n[t]);
        if (s_n[t]) widest++;
    }
    // A chunk where fewer than two terms occur has no pairs at any step.  (A chunk that merely
    // misses ONE term must still run its earlier steps: their pairs count towards the global
    // same-term decision of the reference.)
    if (widest < 2) run = false;
    cap += 2;

    // 2. scratch slab: 2 continuation buffers + 4 (doc,count) buffers
    if (tid == 0) {
        s_ok = 1;
        s_slab = 0;
        if (run) {
            unsigned long long need = 6ull * cap;
            unsigned long long at = atomicAdd(a.arena_used, need);
            s_ok = (at + need <= a.arena_cap);
            s_slab = at;
            if (!s_ok) atomicExch(&a.stats[q].overflow, 1u);
        }
    }
    __syncthreads();
    if (!s_ok) run = false;
    u64 *contA = a.arena + s_slab, *contB = contA + cap;
    u64 *docsA = contB + cap, *docsB = docsA + cap, *docsL = docsB + cap, *docsR = docsL + cap;

    auto slice = [&](u32 t) { return a.words + pq.off[t] + s_lo[t]; };

    // Runs one chain over terms [ta, tb).  lr: left-to-right (cont = RHS) else right-to-left.
    auto run_chain = [&](u32 ta, u32 tb, bool lr, u64 *final_docs) -> ChainResult {
        ChainResult res;
        res.docs = final_docs;
        res.n_docs = 0;
        res.cont = contA;
        res.n_cont = 0;
        const u64 *carry = lr ? slice(ta) : slice(tb - 1);
        u64 n_carry = lr ? s_n[ta] : s_n[tb - 1];
        u64 *cont_bufs[2] = {contA, contB};
        u64 *doc_bufs[2] = {docsA, docsB};
        int flip = 0;
        const u64 *prev_docs = nullptr;
        u64 n_prev = 0;
        const u32 n_steps = tb - ta - 1;
        for (u32 s = 0; s < n_steps; s++) {
            const u32 tnew = lr ? (ta + 1 + s) : (tb - 2 - s);     // also the step id
            const bool same = (pq.same_guess >> tnew) & 1u;
            const u64 *other = slice(tnew);
            const u64 n_other = s_n[tnew];
            if (n_carry == 0 || n_other == 0) {   // no pairs from here on in this doc range
                res.n_docs = 0;
                res.n_cont = 0;
                break;
            }
            u64 *cont_out = cont_bufs[flip];
            u64 *docs_out = (s == n_steps - 1) ? final_docs : doc_bufs[flip];
            // the first step may drive from the shorter side; later steps drive from the carry
            const bool drive_carry = (s > 0) || (n_carry <= n_other);
            if (lr) {
                if (drive_carry) bigram_step<true, true>(carry, n_carry, other, n_other, same, cont_out, docs_out, S);
                else bigram_step<true, false>(other, n_other, carry, n_carry, same, cont_out, docs_out, S);
            } else {
                if (drive_carry) bigram_step<false, false>(carry, n_carry, other, n_other, same, cont_out, docs_out, S);
                else bigram_step<false, true>(other, n_other, carry, n_carry, same, cont_out, docs_out, S);
            }
            const u64 n_cont = S.n_cont, n_docs = S.n_docs;
            if (tid == 0) {
                if (S.st_inner) atomicAdd(&a.stats[q].n_inner[tnew], S.st_inner);
                if (S.st_diff) atomicAdd(&a.stats[q].n_diff[tnew], S.st_diff);
                if (n_cont) atomicAdd(&a.stats[q].n_cont, (unsigned long long)n_cont);
            }
            __syncthreads();
            if (prev_docs) and_min(docs_out, n_docs, prev_docs, n_prev);
            prev_docs = docs_out;
            n_prev = n_docs;
            carry = cont_out;
            n_carry = n_cont;
            res.docs = docs_out;
            res.n_docs = n_docs;
            res.cont = cont_out;
            res.n_cont = n_cont;
            flip ^= 1;
            if (n_docs == 0) {       // nothing can survive the remaining steps
                res.n_docs = 0;
                break;
            }
        }
        return res;
    };

    if (run) {
    if (pq.mode == SA_PHRASE_MODE_LR) {
        fin = run_chain(0, n_terms, true, docsL);
    } else if (pq.mode == SA_PHRASE_MODE_RL) {
        fin = run_chain(0, n_terms, false, docsL);
    } else {
        // both chains always run (their pair statistics feed the speculation check)
        ChainResult left = run_chain(0, pq.split, true, docsL);
        fin = run_chain(pq.split, n_terms, false, docsR);
        if (left.n_docs == 0) fin.n_docs = 0;
        and_min(fin.docs, fin.n_docs, left.docs, left.n_docs);
    }

    }
    // optional dump for the per-op parity export (single chunk)
    if (a.dump.cont) {
        for (u64 i = tid; i < fin.n_cont; i += PT) a.dump.cont[i] = fin.cont[i];
        for (u64 i = tid; i < fin.n_docs; i += PT) a.dump.docs[i] = fin.docs[i];
        if (tid == 0) { *a.dump.n_cont = fin.n_cont; *a.dump.n_docs = fin.n_docs; }
    }

    // 3. materialise the dense vector of this doc range tile by tile (phrase_freqs[ids] = counts,
    //    middle_out.py:441): zeros + the matches that fall in the tile, flushed with 16-byte
    //    streaming stores; the same pass collects the tile's top-k candidates.
    float *out = a.out + (u64)q * a.out_stride;
    Bm25Params p = a.bm25;
    p.idf = pq.idf;
    const u32 row = a.topk_row0 + q;
    const u32 tile0 = (u32)(((u64)chunk * a.docs_per_chunk) / SA_TILE_DOCS);
    const u32 tile1 = (u32)((d1 - a.doc_base + SA_TILE_DOCS - 1) / SA_TILE_DOCS);
    // fin.docs is sorted by doc and the tiles ascend: a running cursor replaces a search per tile.
    // Most tiles hold no match at all: they are written as zeros straight from registers (no shared
    // tile, no barrier), so the bulk of the 4*N write runs at fill speed.
    u64 cur = 0;
    u64 next_doc = fin.n_docs ? (fin.docs[0] >> 32) : ~0ull;          // CTA-uniform
    for (u32 tile = tile0; tile < tile1; tile++) {
        const u64 t_abs1 = a.doc_base + (u64)tile * SA_TILE_DOCS + SA_TILE_DOCS;
        if (next_doc >= t_abs1) {
            store_empty_tile<PT>(out + (u64)tile * SA_TILE_DOCS, a.topk, row, tile);
            continue;
        }
        // first entry at or past the end of this tile: gallop from the cursor, then bisect (uniform)
        const u64 m0 = cur;
        u64 lo = cur + 1, hi = fin.n_docs, st = 1;
        while (lo < hi) {
            const u64 probe = min(lo + st - 1, hi - 1);
            if ((fin.docs[probe] >> 32) < t_abs1) { lo = probe + 1; st <<= 1; }
            else { hi = probe; break; }
        }
        while (lo < hi) {
            const u64 mid = (lo + hi) >> 1;
            if ((fin.docs[mid] >> 32) < t_abs1) lo = mid + 1; else hi = mid;
        }
        const u64 m1 = lo;
        cur = m1;
        next_doc = m1 < fin.n_docs ? (fin.docs[m1] >> 32) : ~0ull;
#pragma unroll
        for (int i = 0; i < SA_TILE_DOCS / PT / 4; i++)
            reinterpret_cast<float4 *>(s_tile)[tid + i * PT] = make_float4(0.f, 0.f, 0.f, 0.f);
        __syncthreads();
        u32 my_max = 0, my_match = 0;
        for (u64 i = m0 + tid; i < m1; i += PT) {
            const u64 e = fin.docs[i];
            const u32 c = (u32)(e & 0xFFFFFFFFull);
            if (c == 0) continue;
            const u64 d = (e >> 32) - a.doc_base;
            if (d >= a.n_docs) continue;
            my_match++;
            const float v = a.score ? bm25_one((float)c, __ldg(a.doc_lens + d), p) : (float)c;
            s_tile[d - (u64)tile * SA_TILE_DOCS] = v;
            if (v > 0.0f) my_max = max(my_max, __float_as_uint(v));
        }
        my_match = __reduce_add_sync(0xffffffffu, my_match);
        if (lane == 0 && my_match) atomicAdd(&a.stats[q].n_match, my_match);
        __syncthreads();
        flush_tile_collect<true, DEEP>(s_tile, out + (u64)tile * SA_TILE_DOCS, a.topk, row, tile, my_max, (u32)(m1 - m0),
                           (u32)min(m1 - m0, (u64)PT), s_top, &s_ncand, &s_tile_max);
    }
}

// ---------------------------------------------------------------------------------------------------------------
// The CONJUNCTION regime (balanced lists): one CTA per (query, 8192-doc tile), like the term scan -- small shared
// memory footprint, five CTAs per SM, latency hidden by occupancy.  A doc can only match if it holds EVERY term of the
// phrase, so the CTA streams the tile's slice of every term ONCE with coalesced loads and sets bits in per-term
// doc-presence bitmaps (shared-memory atomicOr), ANDs them, and in the (rare) tiles where candidate docs exist each
// warp takes its 1,024 docs: lane-parallel binary searches for its sub-slice bounds, ordered compaction of the
// candidates' words by ballots, the whole bigram chain at warp scope (sa_phrase_warp.cuh) -- all inside the warp's own
// 4 KB of the tile.  HBM traffic: 8 * sum(W) + 4 * N, each list read once, sequentially: the B_phrase of SURVEY 8d
// without its continuation term.  A sub-range whose candidates do not fit its compaction area flags the query for
// the exact re-run in the search regime (the host routes phrases whose terms co-occur that often there up front).
// The pair statistics of the same-term speculation cover the candidate docs only: enough to CONFIRM a guess, not to
// derive the reference's global decision from, so any disagreement also re-runs the query in the search regime.
template <bool DEEP>
__global__ void __launch_bounds__(PT, 5)
phrase_tile_kernel(const PhraseArgs a) {
    __shared__ __align__(16) float s_tile[SA_TILE_DOCS];
    __shared__ u32 s_top[(PT / 32) * 8];
    __shared__ u32 s_ncand, s_tile_max;
    __shared__ u32 s_wmatch[PT / 32];
    __shared__ const u64 *s_ptr[PT / 32][SA_MAX_PHRASE_TERMS];
    __shared__ u32 s_n[PT / 32][SA_MAX_PHRASE_TERMS];

    const u32 q = a.qsel ? a.qsel[blockIdx.x] : blockIdx.x;
    const u32 tile = blockIdx.y;
    const PhraseQuery &pq = a.queries[q];
    const u32 n_terms = pq.n_terms;
    const unsigned tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const u64 td0 = a.doc_base + (u64)tile * SA_TILE_DOCS;
    const u64 td1 = min(td0 + SA_TILE_DOCS, a.doc_base + a.n_docs);
    float *out = a.out + (u64)q * a.out_stride;
    const u32 row = a.topk_row0 + q;

    // the tile's slice of term `lane`: its tile directory, or (short lists) a search
    u64 t_lo = 0;
    u32 t_n = 0;
    for (u32 t = 0; t < n_terms; t++) {
        if (pq.dir_plus1[t] && a.tile_dir) continue;
        const u64 *lst = a.words + pq.off[t];                                  // (all lanes search, lane t keeps the result)
        const u64 lo = warp_lower_bound_shifted(lst, 0, pq.len[t], td0, SA_KEY_SHIFT);
        const u64 hi = warp_lower_bound_shifted(lst, lo, pq.len[t], td1, SA_KEY_SHIFT);
        if (lane == t) { t_lo = lo; t_n = (u32)(hi - lo); }
    }
    if (lane < n_terms && pq.dir_plus1[lane] && a.tile_dir) {
        const u32 *dir = a.tile_dir + (pq.dir_plus1[lane] - 1) + tile;
        t_lo = __ldg(dir);
        t_n = __ldg(dir + 1) - (u32)t_lo;
    }
    const bool all_present = __all_sync(0xffffffffu, lane >= n_terms || t_n > 0);

    u32 c = 0;                                                                  // candidate docs: 32 per thread
    if (all_present) {                                                          // CTA-uniform
        u32 *term_bm = reinterpret_cast<u32 *>(s_tile);                         // [n_terms][256]
        for (u32 i = tid; i < n_terms * (SA_TILE_DOCS / 32); i += PT) term_bm[i] = 0u;
        __syncthreads();
        for (u32 t = 0; t < n_terms; t++) {
            const u64 *lst = a.words + pq.off[t] + __shfl_sync(0xffffffffu, t_lo, t);
            const u32 n = __shfl_sync(0xffffffffu, t_n, t);
            u32 *bm = term_bm + t * (SA_TILE_DOCS / 32);
            u32 i = tid;
            for (; i + 3 * PT < n; i += 4 * PT) {                               // four independent loads in flight per thread
                const u64 w0 = ld_stream_u64(lst + i), w1 = ld_stream_u64(lst + i + PT);
                const u64 w2 = ld_stream_u64(lst + i + 2 * PT), w3 = ld_stream_u64(lst + i + 3 * PT);
                const u32 r0 = (u32)((w0 >> SA_KEY_SHIFT) - td0), r1 = (u32)((w1 >> SA_KEY_SHIFT) - td0);
                const u32 r2 = (u32)((w2 >> SA_KEY_SHIFT) - td0), r3 = (u32)((w3 >> SA_KEY_SHIFT) - td0);
                atomicOr(&bm[r0 >> 5], 1u << (r0 & 31u));
                atomicOr(&bm[r1 >> 5], 1u << (r1 & 31u));
                atomicOr(&bm[r2 >> 5], 1u << (r2 & 31u));
                atomicOr(&bm[r3 >> 5], 1u << (r3 & 31u));
            }
            for (; i < n; i += PT) {
                const u32 rel = (u32)((ld_stream_u64(lst + i) >> SA_KEY_SHIFT) - td0);
                atomicOr(&bm[rel >> 5], 1u << (rel & 31u));
            }
        }
        __syncthreads();
        c = term_bm[tid];
        for (u32 t = 1; t < n_terms; t++) c &= term_bm[t * (SA_TILE_DOCS / 32) + tid];
        __syncthreads();                                                        // the bitmaps are dead: the warps' slices are free
    }

    // ---- candidate docs (rare): every warp on its own 1,024 docs, inside its own 4 KB of the tile
    float *my_slice = s_tile + warp * PW_SUB_DOCS;
    u64 res[2] = {0ull, 0ull};                                                  // this lane's (doc << 32 | count) results
    u32 n_res = 0;
    if (__reduce_add_sync(0xffffffffu, (u32)__popc(c))) {                       // warp-uniform
        u32 *wcand = reinterpret_cast<u32 *>(my_slice);                         // [32]
        // capacities so that candidates + the chain's six buffers fit in the slice
        const u32 fb_cap = (PW_SUB_DOCS * 4 - 128 - 96) / (8 * n_terms + 48);
        u64 *fb = reinterpret_cast<u64 *>(wcand + 32);                          // [n_terms][fb_cap]
        u64 *chain_buf = fb + (u64)n_terms * fb_cap;                            // 6 x (fb_cap + 2)
        const u64 w_d0 = td0 + (u64)warp * PW_SUB_DOCS, w_d1 = w_d0 + PW_SUB_DOCS;
        wcand[lane] = c;
        // sub-slice bounds: lane 2t searches the lower, lane 2t+1 the upper doc bound of term t (global memory, L2-hot)
        u32 bound = 0;
        {
            const u32 t = lane >> 1;
            const u64 lo_t = __shfl_sync(0xffffffffu, t_lo, t);
            const u32 n = __shfl_sync(0xffffffffu, t_n, t);
            if (t < n_terms) bound = w_lower_bound_doc(a.words + pq.off[t] + lo_t, n, (lane & 1u) ? w_d1 : w_d0);
        }
        __syncwarp();
        bool fits = true;
        for (u32 t = 0; t < n_terms; t++) {
            const u64 *base = a.words + pq.off[t] + __shfl_sync(0xffffffffu, t_lo, t);
            const u32 lo = __shfl_sync(0xffffffffu, bound, 2 * t), hi = __shfl_sync(0xffffffffu, bound, 2 * t + 1);
            u64 *dst = fb + (u64)t * fb_cap;
            u32 kept = 0;
            for (u32 i0 = lo; i0 < hi; i0 += 32) {                             // ordered compaction by ballots
                const u32 i = i0 + lane;
                u64 w = 0;
                bool keep = false;
                if (i < hi) {
                    w = base[i];
                    const u32 rel = (u32)((w >> SA_KEY_SHIFT) - w_d0);
                    keep = (wcand[rel >> 5] >> (rel & 31u)) & 1u;
                }
                const unsigned m = __ballot_sync(0xffffffffu, keep);
                const u32 at = kept + __popc(m & ((1u << lane) - 1u));
                if (keep && at < fb_cap) dst[at] = w;
                kept += __popc(m);
            }
            fits = fits && kept <= fb_cap;
            if (lane == 0) { s_ptr[warp][t] = dst; s_n[warp][t] = min(kept, fb_cap); }
        }
        __syncwarp();
        if (fits) {
            const WarpFin wf = warp_phrase_chain(pq, s_ptr[warp], s_n[warp], chain_buf, fb_cap + 2, &a.stats[q]);
            n_res = wf.n_docs;                                                   // <= fb_cap + 2 <= 64: two per lane
            if (lane < n_res) res[0] = wf.docs[lane];
            if (lane + 32 < n_res) res[1] = wf.docs[lane + 32];
        } else if (lane == 0) {
            atomicExch(&a.stats[q].overflow, 2u);                               // dense conjunction: re-run in the search regime
        }
        __syncwarp();
    }
    // ---- this warp's 4 KB of the dense tile: zeros + its matches
#pragma unroll
    for (int i = 0; i < PW_SUB_DOCS / 32 / 4; i++)
        reinterpret_cast<float4 *>(my_slice)[lane + i * 32] = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncwarp();
    u32 my_max = 0, my_match = 0;
    Bm25Params p = a.bm25;
    p.idf = pq.idf;
#pragma unroll
    for (int j = 0; j < 2; j++) {
        if (lane + 32 * j >= n_res) continue;
        const u32 cnt = (u32)(res[j] & 0xFFFFFFFFull);
        if (cnt == 0) continue;
        const u64 d = (res[j] >> 32) - a.doc_base;
        if (d >= a.n_docs) continue;
        my_match++;
        const float v = a.score ? bm25_one((float)cnt, __ldg(a.doc_lens + d), p) : (float)cnt;
        s_tile[d - (u64)tile * SA_TILE_DOCS] = v;
        if (v > 0.0f) my_max = max(my_max, __float_as_uint(v));
    }
    my_match = __reduce_add_sync(0xffffffffu, my_match);
    if (lane == 0) {
        if (my_match) atomicAdd(&a.stats[q].n_match, my_match);
        s_wmatch[warp] = my_match;
    }
    __syncthreads();
    u32 total = 0, holders = 0;
#pragma unroll
    for (int w = 0; w < PT / 32; w++) { total += s_wmatch[w]; holders += min(s_wmatch[w], 32u); }
    if (total == 0) {
        store_empty_tile<PT>(out + (u64)tile * SA_TILE_DOCS, a.topk, row, tile);
        return;
    }
    flush_tile_collect<true, DEEP>(s_tile, out + (u64)tile * SA_TILE_DOCS, a.topk, row, tile, my_max, total, holders, s_top,
                                   &s_ncand, &s_tile_max);
}

int launch_phrase(sa_index *ix, const PhraseArgs &a, u32 n_queries) {
    if (n_queries == 0 || a.n_docs == 0) return SA_OK;
    dim3 grid(n_queries, a.n_chunks);
    KernelTimer t(ix, 2);
    if (a.topk.k > SA_TOPK_MAX) phrase_kernel<true><<<grid, PT, 0, ix->stream>>>(a);
    else phrase_kernel<false><<<grid, PT, 0, ix->stream>>>(a);
    SA_CUDA(cudaGetLastError());
    if (a.topk.k > SA_TOPK_MAX) ix->stats.deep_tiles += (u64)n_queries * sa_n_tiles(a.n_docs);
    t.stop();
    ix->stats.phrase_kernel_launches++;
    ix->stats.total_launches++;
    return SA_OK;
}

// conjunction regime: one CTA per (query, tile), like the term scan
static int launch_phrase_tile(sa_index *ix, const PhraseArgs &a, u32 n_queries) {
    if (n_queries == 0 || a.n_docs == 0) return SA_OK;
    KernelTimer t(ix, 2);
    if (a.topk.k > SA_TOPK_MAX) phrase_tile_kernel<true><<<dim3(n_queries, sa_n_tiles(a.n_docs)), PT, 0, ix->stream>>>(a);
    else phrase_tile_kernel<false><<<dim3(n_queries, sa_n_tiles(a.n_docs)), PT, 0, ix->stream>>>(a);
    SA_CUDA(cudaGetLastError());
    if (a.topk.k > SA_TOPK_MAX) ix->stats.deep_tiles += (u64)n_queries * sa_n_tiles(a.n_docs);
    t.stop();
    ix->stats.phrase_kernel_launches++;
    ix->stats.phrase_tile_launches++;
    ix->stats.total_launches++;
    return SA_OK;
}

// Conjunction regime or search regime?  The conjunction regime reads every list once (8 * sum(W) bytes); the search
// path costs about `ratio` bytes (a dozen 32-byte sectors of dependent probes) per driver element of the first step.
bool sa_phrase_use_conjunction(const PhraseQuery &pq, u64 n_docs) {
    const char *s = getenv("SA_PHRASE_STAGE_RATIO");             // read on every call, like the term knobs
    const long env = s ? atol(s) : -1;
    const u64 ratio = env >= 0 ? (u64)env : 50;
    if (ratio == 0) return false;
    const u32 n = pq.n_terms;
    if (n < 2) return false;
    // expected candidate words per 1,024-doc sub-range (terms taken as independent): they must fit the warp's
    // compaction area with room to spare, or the conjunction regime would keep bouncing the query to the search regime
    double est = (double)PW_SUB_DOCS;
    for (u32 t = 0; t < n; t++) est *= std::min(1.0, (double)pq.len[t] / (double)std::max<u64>(n_docs, 1));
    const double fb_cap = (double)((PW_SUB_DOCS * 4 - 128 - 96) / (8 * n + 48));
    if (est * 1.5 * 3.0 > fb_cap) return false;
    u64 sum = 0, drive = ~0ull;
    for (u32 t = 0; t < n; t++) {
        sum += pq.len[t];
        if (pq.len[t] == 0) return false;
    }
    if (pq.mode == SA_PHRASE_MODE_LR) drive = std::min(pq.len[0], pq.len[1]);
    else if (pq.mode == SA_PHRASE_MODE_RL) drive = std::min(pq.len[n - 1], pq.len[n - 2]);
    else {
        drive = std::min(pq.len[n - 1], pq.len[n - 2]);
        if (pq.split >= 2) drive = std::max(drive, std::min(pq.len[0], pq.len[1]));
    }
    return drive * ratio > sum;
}

// ------------------------------------------------------------------------------- host side
// BM25 over every doc (bm25.pyx:20-25) for parameter sets where tf == 0 does not score +0.0.
__global__ void bm25_dense_kernel(float *__restrict__ tf, const float *__restrict__ dl, u64 n, Bm25Params p) {
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) tf[i] = bm25_one(tf[i], dl[i], p);
}

// direction / speculation plan exactly as compute_phrase_freqs picks it (middle_out.py:154-168)
void sa_phrase_plan(PhraseQuery &pq, const u32 *term_ids) {
    const u32 n = pq.n_terms;
    u32 shortest = 0;
    for (u32 i = 1; i < n; i++) if (pq.len[i] < pq.len[shortest]) shortest = i;   // first minimum
    pq.same_guess = 0;
    if (shortest <= 1) {
        pq.mode = SA_PHRASE_MODE_LR;
        if (term_ids[0] == term_ids[1]) pq.same_guess |= 1u << 1;
    } else if (shortest >= n - 2) {
        pq.mode = SA_PHRASE_MODE_RL;
        if (term_ids[n - 2] == term_ids[n - 1]) pq.same_guess |= 1u << (n - 2);
    } else {
        pq.mode = SA_PHRASE_MODE_MID;
        pq.split = shortest;
        if (term_ids[0] == term_ids[1]) pq.same_guess |= 1u << 1;
        if (term_ids[n - 2] == term_ids[n - 1]) pq.same_guess |= 1u << (n - 2);
    }
}

PhraseQuery make_phrase_query(const u32 *term_ids, u32 n, const u64 *offs, const u64 *lens, const u64 *dirs,
                              float idf, bool missing) {
    PhraseQuery pq;
    memset(&pq, 0, sizeof(pq));
    pq.n_terms = n;
    pq.idf = idf;
    for (u32 i = 0; i < n; i++) {
        pq.off[i] = offs[i];
        pq.len[i] = missing ? 0 : lens[i];       // unknown term -> no pairs -> zeros (postings.py:705-708)
        if (!missing && dirs && dirs[i] != SA_NO_DIR) pq.dir_plus1[i] = dirs[i] + 1;
    }
    sa_phrase_plan(pq, term_ids);               // after the zeroing: the plan follows the lengths
    return pq;
}

// order in which the steps of a plan run (for verifying the speculation)
static void step_order(const PhraseQuery &pq, std::vector<u32> &order) {
    order.clear();
    const u32 n = pq.n_terms;
    if (pq.mode == SA_PHRASE_MODE_LR) for (u32 s = 1; s < n; s++) order.push_back(s);
    else if (pq.mode == SA_PHRASE_MODE_RL) for (int s = (int)n - 2; s >= 0; s--) order.push_back((u32)s);
    else {
        for (u32 s = 1; s < pq.split; s++) order.push_back(s);
        for (int s = (int)n - 2; s >= (int)pq.split; s--) order.push_back((u32)s);
    }
}

// Launch arguments of both regimes.  The kernels write every tile of the dense rows themselves: no zero-fill pass.
static PhraseArgs phrase_args(const sa_index *ix, const u64 *d_words, const PhraseQuery *d_pqs, PhraseStats *d_stats,
                              float *dense_rows, u64 stride, DocChunks chunks, u64 *d_arena,
                              unsigned long long *d_arena_used, u64 arena_words, int score, const Bm25Params &p) {
    PhraseArgs a;
    memset(&a, 0, sizeof(a));
    a.words = d_words;
    a.tile_dir = (d_words == ix->d_words.as<u64>()) ? ix->d_tile_dir.as<u32>() : nullptr;
    a.doc_lens = ix->d_doc_lens.as<float>();
    a.n_docs = ix->n_docs;
    a.doc_base = ix->doc_base;
    a.queries = d_pqs;
    a.stats = d_stats;
    a.out = dense_rows;
    a.out_stride = stride;
    a.n_chunks = chunks.n_chunks;
    a.docs_per_chunk = chunks.docs_per_chunk;
    a.arena = d_arena;
    a.arena_used = d_arena_used;
    a.arena_cap = arena_words;
    a.bm25 = p;
    a.score = score;
    return a;
}

// Runs phrase queries (already planned) into ix->dense; loops until the same-term speculation
// of every query is confirmed.  lists may live in ix->d_words (off = absolute word offsets).
// allow_conj: a single query on the index's own lists may take the conjunction regime; otherwise
// every query runs in the search regime, whose pair statistics cover every pair.  A dump runs as one chunk.
int sa_phrase_run_sync(sa_index *ix, std::vector<PhraseQuery> &pqs, const u64 *d_words,
                       int score, const Bm25Params &p, PhraseDump dump, bool allow_conj) {
    const u32 Q = (u32)pqs.size();
    const u64 stride = sa_padded_docs(ix->n_docs);
    int rc;
    if ((rc = ix->dense.reserve((size_t)Q * stride * sizeof(float)))) return rc;
    if ((rc = ix->queries.reserve((size_t)Q * sizeof(PhraseQuery)))) return rc;
    if ((rc = ix->cand_meta.reserve((size_t)Q * sizeof(PhraseStats) + 64))) return rc;
    const DocChunks chunks = dump.cont ? DocChunks{1, stride} : phrase_doc_chunks(ix, Q, 8);
    u64 arena_words = 64;
    for (auto &pq : pqs) arena_words += sa_phrase_arena_words(pq, chunks.n_chunks);
    // the conjunction regime needs no bump arena
    bool conj = allow_conj && Q == 1 && d_words == ix->d_words.as<u64>() && !dump.cont && sa_phrase_use_conjunction(pqs[0], ix->n_docs);
    const u64 full_arena_words = arena_words;
    const std::vector<PhraseQuery> pqs_in = pqs;
    if (conj) arena_words = 64;
    if ((rc = ix->phrase_scratch.reserve(arena_words * sizeof(u64) + 64))) return rc;
    unsigned long long *d_used = (unsigned long long *)ix->phrase_scratch.p;
    u64 *d_arena = (u64 *)ix->phrase_scratch.p + 8;
    PhraseStats *d_stats = (PhraseStats *)ix->cand_meta.p;
    std::vector<PhraseStats> h_stats(Q);

    for (int attempt = 0; attempt < (int)SA_MAX_PHRASE_TERMS + 2; attempt++) {
        SA_CUDA(cudaMemcpyAsync(ix->queries.p, pqs.data(), (size_t)Q * sizeof(PhraseQuery), cudaMemcpyHostToDevice, ix->stream));
        SA_CUDA(cudaMemsetAsync(d_stats, 0, (size_t)Q * sizeof(PhraseStats), ix->stream));
        SA_CUDA(cudaMemsetAsync(d_used, 0, 64, ix->stream));
        PhraseArgs a = phrase_args(ix, d_words, ix->queries.as<PhraseQuery>(), d_stats, ix->dense.as<float>(), stride,
                                   chunks, d_arena, d_used, arena_words, score, p);
        a.dump = dump;
        if ((rc = conj ? launch_phrase_tile(ix, a, Q) : launch_phrase(ix, a, Q))) return rc;
        SA_CUDA(cudaMemcpyAsync(h_stats.data(), d_stats, (size_t)Q * sizeof(PhraseStats), cudaMemcpyDeviceToHost, ix->stream));
        SA_CUDA(cudaStreamSynchronize(ix->stream));
        bool again = false;
        for (u32 q = 0; q < Q; q++) {
            SA_CHECK(h_stats[q].overflow != 1, "phrase scratch arena exhausted (internal sizing error)");
            // overflow 2: dense conjunction, the search regime takes it; a wrong guess is flipped for the next attempt
            if (h_stats[q].overflow == 2 || !sa_phrase_guess_ok(pqs[q], h_stats[q])) again = true;
        }
        if (!again) return SA_OK;
        if (conj) {
            // The conjunction regime's pair statistics only CONFIRM a guess (phrase_tile_kernel): on any disagreement
            // the query starts over in the search regime, whose statistics cover every pair.
            conj = false;
            pqs = pqs_in;
            arena_words = full_arena_words;
            if ((rc = ix->phrase_scratch.reserve(arena_words * sizeof(u64) + 64))) return rc;
            d_used = (unsigned long long *)ix->phrase_scratch.p;
            d_arena = (u64 *)ix->phrase_scratch.p + 8;
        }
    }
    sa_set_error("same-term speculation did not converge");
    return SA_ERR_ARG;
}

// Checks the same-term speculation of one finished query; on the first wrong guess (in step
// order) flips it and returns false: the query must run again.
bool sa_phrase_guess_ok(PhraseQuery &pq, const PhraseStats &st) {
    std::vector<u32> order;
    step_order(pq, order);
    for (u32 s : order) {
        bool actual = st.n_inner[s] > 0 && st.n_diff[s] == 0;
        bool guess = (pq.same_guess >> s) & 1u;
        if (actual != guess) {
            pq.same_guess ^= 1u << s;
            return false;
        }
    }
    return true;
}

u64 sa_phrase_arena_words(const PhraseQuery &pq, u32 n_chunks) {
    u64 sum = 0;
    for (u32 t = 0; t < pq.n_terms; t++) sum += pq.len[t];
    return 6 * (sum + 2ull * n_chunks);
}

// About `ctas_per_sm` CTAs per SM over `n_queries` queries, in chunks of whole tiles: the tile count per chunk is
// rounded up, then the tiles are spread evenly over the chunks that takes.
DocChunks phrase_doc_chunks(const sa_index *ix, u32 n_queries, u32 ctas_per_sm) {
    const u64 n_tiles = sa_n_tiles(ix->n_docs);
    const u64 wanted = std::max<u64>(1, (u64)ix->num_sms * ctas_per_sm / std::max<u32>(n_queries, 1));
    const u64 tiles_per_chunk = std::max<u64>(1, (n_tiles + wanted - 1) / wanted);
    DocChunks c;
    c.n_chunks = (u32)((n_tiles + tiles_per_chunk - 1) / tiles_per_chunk);
    c.docs_per_chunk = c.n_chunks ? (n_tiles + c.n_chunks - 1) / c.n_chunks * SA_TILE_DOCS : 0;
    return c;
}

// Asynchronous launch of already planned phrase queries living in device memory; dense rows,
// stats and the arena counter must have been zeroed by the caller.
int sa_phrase_enqueue(sa_index *ix, const PhraseQuery *d_pqs, PhraseStats *d_stats, u32 Q,
                      float *dense_rows, u64 stride, DocChunks chunks, u64 *d_arena,
                      unsigned long long *d_arena_used, u64 arena_words, int score, const Bm25Params &p,
                      const TopkCtx *topk, u32 topk_row0, const PhraseSplit *split) {
    PhraseArgs a = phrase_args(ix, ix->d_words.as<u64>(), d_pqs, d_stats, dense_rows, stride, chunks, d_arena, d_arena_used,
                               arena_words, score, p);
    if (topk) a.topk = *topk;
    a.topk_row0 = topk_row0;
    if (!split) return launch_phrase(ix, a, Q);
    int rc;
    a.qsel = split->d_search;                   // search regime: one CTA per (query, chunk)
    if ((rc = launch_phrase(ix, a, split->n_search))) return rc;
    a.qsel = split->d_conj;
    return launch_phrase_tile(ix, a, split->n_conj);
}

int sa_phrase_row(sa_index *ix, const u32 *term_ids, u32 n_terms, u32 slop, const u64 *f_offs, const u64 *f_lens,
                  const Bm25Params *bm25, bool *scored) {
    u64 offs[SA_MAX_PHRASE_TERMS], lens[SA_MAX_PHRASE_TERMS], dirs[SA_MAX_PHRASE_TERMS];
    bool missing, literal;
    int rc = sa_resolve_terms(ix, term_ids, n_terms, offs, lens, dirs, &missing, &literal);
    if (rc) return rc;
    const Bm25Params p = bm25 ? *bm25 : make_bm25(0.0f, 1.0f, 1.0f, 0.0f, ix->doc_lens_nonneg);
    // sparse_ok: a zero count scores +0, so the phrase kernels may score the matches alone, and a zero row is scored
    const bool score = bm25 && p.sparse_ok;
    *scored = score && (slop == 0 || missing);
    if (missing) {                   // an unknown term inside a phrase -> zeros (postings.py:705-708)
        const u64 stride = sa_padded_docs(ix->n_docs);
        if ((rc = ix->dense.reserve(stride * sizeof(float)))) return rc;
        SA_CUDA(cudaMemsetAsync(ix->dense.p, 0, stride * sizeof(float), ix->stream));
        return SA_OK;
    }
    const u64 *d_lists = ix->d_words.as<u64>();
    if (f_offs) {
        d_lists = ix->filt.as<u64>();
        for (u32 i = 0; i < n_terms; i++) { offs[i] = f_offs[i]; lens[i] = f_lens[i]; dirs[i] = SA_NO_DIR; }
        if (slop > 0 && (rc = sa_span_is_literal(ix, d_lists, offs, lens, n_terms, &literal))) return rc;
    }
    // span search (phrase/spans.py + roaringish/spans.pyx): raw counts
    if (slop > 0) return sa_span_run(ix, d_lists, offs, lens, dirs, n_terms, slop, literal);
    std::vector<PhraseQuery> pqs(1, make_phrase_query(term_ids, n_terms, offs, lens, dirs, p.idf, false));
    PhraseDump nodump;
    memset(&nodump, 0, sizeof(nodump));
    return sa_phrase_run_sync(ix, pqs, d_lists, score, p, nodump, true);
}

static int phrase_common(sa_index *ix, const uint32_t *term_ids, uint32_t n_terms, uint32_t slop,
                         int score, float idf, float avg_doc_len, float k1, float b,
                         uint64_t min_payload, uint64_t max_payload, float *out_host) {
    SA_CHECK(ix && term_ids && out_host, "NULL argument");
    SA_CHECK(n_terms >= 2, "Must have at least two terms");
    SA_CHECK(n_terms <= SA_MAX_PHRASE_TERMS, "phrases longer than %d terms are not supported", SA_MAX_PHRASE_TERMS);
    std::lock_guard<std::mutex> g(ix->mu);
    SA_CUDA(cudaSetDevice(ix->device));
    if (ix->n_docs == 0) return SA_OK;
    u64 offs[SA_MAX_PHRASE_TERMS], lens[SA_MAX_PHRASE_TERMS], dirs[SA_MAX_PHRASE_TERMS];
    bool missing, literal;
    int rc = sa_resolve_terms(ix, term_ids, n_terms, offs, lens, dirs, &missing, &literal);
    if (rc) return rc;
    if (missing || (score && avg_doc_len == 0.0f)) {
        // unknown term inside a phrase -> zeros (postings.py:705-708); with tf == 0 everywhere BM25
        // still runs over all docs in the reference, which only matters for exotic parameters
        memset(out_host, 0, (ix->rows_active ? ix->n_rows : ix->n_docs) * sizeof(float));
        if (!(score && avg_doc_len != 0.0f) || ix->rows_active) return SA_OK;
    }
    const Bm25Params p = make_bm25(idf, avg_doc_len, k1, b, ix->doc_lens_nonneg);
    const bool use_payload = !(min_payload == 0 && max_payload == SA_ALL_BITS);
    const bool rows = ix->rows_active;
    SA_CHECK(!(rows && score), "score on a sliced array: call termfreqs + bm25 (the Python layer does)");
    // term lists: the index's own, or filtered copies (sliced array / min-max posn), which is what
    // the reference runs on (middle_out.py:427-437: encoder.slice per term, then the same algorithm)
    const bool filtered = !missing && (rows || use_payload);
    std::vector<u64> f_offs, f_lens;
    if (filtered && (rc = sa_filter_terms(ix, term_ids, n_terms, rows, min_payload, max_payload, use_payload, f_offs,
                                          f_lens))) return rc;
    bool scored;
    if ((rc = sa_phrase_row(ix, term_ids, n_terms, slop, filtered ? f_offs.data() : nullptr,
                            filtered ? f_lens.data() : nullptr, score ? &p : nullptr, &scored))) return rc;
    if (score && !scored) {     // bm25.pyx:20-25 over every doc (tf == 0 scores +0.0 for ordinary parameters)
        unsigned blocks = (unsigned)((ix->n_docs + 255) / 256);
        bm25_dense_kernel<<<blocks, 256, 0, ix->stream>>>(ix->dense.as<float>(), ix->d_doc_lens.as<float>(), ix->n_docs, p);
        SA_CUDA(cudaGetLastError());
        ix->stats.total_launches++;
    }
    return sa_copy_out_dense(ix, out_host);
}

extern "C" int sa_phrase_freqs(sa_index *ix, const uint32_t *term_ids, uint32_t n_terms, uint32_t slop,
                               uint64_t min_payload, uint64_t max_payload, float *out_host) {
    return phrase_common(ix, term_ids, n_terms, slop, 0, 0.0f, 1.0f, 1.0f, 0.0f, min_payload, max_payload, out_host);
}

extern "C" int sa_score_phrase(sa_index *ix, const uint32_t *term_ids, uint32_t n_terms, uint32_t slop,
                               float idf, float avg_doc_len, float k1, float b,
                               uint64_t min_payload, uint64_t max_payload, float *out_host) {
    return phrase_common(ix, term_ids, n_terms, slop, 1, idf, avg_doc_len, k1, b, min_payload, max_payload, out_host);
}

// ---------------------------------------------------------------- per-op parity exports
extern "C" int sa_op_bigram_freqs(const uint64_t *lhs, uint64_t n_lhs, const uint64_t *rhs, uint64_t n_rhs,
                                  int cont_rhs, int device,
                                  uint64_t *ids_out, float *counts_out, uint64_t *n_ids_out,
                                  uint64_t *next_out, uint64_t *n_next_out) {
    SA_CHECK(ids_out && counts_out && n_ids_out && next_out && n_next_out, "NULL argument");
    *n_ids_out = 0;
    *n_next_out = 0;
    if (n_lhs == 0 || n_rhs == 0) return SA_OK;
    SA_CHECK(lhs && rhs, "NULL argument");
    // a throw-away two-term index over one shard that covers every doc id present
    std::vector<u64> words(lhs, lhs + n_lhs);
    words.insert(words.end(), rhs, rhs + n_rhs);
    u64 max_doc = std::max(lhs[n_lhs - 1], rhs[n_rhs - 1]) >> SA_KEY_SHIFT;
    std::vector<float> dl(max_doc + 1, 1.0f);
    u64 offs[2] = {0, n_lhs}, lens[2] = {n_lhs, n_rhs};
    sa_index *created = nullptr;
    int rc = sa_index_create_blocks(words.data(), words.size(), offs, lens, 2, dl.data(), max_doc + 1, 0, device, false,
                                    &created);
    if (rc) return rc;
    std::unique_ptr<sa_index> ix(created);
    std::lock_guard<std::mutex> g(ix->mu);
    std::vector<PhraseQuery> pqs(1);
    PhraseQuery &pq = pqs[0];
    memset(&pq, 0, sizeof(pq));
    pq.n_terms = 2;
    pq.off[0] = 0; pq.len[0] = n_lhs;
    pq.off[1] = n_lhs; pq.len[1] = n_rhs;
    pq.mode = cont_rhs ? SA_PHRASE_MODE_LR : SA_PHRASE_MODE_RL;
    pq.same_guess = 0;
    const u64 cap = 2 * std::min(n_lhs, n_rhs) + std::max(n_lhs, n_rhs) + 8;
    DevBuf dbuf;
    if ((rc = dbuf.reserve((2 * cap + 2) * sizeof(u64)))) return rc;
    PhraseDump dump;
    dump.cont = dbuf.as<u64>();
    dump.docs = dump.cont + cap;
    dump.n_cont = dump.docs + cap;
    dump.n_docs = dump.n_cont + 1;
    SA_CUDA(cudaMemsetAsync(dump.n_cont, 0, 2 * sizeof(u64), ix->stream));
    Bm25Params p;
    memset(&p, 0, sizeof(p));
    if ((rc = sa_phrase_run_sync(ix.get(), pqs, ix->d_words.as<u64>(), 0, p, dump, false))) return rc;
    u64 n[2];
    SA_CUDA(cudaMemcpy(n, dump.n_cont, 2 * sizeof(u64), cudaMemcpyDeviceToHost));
    std::vector<u64> docs(n[1]);
    SA_CUDA(cudaMemcpy(next_out, dump.cont, n[0] * sizeof(u64), cudaMemcpyDeviceToHost));
    if (n[1]) SA_CUDA(cudaMemcpy(docs.data(), dump.docs, n[1] * sizeof(u64), cudaMemcpyDeviceToHost));
    for (u64 i = 0; i < n[1]; i++) {
        ids_out[i] = docs[i] >> 32;
        counts_out[i] = (float)(u32)(docs[i] & 0xFFFFFFFFull);
    }
    *n_next_out = n[0];
    *n_ids_out = n[1];
    return SA_OK;
}

// bm25_score on a raw array
extern "C" int sa_op_bm25_score(float *tf_inout, const float *doc_lens, uint64_t n, float avg_doc_len,
                                float idf, float k1, float b, int device) {
    if (n == 0) return SA_OK;
    SA_CHECK(tf_inout && doc_lens, "NULL argument");
    SA_CUDA(cudaSetDevice(device));
    DevBuf d_tf, d_dl;
    int rc;
    if ((rc = d_tf.allocate(n * sizeof(float))) || (rc = d_dl.allocate(n * sizeof(float)))) return rc;
    SA_CUDA(cudaMemcpy(d_tf.p, tf_inout, n * sizeof(float), cudaMemcpyHostToDevice));
    SA_CUDA(cudaMemcpy(d_dl.p, doc_lens, n * sizeof(float), cudaMemcpyHostToDevice));
    bm25_dense_kernel<<<(unsigned)((n + 255) / 256), 256>>>(d_tf.as<float>(), d_dl.as<float>(), n,
                                                          make_bm25(idf, avg_doc_len, k1, b, false));
    SA_CUDA(cudaGetLastError());
    SA_CUDA(cudaMemcpy(tf_inout, d_tf.p, n * sizeof(float), cudaMemcpyDeviceToHost));
    return SA_OK;
}

