// sa_phrase_warp.cuh -- the bigram chain at WARP scope, for the conjunction regime of sa_phrase.cu (phrase_tile_kernel).
//
// A warp runs the whole n-term chain on its own sub-range of docs without a single block barrier: driver elements are
// taken 32 at a time, partners are found by binary search, continuation words are emitted in order through ballots
// (`__ballot_sync` + popcount prefix), the per-doc counts are a segmented warp reduction (`__match_any_sync` groups of
// equal doc id, `__reduce_add_sync` inside the group), and a doc run crossing an iteration boundary is carried in
// registers.  Phrase matching never crosses a document, so the sub-ranges are independent (reference
// phrase/bigram_freqs.py:213-307 semantics per doc).
#pragma once
#include "sa_phrase.cuh"

// first index i in [0, n) with (a[i] >> 36) >= doc; plain loads (shared or global memory); every lane runs the same
// search on the same arguments (broadcast loads, no divergence)
__device__ __forceinline__ u32 w_lower_bound_doc(const u64 *a, u32 n, u64 doc) {
    u32 lo = 0, hi = n;
    while (lo < hi) {
        const u32 mid = (lo + hi) >> 1;
        if ((a[mid] >> SA_KEY_SHIFT) < doc) lo = mid + 1; else hi = mid;
    }
    return lo;
}

struct WarpStepOut { u32 n_cont, n_docs, st_inner, st_diff; };

// One bigram step over a warp's sub-range: the warp-scope twin of bigram_step (sa_phrase.cu).  Writes the
// continuation list (sorted) to cont_out and the per-doc counts (doc << 32 | count, sorted by doc, zero counts kept)
// to docs_out.  All 32 lanes call with identical arguments.
template <bool CONT_RHS, bool DRIVER_LHS>
__device__ __forceinline__ WarpStepOut warp_bigram_step(const u64 *D, u32 nD, const u64 *O, u32 nO, bool same,
                                                        u64 *cont_out, u64 *docs_out) {
    const unsigned lane = threadIdx.x & 31;
    const unsigned lt = (1u << lane) - 1u;
    WarpStepOut r;
    r.n_cont = r.n_docs = r.st_inner = r.st_diff = 0;
    u32 carry_doc = 0, carry_cnt = 0;
    bool carry_valid = false;
    for (u32 i0 = 0; i0 < nD; i0 += 32) {
        const u32 i = i0 + lane;
        Elem e;
        e.w0 = e.w1 = 0;
        e.n_emit = e.cnt = e.doc = 0;
        e.entry = e.inner = e.diff = false;
        if (i < nD) e = compute_elem<CONT_RHS, DRIVER_LHS>(D, (u64)nD, (u64)i, O, (u64)nO, same);
        r.st_inner += __popc(__ballot_sync(0xffffffffu, e.inner));
        r.st_diff += __popc(__ballot_sync(0xffffffffu, e.diff));
        // continuation words, in order
        const unsigned m1 = __ballot_sync(0xffffffffu, e.n_emit >= 1), m2 = __ballot_sync(0xffffffffu, e.n_emit == 2);
        const u32 off = r.n_cont + __popc(m1 & lt) + __popc(m2 & lt);
        if (e.n_emit >= 1) cont_out[off] = e.w0;
        if (e.n_emit == 2) cont_out[off + 1] = e.w1;
        r.n_cont += __popc(m1) + __popc(m2);
        // (doc, count) entries: docs ascend with the lane, equal docs are adjacent
        const unsigned me = __ballot_sync(0xffffffffu, e.entry);
        if (me == 0) continue;
        unsigned peers = 0;
        u32 sum = 0;
        if (e.entry) {
            peers = __match_any_sync(me, e.doc);
            sum = __reduce_add_sync(peers, e.cnt);
        }
        const int lo_lane = __ffs(me) - 1, hi_lane = 31 - __clz(me);
        const u32 first_doc = __shfl_sync(0xffffffffu, e.doc, lo_lane);
        const unsigned peers_hi = __shfl_sync(0xffffffffu, peers, hi_lane);          // the last (highest-doc) group
        const bool merge = carry_valid && first_doc == carry_doc;
        const bool flush = carry_valid && !merge;
        const bool leader = e.entry && (lane == (unsigned)(__ffs(peers) - 1));
        if (leader && merge && ((peers >> lo_lane) & 1u)) sum += carry_cnt;            // the run continues from the last iteration
        const unsigned leaders = __ballot_sync(0xffffffffu, leader);
        const int last_leader = __ffs(peers_hi) - 1;
        const unsigned emit = leaders & ~(1u << last_leader);                          // the last group stays in the carry
        const u32 base = r.n_docs + (flush ? 1u : 0u);
        if (flush && lane == 0) docs_out[r.n_docs] = ((u64)carry_doc << 32) | carry_cnt;
        if (leader && ((emit >> lane) & 1u)) docs_out[base + __popc(emit & lt)] = ((u64)e.doc << 32) | sum;
        r.n_docs = base + __popc(emit);
        carry_doc = __shfl_sync(0xffffffffu, e.doc, last_leader);
        carry_cnt = __shfl_sync(0xffffffffu, sum, last_leader);
        carry_valid = true;
    }
    if (carry_valid) {
        if (lane == 0) docs_out[r.n_docs] = ((u64)carry_doc << 32) | carry_cnt;
        r.n_docs++;
    }
    __syncwarp();
    return r;
}

// cur[i].count = min(cur[i].count, prev[doc].count) (0 if the doc is not in prev): and_min at warp scope
__device__ __forceinline__ void warp_and_min(u64 *cur, u32 n_cur, const u64 *prev, u32 n_prev) {
    for (u32 i = threadIdx.x & 31; i < n_cur; i += 32) {
        const u64 e = cur[i];
        const u64 doc = e >> 32;
        u32 lo = 0, hi = n_prev;
        while (lo < hi) {
            const u32 mid = (lo + hi) >> 1;
            if ((prev[mid] >> 32) < doc) lo = mid + 1; else hi = mid;
        }
        u32 c = 0;
        if (lo < n_prev && (prev[lo] >> 32) == doc) c = min((u32)(prev[lo] & 0xFFFFFFFFull), (u32)(e & 0xFFFFFFFFull));
        cur[i] = (doc << 32) | c;
    }
    __syncwarp();
}

struct WarpFin { u64 *docs; u32 n_docs; };

// The whole chain of one query on one warp's sub-range.  ptr[t] / n[t]: the warp's sub-slice of every term (shared or
// global memory).  buf: the warp's scratch, 6 buffers of `cap` entries.  Pair statistics and the continuation count
// go to the query's global stats (one atomic per step and warp, only when non-zero).
__device__ __forceinline__ WarpFin warp_phrase_chain(const PhraseQuery &pq, const u64 *const *ptr, const u32 *n, u64 *buf,
                                                     u64 cap, PhraseStats *stats) {
    const unsigned lane = threadIdx.x & 31;
    u64 *contA = buf, *contB = contA + cap, *docsA = contB + cap, *docsB = docsA + cap, *docsL = docsB + cap, *docsR = docsL + cap;
    const u32 n_terms = pq.n_terms;

    auto run_chain = [&](u32 ta, u32 tb, bool lr, u64 *final_docs) -> WarpFin {
        WarpFin res;
        res.docs = final_docs;
        res.n_docs = 0;
        const u64 *carry = lr ? ptr[ta] : ptr[tb - 1];
        u32 n_carry = lr ? n[ta] : n[tb - 1];
        u64 *cont_bufs[2] = {contA, contB};
        u64 *doc_bufs[2] = {docsA, docsB};
        int flip = 0;
        const u64 *prev_docs = nullptr;
        u32 n_prev = 0;
        const u32 n_steps = tb - ta - 1;
        for (u32 s = 0; s < n_steps; s++) {
            const u32 tnew = lr ? (ta + 1 + s) : (tb - 2 - s);     // also the step id
            const bool same = (pq.same_guess >> tnew) & 1u;
            const u64 *other = ptr[tnew];
            const u32 n_other = n[tnew];
            if (n_carry == 0 || n_other == 0) {                    // no pairs from here on in this sub-range
                res.n_docs = 0;
                break;
            }
            u64 *cont_out = cont_bufs[flip];
            u64 *docs_out = (s == n_steps - 1) ? final_docs : doc_bufs[flip];
            const bool drive_carry = (s > 0) || (n_carry <= n_other);
            WarpStepOut o;
            if (lr) {
                if (drive_carry) o = warp_bigram_step<true, true>(carry, n_carry, other, n_other, same, cont_out, docs_out);
                else o = warp_bigram_step<true, false>(other, n_other, carry, n_carry, same, cont_out, docs_out);
            } else {
                if (drive_carry) o = warp_bigram_step<false, false>(carry, n_carry, other, n_other, same, cont_out, docs_out);
                else o = warp_bigram_step<false, true>(other, n_other, carry, n_carry, same, cont_out, docs_out);
            }
            if (lane == 0) {
                if (o.st_inner) atomicAdd(&stats->n_inner[tnew], o.st_inner);
                if (o.st_diff) atomicAdd(&stats->n_diff[tnew], o.st_diff);
                if (o.n_cont) atomicAdd(&stats->n_cont, (unsigned long long)o.n_cont);
            }
            if (prev_docs) warp_and_min(docs_out, o.n_docs, prev_docs, n_prev);
            prev_docs = docs_out;
            n_prev = o.n_docs;
            carry = cont_out;
            n_carry = o.n_cont;
            res.docs = docs_out;
            res.n_docs = o.n_docs;
            flip ^= 1;
            if (o.n_docs == 0) break;                              // nothing can survive the remaining steps
        }
        return res;
    };

    WarpFin fin;
    if (pq.mode == SA_PHRASE_MODE_LR) {
        fin = run_chain(0, n_terms, true, docsL);
    } else if (pq.mode == SA_PHRASE_MODE_RL) {
        fin = run_chain(0, n_terms, false, docsL);
    } else {
        // both chains always run (their pair statistics feed the speculation check)
        WarpFin left = run_chain(0, pq.split, true, docsL);
        fin = run_chain(pq.split, n_terms, false, docsR);
        if (left.n_docs == 0) fin.n_docs = 0;
        warp_and_min(fin.docs, fin.n_docs, left.docs, left.n_docs);
    }
    return fin;
}
