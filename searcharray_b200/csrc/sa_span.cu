// sa_span.cu -- phrase matching with slop > 0 ("span search").
//
// Replaces (reference paths relative to softwaredoug/searcharray):
//   span_search / _intersect_all            searcharray/phrase/spans.py:71-187
//   _span_freqs, _compact_spans, _collect_spans, ActiveSpans   searcharray/roaringish/spans.pyx:70-319
//
// Phase 1 restates _intersect_all as a membership test.  With A = headers of term 0 and B_k = headers
// of term k (header = doc|block), the reference keeps, for every term, the words whose header lies in
//   H = L u R u (L - 1) u (R + 1)  where
//   L = AND_k [ (A(x)&B_k(x)) | (B_k(x)&A(x-1)) | (A(x)&B_k(x-1)) ]
//   R = AND_k [ (A(x)&B_k(x)) | (A(x)&B_k(x+1)) | (B_k(x)&A(x+1)) ]
// (the merges / intersects / adjacents of spans.py:79-112 reduce to these presence tests because
// they are applied with the header mask and set semantics).  Every x in H has each term within two
// blocks, so the candidates are enumerated, already sorted and unique, from the shortest list:
// word s (header hs) emits hs-2..hs+2, each only if no earlier word of that list covers it.
//   span_presence_kernel  one thread per generator word (grid = generator CTAs x queries): ONE
//                         search per term (narrowed by the term's tile directory) gives the presence
//                         of headers hs-3..hs+3; the five candidates are evaluated from those bits.
//                         Kept words are counted per (term, CTA) together with their doc-group starts.
//   span_scan_kernel      per query: exclusive scans over the generator CTAs (word offsets, group
//                         offsets; a group that continues across a CTA boundary is not a new start).
//   span_write_kernel     writes every term's sliced list and its doc-group starts, in order.
// Phase 2 (span_groups_kernel) replays _span_freqs.  The reference walks all terms "up to the next
// doc change" in lock step, i.e. iteration i consumes the i-th DOC GROUP of every term's sliced list
// (normally the same doc; the lists can be misaligned, and then this pairing is what defines the
// result).  Iterations are independent: one warp runs one iteration with the <= 512-entry span table
// in shared memory, lanes sharing the "extend every live span" loop, forks appended in order through
// ballots.  Counts are accumulated per `last_key` like the reference's Counter.
#include <algorithm>

#include "sa_phrase.cuh"
#include "sa_scan.cuh"
#include "sa_span.cuh"
#include "sa_term.cuh"

#define SPAN_CAP 512
#define SPAN_WARPS 4
#define GEN_THREADS 256

struct CtaRec {                          // per (query, term, generator CTA)
    u32 count;                           // kept words            -> after the scan: word offset
    u32 starts;                          // doc-group starts      -> after the scan: group offset
    u32 first_p1;                        // doc + 1 of the first kept word (0 = none) -> after the scan: 1 = first word continues a group
    u32 last_p1;                         // doc + 1 of the last kept word
};

struct SpanArgs {
    const u64 *words;
    const u32 *tile_dir;
    const SpanQuery *queries;
    SpanCounts *counts;
    u64 *word_arena;
    u32 *group_arena;
    u64 *rec;                            // p | mask7 << 32 | put5 << 39 | start5 << 44
    u32 *rec2;                           // local word offset | local start rank << 16
    CtaRec *cta;
    float *out;                          // [Q][out_stride]
    u64 out_stride;
    u64 n_docs, doc_base;
    // matches != NULL: phase 2 writes one record (local doc << 32 | count) per iteration instead of
    // adding into `out`; span_tiles_kernel then materialises the rows (BM25 + top-k collection)
    u64 *matches;
    const float *norm;
    TopkCtx topk;
    u32 topk_row0;
    u32 n_chunks;                        // doc-range chunks per query of span_tiles_kernel
    u64 docs_per_chunk;                  // a multiple of SA_TILE_DOCS
    u32 *cand_bits;                      // candidate-doc bitmaps (conjunction prefilter), one bit per local doc
    const u32 *conj;                     // indices of the queries that have one
};

// first index in [0, len) whose header is >= target
__device__ __forceinline__ u32 lb_hdr(const u64 *__restrict__ a, u64 len, const u32 *__restrict__ dir,
                                      u64 target, u64 doc_base) {
    u64 lo = 0, hi = len;
    if (dir) {
        const u64 doc = target >> SA_KEY_SHIFT;
        if (doc < doc_base) return 0;                       // below the shard: every word is >= target
        const u64 tile = (doc - doc_base) / SA_TILE_DOCS;
        lo = __ldg(dir + tile);
        hi = __ldg(dir + tile + 1);
    }
    while (lo < hi) {
        const u64 mid = (lo + hi) >> 1;
        if ((__ldg(a + mid) & SA_HDR_MASK) < target) lo = mid + 1; else hi = mid;
    }
    return (u32)lo;
}

// exclusive running maximum (0 = nothing before); `total` = maximum over the block
__device__ __forceinline__ u32 block_scan_excl_max(u32 v, u32 *warp_max, u32 &total) {
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u32 incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        u32 t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl = max(incl, t);
    }
    u32 excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = 0;
    __syncthreads();
    if (lane == 31) warp_max[warp] = incl;
    __syncthreads();
    u32 base = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < GEN_THREADS / 32; w++) {
        u32 s = warp_max[w];
        if (w < (int)warp) base = max(base, s);
        tot = max(tot, s);
    }
    total = tot;
    return max(base, excl);
}

// ---------------------------------------------------------------------------- phase 0 (balanced lists)
// A header can only become a candidate if every term has a word within one block of it -- in particular the doc
// holds EVERY term.  For balanced lists that conjunction is rare, and testing it per generator word by searching
// every list is what phase 1 spends its time on; so these queries first get a candidate-doc bitmap, built like the
// phrase conjunction regime does (sa_phrase.cu): one CTA per (query, 8192-doc tile) streams the tile's slice of
// every term once, sets bits in per-term presence bitmaps (shared-memory atomicOr) and ANDs them.  Phase 1 then
// skips every generator word whose doc is not a candidate (its five candidates cannot pass the presence test).
__global__ void __launch_bounds__(256)
span_cand_kernel(const SpanArgs a) {
    __shared__ u32 s_bm[SA_MAX_PHRASE_TERMS * (SA_TILE_DOCS / 32)];
    const SpanQuery &sq = a.queries[a.conj[blockIdx.x]];
    const u32 tile = blockIdx.y, n = sq.n_terms;
    const unsigned tid = threadIdx.x;
    const u64 td0 = a.doc_base + (u64)tile * SA_TILE_DOCS;
    for (u32 i = tid; i < n * (SA_TILE_DOCS / 32); i += 256) s_bm[i] = 0u;
    __syncthreads();
    for (u32 t = 0; t < n; t++) {
        const u32 *dir = a.tile_dir + sq.dir_off[t] + tile;
        const u32 lo = __ldg(dir), hi = __ldg(dir + 1);
        const u64 *__restrict__ lst = a.words + sq.off[t];
        u32 *bm = s_bm + t * (SA_TILE_DOCS / 32);
        u32 i = lo + tid;
        for (; i + 3 * 256 < hi; i += 4 * 256) {
            const u64 w0 = ld_stream_u64(lst + i), w1 = ld_stream_u64(lst + i + 256);
            const u64 w2 = ld_stream_u64(lst + i + 512), w3 = ld_stream_u64(lst + i + 768);
            const u32 r0 = (u32)((w0 >> SA_KEY_SHIFT) - td0), r1 = (u32)((w1 >> SA_KEY_SHIFT) - td0);
            const u32 r2 = (u32)((w2 >> SA_KEY_SHIFT) - td0), r3 = (u32)((w3 >> SA_KEY_SHIFT) - td0);
            atomicOr(&bm[r0 >> 5], 1u << (r0 & 31u));
            atomicOr(&bm[r1 >> 5], 1u << (r1 & 31u));
            atomicOr(&bm[r2 >> 5], 1u << (r2 & 31u));
            atomicOr(&bm[r3 >> 5], 1u << (r3 & 31u));
        }
        for (; i < hi; i += 256) {
            const u32 rel = (u32)((ld_stream_u64(lst + i) >> SA_KEY_SHIFT) - td0);
            atomicOr(&bm[rel >> 5], 1u << (rel & 31u));
        }
    }
    __syncthreads();
    u32 c = s_bm[tid];
    for (u32 t = 1; t < n; t++) c &= s_bm[t * (SA_TILE_DOCS / 32) + tid];
    a.cand_bits[sq.cand_off + (u64)tile * (SA_TILE_DOCS / 32) + tid] = c;
}

// ---------------------------------------------------------------------------- phase 1
__global__ void __launch_bounds__(GEN_THREADS)
span_presence_kernel(const SpanArgs a) {
    __shared__ u32 s_warp[GEN_THREADS / 32];
    __shared__ u32 s_first;
    const u32 q = blockIdx.y;
    const SpanQuery &sq = a.queries[q];
    if (sq.literal || blockIdx.x >= sq.n_ctas) return;                 // CTA-uniform
    const u32 n = sq.n_terms;
    const unsigned tid = threadIdx.x;
    const u64 *__restrict__ S = a.words + sq.off[sq.shortest];
    const u64 nS = sq.len[sq.shortest];
    const u64 si = (u64)blockIdx.x * GEN_THREADS + tid;
    const bool active = si < nS;
    u64 hs = 0, hp = 0;
    if (active) {
        hs = __ldg(S + si) & SA_HDR_MASK;
        if (si > 0) hp = __ldg(S + si - 1) & SA_HDR_MASK;
    }
    u64 *__restrict__ rec = a.rec + sq.rec_off + si * n;
    u32 *__restrict__ rec2 = a.rec2 + sq.rec_off + si * n;

    // A. presence of every term at hs-3 .. hs+3 (bit o <-> header hs + (o-3) blocks)
    u64 mm[2] = {0, 0};                                                 // 8 bits per term
    bool doc_ok = active;
    if (active && sq.cand_off != SA_NO_DIR) {                           // conjunction prefilter (phase 0)
        const u64 d = (hs >> SA_KEY_SHIFT) - a.doc_base;
        doc_ok = (__ldg(a.cand_bits + sq.cand_off + (d >> 5)) >> (d & 31u)) & 1u;
        if (!doc_ok)
            for (u32 t = 0; t < n; t++) rec[t] = 0;                     // nothing of this word is kept
    }
    if (doc_ok) {
        const u64 target = hs >= 3 * SA_ONE_BLOCK ? hs - 3 * SA_ONE_BLOCK : 0;
        const u64 top = hs + 3 * SA_ONE_BLOCK;
        for (u32 t = 0; t < n; t++) {
            const u64 *__restrict__ lst = a.words + sq.off[t];
            const u64 len = sq.len[t];
            const u32 *dir = (sq.dir_off[t] != SA_NO_DIR && a.tile_dir) ? a.tile_dir + sq.dir_off[t] : nullptr;
            const u32 p = lb_hdr(lst, len, dir, target, a.doc_base);
            u32 m7 = 0;
            for (u32 r = 0; r < 7 && (u64)p + r < len; r++) {
                const u64 h = __ldg(lst + p + r) & SA_HDR_MASK;
                if (h > top) break;
                const int o = (int)((i64)(h - hs) >> SA_LSB_BITS) + 3;   // headers are multiples of one block
                m7 |= 1u << o;
            }
            rec[t] = (u64)p | ((u64)m7 << 32);
            if (t < 8) mm[0] |= (u64)m7 << (8 * t); else mm[1] |= (u64)m7 << (8 * (t - 8));
        }
    }
    auto m7_of = [&](u32 t) -> u32 { return (u32)(((t < 8) ? (mm[0] >> (8 * t)) : (mm[1] >> (8 * (t - 8)))) & 0x7Fu); };

    // B. the five candidates x = hs + d blocks, d = -2..2 (bit d+2 of keep5)
    u32 keep5 = 0;
    if (active) {
        for (int d = -2; d <= 2; d++) {
            if (d < 0 && hs < (u64)(-d) * SA_ONE_BLOCK) continue;
            const u64 x = hs + (u64)((i64)d * (i64)SA_ONE_BLOCK);
            // emitted by the FIRST generator word within two blocks of x
            if (si > 0 && hp + 2 * SA_ONE_BLOCK >= x) continue;
            // presence at x-1, x, x+1 = bits d+2, d+3, d+4
            const u32 pa = (m7_of(0) >> (d + 2)) & 7u;
            auto A = [&](int o) { return (pa >> (o + 1)) & 1u; };       // o in {-1,0,1}
            u32 Lx = 1, Rx = 1, Lx1 = 1, Rxm1 = 1;
            for (u32 k = 1; k < n; k++) {
                const u32 pb = (m7_of(k) >> (d + 2)) & 7u;
                auto Bk = [&](int o) { return (pb >> (o + 1)) & 1u; };
                Lx &= (A(0) & Bk(0)) | (Bk(0) & A(-1)) | (A(0) & Bk(-1));
                Rx &= (A(0) & Bk(0)) | (A(0) & Bk(1)) | (Bk(0) & A(1));
                Lx1 &= (A(1) & Bk(1)) | (Bk(1) & A(0)) | (A(1) & Bk(0));          // L(x+1)
                Rxm1 &= (A(-1) & Bk(-1)) | (A(-1) & Bk(0)) | (Bk(-1) & A(0));      // R(x-1)
            }
            if (Lx | Rx | Lx1 | Rxm1) keep5 |= 1u << (d + 2);
        }
    }

    // C. per term: which candidates hold a word of the term, where its doc groups start, and this
    //    thread's offsets inside the CTA
    for (u32 t = 0; t < n; t++) {                                       // CTA-uniform
        const u32 put5 = active ? (keep5 & (m7_of(t) >> 1) & 0x1Fu) : 0u;
        const u32 cnt = __popc(put5);
        u32 first_p1 = 0, last_p1 = 0;
        if (cnt) {
            const int d_lo = __ffs(put5) - 3, d_hi = (31 - __clz(put5)) - 2;
            first_p1 = (u32)((hs + (u64)((i64)d_lo * (i64)SA_ONE_BLOCK)) >> SA_KEY_SHIFT) + 1;
            last_p1 = (u32)((hs + (u64)((i64)d_hi * (i64)SA_ONE_BLOCK)) >> SA_KEY_SHIFT) + 1;
        }
        u32 cta_last;
        u32 prev_p1 = block_scan_excl_max(last_p1, s_warp, cta_last);   // docs ascend: max = most recent
        u32 start5 = 0;
        for (int d = -2; d <= 2; d++) {
            if (!((put5 >> (d + 2)) & 1u)) continue;
            const u32 doc_p1 = (u32)((hs + (u64)((i64)d * (i64)SA_ONE_BLOCK)) >> SA_KEY_SHIFT) + 1;
            if (doc_p1 != prev_p1) start5 |= 1u << (d + 2);
            prev_p1 = doc_p1;
        }
        u32 total;
        const u32 off = block_exclusive_sum<GEN_THREADS>(cnt | ((u32)__popc(start5) << 16), s_warp, total);
        if (tid == 0) s_first = 0;
        __syncthreads();
        if (cnt && (off & 0xFFFFu) == 0) s_first = first_p1;            // the CTA's first kept word
        if (active) {
            rec[t] |= ((u64)put5 << 39) | ((u64)start5 << 44);
            rec2[t] = off;
        }
        __syncthreads();
        if (tid == 0) {
            CtaRec r;
            r.count = total & 0xFFFFu;
            r.starts = total >> 16;
            r.first_p1 = s_first;
            r.last_p1 = cta_last;
            a.cta[sq.cta_off + (u64)t * sq.n_ctas + blockIdx.x] = r;
        }
        __syncthreads();
    }
}

// exclusive scans over the generator CTAs of every term of one query
__global__ void __launch_bounds__(GEN_THREADS)
span_scan_kernel(const SpanArgs a) {
    __shared__ u32 s_warp[GEN_THREADS / 32];
    const u32 q = blockIdx.x;
    const SpanQuery &sq = a.queries[q];
    if (sq.literal) return;
    const unsigned tid = threadIdx.x;
    for (u32 t = 0; t < sq.n_terms; t++) {
        CtaRec *__restrict__ recs = a.cta + sq.cta_off + (u64)t * sq.n_ctas;
        u32 carry_w = 0, carry_g = 0, carry_last = 0;
        for (u32 base = 0; base < sq.n_ctas; base += GEN_THREADS) {
            const u32 c = base + tid;
            CtaRec r = {0, 0, 0, 0};
            if (c < sq.n_ctas) r = recs[c];
            u32 blk_last, tot_w, tot_g;
            const u32 prev_last = max(block_scan_excl_max(r.last_p1, s_warp, blk_last), carry_last);
            const u32 adj = (r.count && r.first_p1 == prev_last) ? 1u : 0u;
            const u32 w_off = block_exclusive_sum<GEN_THREADS>(r.count, s_warp, tot_w) + carry_w;
            const u32 g_off = block_exclusive_sum<GEN_THREADS>(r.starts - adj, s_warp, tot_g) + carry_g;
            if (c < sq.n_ctas) {
                r.count = w_off; r.starts = g_off; r.first_p1 = adj;
                recs[c] = r;
            }
            carry_w += tot_w;
            carry_g += tot_g;
            carry_last = max(carry_last, blk_last);
            __syncthreads();
        }
        if (tid == 0) {
            if (carry_w > sq.s_cap[t]) a.counts[q].overflow = 1;
            a.counts[q].n_sliced[t] = carry_w;
            a.counts[q].n_groups[t] = carry_g;
            a.group_arena[sq.g_off[t] + carry_g] = carry_w;              // sentinel: end of the last group
        }
    }
}

__global__ void __launch_bounds__(GEN_THREADS)
span_write_kernel(const SpanArgs a) {
    const u32 q = blockIdx.y;
    const SpanQuery &sq = a.queries[q];
    if (sq.literal || blockIdx.x >= sq.n_ctas || a.counts[q].overflow) return;
    const u32 n = sq.n_terms;
    const u64 si = (u64)blockIdx.x * GEN_THREADS + threadIdx.x;
    if (si >= sq.len[sq.shortest]) return;
    const u64 *__restrict__ rec = a.rec + sq.rec_off + si * n;
    const u32 *__restrict__ rec2 = a.rec2 + sq.rec_off + si * n;
    for (u32 t = 0; t < n; t++) {
        const u64 r = rec[t];
        const u32 put5 = (u32)(r >> 39) & 0x1Fu;
        if (!put5) continue;
        const u32 start5 = (u32)(r >> 44) & 0x1Fu, m7 = (u32)(r >> 32) & 0x7Fu, p = (u32)r;
        const u32 r2 = rec2[t];
        const CtaRec c = a.cta[sq.cta_off + (u64)t * sq.n_ctas + blockIdx.x];
        u32 pos = c.count + (r2 & 0xFFFFu);
        u32 rank = r2 >> 16;
        const u64 *__restrict__ lst = a.words + sq.off[t];
        u64 *__restrict__ sl = a.word_arena + sq.s_off[t];
        u32 *__restrict__ gs = a.group_arena + sq.g_off[t];
        for (int b = 0; b < 5; b++) {
            if (!((put5 >> b) & 1u)) continue;
            const u32 widx = p + __popc(m7 & ((1u << (b + 1)) - 1u));   // header hs + (b-2) blocks <-> bit b+1
            sl[pos] = __ldg(lst + widx);
            if ((start5 >> b) & 1u) {
                // the CTA's first kept word continues the previous CTA's doc group when c.first_p1 == 1
                if (!(rank == 0 && c.first_p1)) gs[c.starts + rank - c.first_p1] = pos;
                rank++;
            }
            pos++;
        }
    }
}

// doc groups of every sliced list, single CTA (used after the literal candidate kernel)
__global__ void __launch_bounds__(GEN_THREADS)
span_groups_build_kernel(const SpanArgs a, u32 q) {
    __shared__ u32 s_warp[GEN_THREADS / 32];
    __shared__ u32 s_groups;
    const SpanQuery &sq = a.queries[q];
    const unsigned tid = threadIdx.x;
    for (u32 t = 0; t < sq.n_terms; t++) {
        const u32 cnt = a.counts[q].n_sliced[t];
        const u64 *sl = a.word_arena + sq.s_off[t];
        if (tid == 0) s_groups = 0;
        __syncthreads();
        for (u32 base = 0; base < cnt; base += GEN_THREADS) {
            const u32 i = base + tid;
            bool start = false;
            if (i < cnt) start = (i == 0) || ((sl[i] >> SA_KEY_SHIFT) != (sl[i - 1] >> SA_KEY_SHIFT));
            u32 total;
            u32 off = block_exclusive_sum<GEN_THREADS>(start ? 1u : 0u, s_warp, total);
            const u32 g0 = s_groups;
            if (start) a.group_arena[sq.g_off[t] + g0 + off] = i;
            __syncthreads();
            if (tid == 0) s_groups = g0 + total;
            __syncthreads();
        }
        if (tid == 0) {
            a.group_arena[sq.g_off[t] + s_groups] = cnt;          // sentinel: end of the last group
            a.counts[q].n_groups[t] = s_groups;
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------- phase 1, literal (rare) variant
// When every term has a word at header 0 (doc 0, block 0) the reference's `last_lhs_headers - 1
// block` (spans.py:104) underflows on its first element; the merges and the galloping slice that
// follow then run on a list that is no longer sorted, and WHICH candidate words survive depends on
// the exact pointer walk.  That is deterministic, so it is replayed literally -- one thread, the
// reference's own sequence of galloping intersects / adjacents / merges (the restatement follows
// searcharray/roaringish/intersect.pyx:32-190 and merge.pyx:54-134).  Only this corner takes it.
struct U64Buf { u64 *p; u64 n; };

#define DEV_GALLOP(ptr, end, cond)                    \
    do {                                              \
        u64 stride_ = 1;                              \
        while ((ptr) < (end) && (cond)) {             \
            (ptr) += stride_;                         \
            stride_ <<= 1;                            \
        }                                             \
        (ptr) -= (stride_ >> 1);                      \
    } while (0)

__device__ u64 dev_intersect_drop(const u64 *lhs, u64 nl, const u64 *rhs, u64 nr, u64 mask, u64 *li, u64 *ri) {
    const u64 *l = lhs, *r = rhs, *le = lhs + nl, *re = rhs + nr;
    u64 m = 0, last = ~0ull;
    while (l < le && r < re) {
        DEV_GALLOP(l, le, (*l & mask) < (*r & mask));
        DEV_GALLOP(r, re, (*r & mask) < (*l & mask));
        const u64 x = *l & mask, y = *r & mask;
        if (x < y) l++;
        else if (y < x) r++;
        else {
            if ((last & mask) != x) { li[m] = (u64)(l - lhs); if (ri) ri[m] = (u64)(r - rhs); last = *l; m++; }
            l++; r++;
        }
    }
    return m;
}

__device__ u64 dev_adjacent(const u64 *lhs, u64 nl, const u64 *rhs, u64 nr, u64 mask, u64 *li, u64 *ri) {
    const u64 delta = mask & (~mask + 1);
    const u64 *l = lhs, *r = rhs, *le = lhs + nl, *re = rhs + nr;
    u64 m = 0, last = ~0ull;
    while (r < re && (*r & mask) == 0) r++;
    while (l < le && r < re) {
        DEV_GALLOP(l, le, (*l & mask) < ((*r & mask) - delta));
        DEV_GALLOP(r, re, ((*r & mask) - delta) < (*l & mask));
        const u64 x = *l & mask, y = (*r & mask) - delta;
        if (x < y) l++;
        else if (y < x) r++;
        else {
            if ((last & mask) != x) { li[m] = (u64)(l - lhs); ri[m] = (u64)(r - rhs); last = *l; m++; }
            l++; r++;
        }
    }
    return m;
}

__device__ u64 dev_merge(const u64 *lhs, u64 nl, const u64 *rhs, u64 nr, bool drop, u64 *out) {
    u64 i = 0, j = 0, m = 0;
    while (i < nl && j < nr) {
        if (lhs[i] < rhs[j]) out[m++] = lhs[i++];
        else if (rhs[j] < lhs[i]) out[m++] = rhs[j++];
        else { out[m++] = lhs[i]; if (!drop) out[m++] = rhs[j]; i++; j++; }
    }
    while (j < nr) out[m++] = rhs[j++];
    while (i < nl) out[m++] = lhs[i++];
    return m;
}

// all rhs elements whose value occurs in lhs, found the way _gallop_intersect_keep walks
__device__ u64 dev_intersect_keep_rhs(const u64 *lhs, u64 nl, const u64 *rhs, u64 nr, u64 hdr_mask_rhs, u64 *r_out) {
    // lhs: header values (possibly unsorted here!), rhs: words compared by (word & hdr_mask_rhs)
    const u64 *l = lhs, *r = rhs, *le = lhs + nl, *re = rhs + nr;
    u64 m = 0;
    while (l < le && r < re) {
        DEV_GALLOP(l, le, *l < (*r & hdr_mask_rhs));
        DEV_GALLOP(r, re, (*r & hdr_mask_rhs) < *l);
        const u64 x = *l, y = *r & hdr_mask_rhs;
        if (x < y) l++;
        else if (y < x) r++;
        else {
            while (l < le && *l == x) l++;
            while (r < re && (*r & hdr_mask_rhs) == x) { r_out[m++] = *r; r++; }
        }
    }
    return m;
}

__global__ void span_candidates_literal_kernel(const SpanArgs a, u32 q, u64 *scratch, u64 cap3 /* 3*|A| + 8 */) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const SpanQuery &sq = a.queries[q];
    const u32 n = sq.n_terms;
    const u64 M = SA_HDR_MASK;
    u64 *lh = scratch, *rh = lh + cap3, *tmp = rh + cap3, *tmp2 = tmp + cap3;
    u64 *last_l = tmp2 + cap3, *last_r = last_l + cap3;
    u64 *i0 = last_r + cap3, *i1 = i0 + cap3, *allh = i1 + cap3, *allh2 = allh + 4 * cap3;
    u64 n_ll = 0, n_lr = 0;
    const u64 *curr = a.words + sq.off[0];
    const u64 nc = sq.len[0];
    for (u32 k = 1; k < n; k++) {
        const u64 *nxt = a.words + sq.off[k];
        const u64 nn = sq.len[k];
        u64 m = dev_intersect_drop(curr, nc, nxt, nn, M, i0, nullptr);
        for (u64 j = 0; j < m; j++) tmp[j] = curr[i0[j]] & M;                     // int_headers
        u64 ma = dev_adjacent(curr, nc, nxt, nn, M, i0, i1);                      // curr_to_right, next_to_left
        for (u64 j = 0; j < ma; j++) tmp2[j] = nxt[i1[j]];
        u64 n_lh = dev_merge(tmp, m, tmp2, ma, false, lh);
        for (u64 j = 0; j < ma; j++) tmp2[j] = curr[i0[j]];
        u64 n_rh = dev_merge(tmp, m, tmp2, ma, false, rh);
        u64 mb = dev_adjacent(nxt, nn, curr, nc, M, i0, i1);                      // next_to_right, curr_to_left
        for (u64 j = 0; j < mb; j++) tmp2[j] = curr[i1[j]];
        n_lh = dev_merge(lh, n_lh, tmp2, mb, false, tmp);
        for (u64 j = 0; j < n_lh; j++) lh[j] = tmp[j];
        for (u64 j = 0; j < mb; j++) tmp2[j] = nxt[i0[j]];
        n_rh = dev_merge(rh, n_rh, tmp2, mb, false, tmp);
        for (u64 j = 0; j < n_rh; j++) rh[j] = tmp[j];
        if (k > 1) {
            u64 ml = dev_intersect_drop(last_l, n_ll, lh, n_lh, M, i0, nullptr);
            for (u64 j = 0; j < ml; j++) last_l[j] = last_l[i0[j]];              // ascending: in place is safe
            n_ll = ml;
            u64 mr = dev_intersect_drop(last_r, n_lr, rh, n_rh, M, i0, nullptr);
            for (u64 j = 0; j < mr; j++) last_r[j] = last_r[i0[j]];
            n_lr = mr;
        } else {
            for (u64 j = 0; j < n_lh; j++) last_l[j] = lh[j];
            for (u64 j = 0; j < n_rh; j++) last_r[j] = rh[j];
            n_ll = n_lh;
            n_lr = n_rh;
        }
    }
    for (u64 j = 0; j < n_lr; j++) tmp[j] = last_r[j] + SA_ONE_BLOCK;             // to_rhs
    for (u64 j = 0; j < n_ll; j++) tmp2[j] = last_l[j] - SA_ONE_BLOCK;            // to_lhs (may underflow)
    u64 na = dev_merge(tmp, n_lr, tmp2, n_ll, true, allh);
    na = dev_merge(last_l, n_ll, allh, na, true, allh2);
    na = dev_merge(last_r, n_lr, allh2, na, true, allh);
    for (u64 j = 0; j < na; j++) allh[j] &= M;
    for (u32 t = 0; t < n; t++) {
        u64 m = dev_intersect_keep_rhs(allh, na, a.words + sq.off[t], sq.len[t], M, a.word_arena + sq.s_off[t]);
        a.counts[q].n_sliced[t] = (u32)m;
    }
}

// ---------------------------------------------------------------------------- phase 2
struct WarpSpans {                        // one per warp, in dynamic shared memory
    u64 posns[SPAN_CAP];
    u32 terms[SPAN_CAP];
    int beg[SPAN_CAP];
    int end[SPAN_CAP];
    int cbeg[SPAN_CAP];                   // collected spans (_collect_spans)
    int cend[SPAN_CAP];
};

__device__ __forceinline__ int iabs(int v) { return v < 0 ? -v : v; }

// _compact_spans (spans.pyx:141-154): keep width <= max_w and >= 1 term, order preserved
__device__ u32 compact_spans(WarpSpans &S, u32 cursor, int max_w) {
    const unsigned lane = threadIdx.x & 31;
    u32 w = 0;
    for (u32 base = 0; base < cursor; base += 32) {
        const u32 s = base + lane;
        bool keep = false;
        u64 po = 0; u32 te = 0; int be = 0, en = 0;
        if (s < cursor) {
            po = S.posns[s]; te = S.terms[s]; be = S.beg[s]; en = S.end[s];
            keep = (iabs(en - be) <= max_w) && (__popc(te) > 0);
        }
        unsigned m = __ballot_sync(0xffffffffu, keep);
        __syncwarp();
        if (keep) {
            const u32 d = w + __popc(m & ((1u << lane) - 1));
            S.posns[d] = po; S.terms[d] = te; S.beg[d] = be; S.end[d] = en;
        }
        w += __popc(m);
        __syncwarp();
    }
    return w;
}

// _collect_spans (spans.pyx:157-186): complete, narrow-enough spans after first-come overlap
// replacement; returns how many were collected
__device__ u32 collect_spans(WarpSpans &S, u32 cursor, u32 n_terms, int max_w) {
    const unsigned lane = threadIdx.x & 31;
    u32 ncoll = 0;
    for (u32 s = 0; s < cursor; s++) {
        const u32 te = S.terms[s];
        const u64 po = S.posns[s];
        const int be = S.beg[s], en = S.end[s];
        const bool complete = ((u32)__popc(te) == n_terms) || ((u32)__popcll(po) == n_terms);
        const int nw = iabs(en - be);
        if (!(complete && nw < max_w)) continue;            // warp-uniform
        bool replaced = false;
        for (u32 base = 0; base < ncoll && !replaced; base += 32) {
            const u32 c = base + lane;
            bool hit = false;
            if (c < ncoll) {
                const int cb = S.cbeg[c], ce = S.cend[c];
                hit = (be <= ce && en >= cb) && (nw < iabs(ce - cb));
            }
            unsigned m = __ballot_sync(0xffffffffu, hit);
            if (m) {
                const u32 first = base + (u32)(__ffs(m) - 1);
                if (lane == 0) { S.cbeg[first] = be; S.cend[first] = en; }
                replaced = true;
            }
            __syncwarp();
        }
        if (!replaced) {
            if (lane == 0 && ncoll < SPAN_CAP) { S.cbeg[ncoll] = be; S.cend[ncoll] = en; }
            ncoll++;
            __syncwarp();
        }
    }
    return ncoll;
}

__global__ void __launch_bounds__(SPAN_WARPS * 32)
span_groups_kernel(const SpanArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const unsigned warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    WarpSpans &S = reinterpret_cast<WarpSpans *>(smem_raw)[warp];
    const u32 warps_total = gridDim.x * SPAN_WARPS;
    const u32 warp_global = blockIdx.x * SPAN_WARPS + warp;

    {
        const u32 q = blockIdx.y;
        const SpanQuery &sq = a.queries[q];
        const SpanCounts &sc = a.counts[q];
        const u32 n = sq.n_terms;
        const int max_w = (int)(n + sq.slop);
        const u32 iters = sc.n_groups[0];                    // while curr_idx[0] < lengths[1]
        for (u32 it = warp_global; it < iters; it += warps_total) {
            u32 cursor = 0;
            bool full = false;
            u32 last_key = 0;
            u32 mn_pop = 0;                                    // running "min" with the reference's rule
            bool undefined = false;
            for (u32 t = 0; t < n; t++) {
                u32 sum_pop = 0;
                if (it < sc.n_groups[t]) {
                    const u64 *sl = a.word_arena + sq.s_off[t];
                    const u32 *gs = a.group_arena + sq.g_off[t];
                    const u32 w0 = gs[it], w1 = gs[it + 1];
                    const bool has_next_group = (it + 1 < sc.n_groups[t]);
                    const u32 term_bit = 1u << t;
                    bool give_up = false;
                    for (u32 wi = w0; wi < w1 && !give_up; wi++) {
                        const u64 word = sl[wi];
                        last_key = (u32)(word >> SA_KEY_SHIFT);
                        const int payload_base = (int)((word >> SA_LSB_BITS) & 0x3FFFFu) * SA_LSB_BITS;
                        u32 bits = (u32)(word & SA_LSB_MASK);
                        sum_pop += __popc(bits);
                        while (bits) {
                            const int set_idx = __ffs(bits) - 1;
                            bits &= bits - 1;
                            const int posn = set_idx + payload_base;
                            // spans.pyx:107-108 compiled as a 32-bit shift, sign-extended (see oracle)
                            const u64 posn_bit = (u64)(i64)(int)(1u << ((posn % 64) & 31));
                            const u32 fresh = cursor;
                            if (fresh >= SPAN_CAP) {           // reference: out-of-bounds write (undefined)
                                full = true;
                                undefined = true;
                                break;
                            }
                            if (lane == 0) { S.terms[fresh] = term_bit; S.posns[fresh] = posn_bit; S.beg[fresh] = posn; S.end[fresh] = posn; }
                            cursor++;
                            __syncwarp();
                            bool any_fail = false, any_ok = false;
                            for (u32 base = 0; base < fresh; base += 32) {
                                const u32 s = base + lane;
                                bool want_fork = false;
                                u32 te = 0; u64 po = 0; int be = 0, en = 0;
                                if (s < fresh) {
                                    te = S.terms[s]; po = S.posns[s];
                                    const u32 nt_before = __popc(te), np_before = __popcll(po);
                                    if (!(nt_before < n && np_before == n) && !(te & term_bit)) {
                                        const u64 po_new = po | posn_bit;
                                        S.posns[s] = po_new;                       // kept even when cancelled
                                        be = S.beg[s]; en = S.end[s];
                                        const bool cancel = ((u32)__popcll(po_new) == np_before) || (iabs(posn - be) > max_w);
                                        if (!cancel) {
                                            want_fork = true;
                                            te |= term_bit;
                                            S.terms[s] = te;
                                            po = po_new;
                                        }
                                    }
                                }
                                unsigned m = __ballot_sync(0xffffffffu, want_fork);
                                if (want_fork) {
                                    const u32 slot = cursor + __popc(m & ((1u << lane) - 1));
                                    if (slot < SPAN_CAP) {
                                        S.terms[slot] = te; S.posns[slot] = po & ~posn_bit; S.beg[slot] = be; S.end[slot] = en;
                                    }
                                    S.end[s] = posn;
                                }
                                const u32 nf = __popc(m);
                                if (nf) {
                                    if (cursor + nf > SPAN_CAP) any_fail = true;
                                    if (cursor < SPAN_CAP) any_ok = true;
                                    cursor = min(cursor + nf, (u32)SPAN_CAP);
                                }
                                __syncwarp();
                            }
                            if (any_fail) full = true; else if (any_ok) full = false;
                            if (cursor >= SPAN_CAP) break;
                        }
                        if (cursor >= SPAN_CAP) {
                            cursor = compact_spans(S, cursor, max_w);
                            if (cursor >= SPAN_CAP && has_next_group) give_up = true;   // skip to the next doc group
                        }
                    }
                }
                if (mn_pop == 0 || sum_pop < mn_pop) mn_pop = sum_pop;
            }
            u32 add;
            if (full) add = mn_pop;
            else add = collect_spans(S, cursor, n, max_w);
            if (lane == 0) {
                const u64 d = (u64)last_key - a.doc_base;
                if (a.matches) a.matches[sq.m_off + it] = d < a.n_docs ? ((d << 32) | add) : ~0ull;
                else if (d < a.n_docs) atomicAdd(a.out + (u64)q * a.out_stride + d, (float)add);
                if (undefined) atomicAdd(&a.counts[q].undefined, 1u);
            }
            __syncwarp();
        }
    }
}


// ---------------------------------------------------------------------------- phase 3 (batched path)
// are the match records of every query in doc order?  (they are whenever the terms' doc groups pair up)
// Record i carries the doc of doc group i of the last term that has one.  Outside the literal corner every term's
// sliced list holds words in the same docs (a candidate header has every term within one block, and positions stay
// below 2^18, so one block more or less never reaches another doc), so group i is one doc for every term and the records
// ascend; a record is ~0 only for a doc outside the shard, which the shard's own lists cannot hold.  Only the literal
// corner's replayed lists can pair groups of different docs, and no literal input found so far does: the unsorted
// loop of span_tiles_kernel is a guard that no known index reaches, and no test covers it.
__global__ void __launch_bounds__(GEN_THREADS)
span_sorted_kernel(const SpanArgs a) {
    const u32 q = blockIdx.y;
    const SpanQuery &sq = a.queries[q];
    const u32 iters = a.counts[q].n_groups[0];
    const u64 *__restrict__ m = a.matches + sq.m_off;
    bool bad = false;
    for (u32 i = blockIdx.x * GEN_THREADS + threadIdx.x + 1; i < iters; i += gridDim.x * GEN_THREADS)
        if ((m[i] >> 32) < (m[i - 1] >> 32) || m[i] == ~0ull || m[i - 1] == ~0ull) bad = true;
    if (iters && threadIdx.x == 0 && blockIdx.x == 0 && m[0] == ~0ull) bad = true;
    if (__syncthreads_or(bad) && threadIdx.x == 0) a.counts[q].unsorted = 1;
}

// One CTA per (doc-range chunk, query): writes the chunk's dense tiles -- zeros, plus the BM25 of the
// accumulated span counts where there are matches -- and collects every tile's top-k candidates.
// DEEP: k > SA_TOPK_MAX, collected by deep_tile_collect.
template <bool DEEP>
__global__ void __launch_bounds__(SA_TERM_THREADS)
span_tiles_kernel(const SpanArgs a) {
    __shared__ __align__(16) float s_tile[SA_TILE_DOCS];
    __shared__ u32 s_top[(SA_TERM_THREADS / 32) * 8];
    __shared__ u32 s_ncand, s_tile_max;
    const u32 q = blockIdx.x;            // grid = (queries, chunks)
    const u32 chunk = blockIdx.y;
    const SpanQuery &sq = a.queries[q];
    const unsigned tid = threadIdx.x;
    const u32 iters = a.counts[q].n_groups[0];
    const bool sorted = a.counts[q].unsorted == 0;
    const u64 *__restrict__ m = a.matches + sq.m_off;
    const u32 row = a.topk_row0 + q;
    float *out = a.out + (u64)row * a.out_stride;
    const u32 n_tiles = (u32)((a.n_docs + SA_TILE_DOCS - 1) / SA_TILE_DOCS);
    const u32 tile0 = (u32)(((u64)chunk * a.docs_per_chunk) / SA_TILE_DOCS);
    const u32 tile1 = min(n_tiles, (u32)((((u64)chunk + 1) * a.docs_per_chunk) / SA_TILE_DOCS));
    // sorted records: cursor at the first record of this chunk (uniform bisect)
    u64 cur = 0;
    if (sorted) {
        const u64 key = (u64)tile0 * SA_TILE_DOCS;
        u64 lo = 0, hi = iters;
        while (lo < hi) {
            const u64 mid = (lo + hi) >> 1;
            if ((m[mid] >> 32) < key) lo = mid + 1; else hi = mid;
        }
        cur = lo;
    }
    u64 next_doc = (sorted && cur < iters) ? (m[cur] >> 32) : ~0ull;
    for (u32 tile = tile0; tile < tile1; tile++) {
        const u64 t0 = (u64)tile * SA_TILE_DOCS, t1 = t0 + SA_TILE_DOCS;
        if (sorted && next_doc >= t1) {                                   // no match in this tile
            store_empty_tile<SA_TERM_THREADS>(out + t0, a.topk, row, tile);
            continue;
        }
#pragma unroll
        for (int i = 0; i < SA_TILE_DOCS / SA_TERM_THREADS / 4; i++)
            reinterpret_cast<float4 *>(s_tile)[tid + i * SA_TERM_THREADS] = make_float4(0.f, 0.f, 0.f, 0.f);
        __syncthreads();
        u32 n_items = 0;
        if (sorted) {
            u64 end = cur;                                                 // records of this tile: [cur, end)
            {
                u64 lo = cur + 1, hi = iters, st = 1;
                while (lo < hi) {
                    const u64 probe = min(lo + st - 1, hi - 1);
                    if ((m[probe] >> 32) < t1) { lo = probe + 1; st <<= 1; }
                    else { hi = probe; break; }
                }
                while (lo < hi) {
                    const u64 mid = (lo + hi) >> 1;
                    if ((m[mid] >> 32) < t1) lo = mid + 1; else hi = mid;
                }
                end = lo;
            }
            for (u64 i = cur + tid; i < end; i += SA_TERM_THREADS) {
                const u64 e = m[i];
                const u32 c = (u32)e;
                if (c) atomicAdd(&s_tile[(e >> 32) - t0], (float)c);       // equal docs may repeat: counts add up
            }
            n_items = (u32)(end - cur);
            cur = end;
            next_doc = cur < iters ? (m[cur] >> 32) : ~0ull;
        } else {
            for (u32 i = tid; i < iters; i += SA_TERM_THREADS) {
                const u64 e = m[i];
                if (e == ~0ull) continue;
                const u64 d = e >> 32;
                if (d >= t0 && d < t1 && (u32)e) atomicAdd(&s_tile[d - t0], (float)(u32)e);
            }
            n_items = SA_TILE_DOCS;                                        // unknown: always derive a bound
        }
        __syncthreads();
        // counts -> BM25 in place (bm25.pyx:20-25 with the precomputed length norm); each thread owns
        // the elements it will flush
        u32 my_max = 0;
#pragma unroll
        for (int i = 0; i < SA_TILE_DOCS / SA_TERM_THREADS / 4; i++) {
            const unsigned g = tid + i * SA_TERM_THREADS;
            float4 v = reinterpret_cast<float4 *>(s_tile)[g];
            if ((v.x != 0.0f) | (v.y != 0.0f) | (v.z != 0.0f) | (v.w != 0.0f)) {
                float vs[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    if (vs[e] != 0.0f) {
                        const float nrm = __ldg(a.norm + t0 + g * 4 + e);
                        vs[e] = __fmul_rn(__fdiv_rn(vs[e], __fadd_rn(vs[e], nrm)), sq.idf);
                        if (vs[e] > 0.0f) my_max = max(my_max, __float_as_uint(vs[e]));
                    }
                }
                reinterpret_cast<float4 *>(s_tile)[g] = make_float4(vs[0], vs[1], vs[2], vs[3]);
            }
        }
        __syncthreads();
        flush_tile_collect<true, DEEP>(s_tile, out + t0, a.topk, row, tile, my_max, n_items,
                                       min(n_items, (u32)SA_TERM_THREADS), s_top, &s_ncand, &s_tile_max);
    }
}

// --------------------------------------------------------------------------------- host
static u64 align_up(u64 v, u64 a) { return (v + a - 1) / a * a; }

void sa_span_plan_add(SpanPlan &plan, const u64 *offs, const u64 *lens, const u64 *dir_offs, u32 n_terms,
                      u32 slop, float idf, bool literal, u64 n_docs) {
    SpanQuery sq;
    memset(&sq, 0, sizeof(sq));
    sq.n_terms = n_terms;
    sq.slop = slop;
    sq.idf = idf;
    sq.literal = literal ? 1u : 0u;
    u64 shortest_len = ~0ull;
    for (u32 t = 0; t < n_terms; t++) {
        sq.off[t] = offs[t];
        sq.len[t] = lens[t];
        sq.dir_off[t] = dir_offs ? dir_offs[t] : SA_NO_DIR;
        if (sq.len[t] < shortest_len) { shortest_len = sq.len[t]; sq.shortest = t; }
    }
    if (n_terms == 0) shortest_len = 0;
    for (u32 t = 0; t < n_terms; t++) {
        sq.s_cap[t] = std::min<u64>(sq.len[t], 5 * shortest_len);
        sq.s_off[t] = plan.words_total;
        sq.g_off[t] = plan.groups_total;
        plan.words_total += sq.s_cap[t] + 2;
        plan.groups_total += sq.s_cap[t] + 2;
    }
    sq.m_off = plan.match_total;
    plan.match_total += (n_terms ? sq.s_cap[0] : 0) + 2;                 // one record per doc group of term 0
    sq.n_ctas = literal ? 0u : (u32)((shortest_len + GEN_THREADS - 1) / GEN_THREADS);
    sq.rec_off = plan.rec_total;
    sq.cta_off = plan.cta_total;
    if (!literal) {
        plan.rec_total += shortest_len * n_terms;
        plan.cta_total += (u64)sq.n_ctas * n_terms;
    }
    plan.max_ctas = std::max(plan.max_ctas, sq.n_ctas);
    plan.max_shortest = std::max(plan.max_shortest, shortest_len);
    plan.any_literal |= literal;
    // conjunction prefilter: balanced lists (the generator list is not much shorter than the rest), all with a directory
    sq.cand_off = SA_NO_DIR;
    if (n_docs && !literal && dir_offs && n_terms >= 2) {
        const char *s = getenv("SA_SPAN_CONJ_RATIO");             // read on every call, like the term knobs
        const long env = s ? atol(s) : -1;
        const u64 ratio = env >= 0 ? (u64)env : 50;
        u64 sum = 0;
        bool dirs = true;
        for (u32 t = 0; t < n_terms; t++) { sum += lens[t]; dirs = dirs && dir_offs[t] != SA_NO_DIR; }
        if (dirs && ratio && shortest_len * ratio > sum) {
            sq.cand_off = plan.cand_total;
            plan.cand_total += (u64)sa_n_tiles(n_docs) * (SA_TILE_DOCS / 32);
            plan.conj.push_back((u32)plan.qs.size());
        }
    }
    plan.qs.push_back(sq);
}

struct SpanLayout { u64 words, groups, rec, rec2, cta, matches, cand, conj, total; };
static SpanLayout span_layout(const SpanPlan &plan) {
    SpanLayout L;
    L.words = 0;
    L.groups = align_up(L.words + plan.words_total * sizeof(u64), 256);
    L.rec = align_up(L.groups + plan.groups_total * sizeof(u32), 256);
    L.rec2 = align_up(L.rec + plan.rec_total * sizeof(u64), 256);
    L.cta = align_up(L.rec2 + plan.rec_total * sizeof(u32), 256);
    L.matches = align_up(L.cta + plan.cta_total * sizeof(CtaRec), 256);
    L.cand = align_up(L.matches + plan.match_total * sizeof(u64), 256);
    L.conj = align_up(L.cand + plan.cand_total * sizeof(u32), 256);
    L.total = align_up(L.conj + plan.conj.size() * sizeof(u32), 256) + 256;
    return L;
}

size_t sa_span_scratch_bytes(const SpanPlan &plan) { return (size_t)span_layout(plan).total; }

int sa_span_is_literal(sa_index *ix, const u64 *d_lists, const u64 *offs, const u64 *lens, u32 n_terms, bool *out) {
    *out = false;
    for (u32 t = 0; t < n_terms; t++) {
        if (lens[t] == 0) return SA_OK;
        u64 first = 0;
        SA_CUDA(cudaMemcpyAsync(&first, d_lists + offs[t], sizeof(u64), cudaMemcpyDeviceToHost, ix->stream));
        SA_CUDA(cudaStreamSynchronize(ix->stream));
        if ((first & SA_HDR_MASK) != 0) return SA_OK;
    }
    *out = n_terms > 0;
    return SA_OK;
}

int sa_span_enqueue(sa_index *ix, const u64 *d_lists, const SpanPlan &plan, const SpanQuery *d_qs,
                    SpanCounts *d_counts, void *d_scratch, float *dense_rows, u64 stride,
                    const TopkCtx *topk, u32 topk_row0) {
    const u32 Q = (u32)plan.qs.size();
    if (Q == 0) return SA_OK;
    SA_CHECK(plan.groups_total < 0xFFFFFFFFull && plan.words_total < 0xFFFFFFFFull, "slop query too large");
    const SpanLayout L = span_layout(plan);
    char *base = (char *)d_scratch;
    SpanArgs a;
    memset(&a, 0, sizeof(a));
    a.words = d_lists;
    a.tile_dir = (d_lists == ix->d_words.as<u64>()) ? ix->d_tile_dir.as<u32>() : nullptr;
    a.queries = d_qs;
    a.counts = d_counts;
    a.word_arena = (u64 *)(base + L.words);
    a.group_arena = (u32 *)(base + L.groups);
    a.rec = (u64 *)(base + L.rec);
    a.rec2 = (u32 *)(base + L.rec2);
    a.cta = (CtaRec *)(base + L.cta);
    a.out = dense_rows;
    a.out_stride = stride;
    a.n_docs = ix->n_docs;
    a.doc_base = ix->doc_base;
    SA_CUDA(cudaMemsetAsync(d_counts, 0, (size_t)Q * sizeof(SpanCounts), ix->stream));
    if (topk) {
        a.matches = (u64 *)(base + L.matches);
        a.norm = ix->d_norm.as<float>();
        a.topk = *topk;
        a.topk_row0 = topk_row0;
        const DocChunks chunks = phrase_doc_chunks(ix, Q, 16);
        a.n_chunks = chunks.n_chunks;
        a.docs_per_chunk = chunks.docs_per_chunk;
        // rows are addressed by absolute row (topk_row0 + q) in span_tiles_kernel
        a.out = dense_rows - (u64)topk_row0 * stride;
    } else {
        SA_CUDA(cudaMemsetAsync(dense_rows, 0, (size_t)Q * stride * sizeof(float), ix->stream));
    }
    a.cand_bits = (u32 *)(base + L.cand);
    a.conj = (const u32 *)(base + L.conj);
    KernelTimer t(ix, 2);
    if (!plan.conj.empty()) {
        SA_CHECK(a.tile_dir, "span conjunction prefilter needs the index's own lists");
        SA_CUDA(cudaMemcpyAsync(base + L.conj, plan.conj.data(), plan.conj.size() * sizeof(u32), cudaMemcpyHostToDevice, ix->stream));
        span_cand_kernel<<<dim3((unsigned)plan.conj.size(), sa_n_tiles(ix->n_docs)), 256, 0, ix->stream>>>(a);
        SA_CUDA(cudaGetLastError());
        ix->stats.phrase_kernel_launches += 1;
        ix->stats.total_launches += 1;
    }
    if (plan.max_ctas) {
        dim3 grid(plan.max_ctas, Q);
        span_presence_kernel<<<grid, GEN_THREADS, 0, ix->stream>>>(a);
        SA_CUDA(cudaGetLastError());
        span_scan_kernel<<<Q, GEN_THREADS, 0, ix->stream>>>(a);
        SA_CUDA(cudaGetLastError());
        span_write_kernel<<<grid, GEN_THREADS, 0, ix->stream>>>(a);
        SA_CUDA(cudaGetLastError());
        ix->stats.phrase_kernel_launches += 3;
        ix->stats.total_launches += 3;
    }
    if (plan.any_literal) {
        // the reference's header-0 underflow corner (see span_candidates_literal_kernel)
        for (u32 q = 0; q < Q; q++) {
            const SpanQuery &sq = plan.qs[q];
            if (!sq.literal) continue;
            const u64 cap3 = 3 * sq.len[0] + 3 * sq.len[sq.shortest] + 16;
            DevBuf lit;
            int rc;
            if ((rc = lit.reserve((9 * cap3 + 8 * cap3) * sizeof(u64)))) return rc;
            span_candidates_literal_kernel<<<1, 1, 0, ix->stream>>>(a, q, lit.as<u64>(), cap3);
            SA_CUDA(cudaGetLastError());
            span_groups_build_kernel<<<1, GEN_THREADS, 0, ix->stream>>>(a, q);
            SA_CUDA(cudaGetLastError());
            SA_CUDA(cudaStreamSynchronize(ix->stream));
            ix->stats.phrase_kernel_launches += 2;
            ix->stats.total_launches += 2;
        }
    }
    SA_CUDA(cudaFuncSetAttribute(span_groups_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)(SPAN_WARPS * sizeof(WarpSpans))));
    const u64 max_iters = std::max<u64>(1, 5 * plan.max_shortest);
    const u64 want = (max_iters + SPAN_WARPS - 1) / SPAN_WARPS;
    const u64 budget = std::max<u64>(8, (u64)ix->num_sms * 4 / Q);
    dim3 grid2((unsigned)std::max<u64>(1, std::min<u64>(want, budget)), Q);
    span_groups_kernel<<<grid2, SPAN_WARPS * 32, SPAN_WARPS * sizeof(WarpSpans), ix->stream>>>(a);
    SA_CUDA(cudaGetLastError());
    ix->stats.phrase_kernel_launches += 1;
    ix->stats.total_launches += 1;
    if (topk) {
        span_sorted_kernel<<<dim3(8, Q), GEN_THREADS, 0, ix->stream>>>(a);
        SA_CUDA(cudaGetLastError());
        if (a.topk.k > SA_TOPK_MAX) span_tiles_kernel<true><<<dim3(Q, a.n_chunks), SA_TERM_THREADS, 0, ix->stream>>>(a);
        else span_tiles_kernel<false><<<dim3(Q, a.n_chunks), SA_TERM_THREADS, 0, ix->stream>>>(a);
        SA_CUDA(cudaGetLastError());
        if (a.topk.k > SA_TOPK_MAX) ix->stats.deep_tiles += (u64)Q * sa_n_tiles(ix->n_docs);
        ix->stats.phrase_kernel_launches += 2;
        ix->stats.total_launches += 2;
    }
    t.stop();
    return SA_OK;
}

// Span search of one query into ix->dense row 0 (raw counts).  Caller holds ix->mu.
int sa_span_run(sa_index *ix, const u64 *d_lists, const u64 *offs, const u64 *lens, const u64 *dir_offs,
                uint32_t n_terms, uint32_t slop, bool literal) {
    const u64 stride = sa_padded_docs(ix->n_docs);
    int rc;
    if ((rc = ix->dense.reserve(stride * sizeof(float)))) return rc;
    SpanPlan plan;
    sa_span_plan_add(plan, offs, lens, dir_offs, n_terms, slop, 0.0f, literal, d_lists == ix->d_words.as<u64>() ? ix->n_docs : 0);
    if ((rc = ix->phrase_scratch.reserve(sa_span_scratch_bytes(plan)))) return rc;
    if ((rc = ix->queries.reserve(sizeof(SpanQuery)))) return rc;
    if ((rc = ix->cand_meta.reserve(sizeof(SpanCounts)))) return rc;
    SA_CUDA(cudaMemcpyAsync(ix->queries.p, plan.qs.data(), sizeof(SpanQuery), cudaMemcpyHostToDevice, ix->stream));
    if ((rc = sa_span_enqueue(ix, d_lists, plan, ix->queries.as<SpanQuery>(), ix->cand_meta.as<SpanCounts>(),
                              ix->phrase_scratch.p, ix->dense.as<float>(), stride))) return rc;
    SpanCounts h;
    SA_CUDA(cudaMemcpyAsync(&h, ix->cand_meta.p, sizeof(h), cudaMemcpyDeviceToHost, ix->stream));
    SA_CUDA(cudaStreamSynchronize(ix->stream));
    SA_CHECK(!h.overflow, "span candidate arena exhausted (internal sizing error)");
    return SA_OK;
}
