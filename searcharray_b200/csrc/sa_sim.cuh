// sa_sim.cuh -- the per-element formulas of the reference's non-default similarities (searcharray/similarity.py:41-89),
// shared by sa_op_similarity (SearchArray.score) and the batched top-k (sim_tile_kernel, sa_view.cu) so that the two
// cannot drift apart.  What parity depends on is numpy's dtype promotion: the Python-float parameters become float32
// next to the float32 arrays (k1, b, `1 - b` and `k1 + 1` are computed in double and THEN rounded), the idf scalars
// are float64 and make the final product float64 (legacy, classic).  Every operation is individually rounded
// (-fmad=false, *_rn).
#pragma once
#include "sa_common.cuh"

struct SimParams {
    float k1, b, one_minus_b, k1_plus_1, avgdl;
};

// the float32 parameters from the Python floats, as numpy rounds them
inline SimParams make_sim_params(double avg_doc_len, double k1, double b) {
    SimParams p;
    p.k1 = (float)k1;
    p.b = (float)b;
    p.one_minus_b = (float)(1 - b);          // Python: `1 - b` in double, rounded when it meets the array
    p.k1_plus_1 = (float)(k1 + 1);
    p.avgdl = (float)avg_doc_len;
    return p;
}

#ifdef __CUDACC__
__device__ __forceinline__ float saturation_denominator(float tf, float dl, const SimParams &a) {
    // tf + k1 * (1 - b + b * doc_lens / avg_doc_lens), left to right as numpy evaluates it
    const float ratio = __fdiv_rn(__fmul_rn(a.b, dl), a.avgdl);
    return __fadd_rn(tf, __fmul_rn(a.k1, __fadd_rn(a.one_minus_b, ratio)));
}

// bm25_impact: float32
__device__ __forceinline__ float sim_impact(float tf, float dl, const SimParams &a) {
    return __fdiv_rn(tf, saturation_denominator(tf, dl, a));
}

// bm25_legacy_similarity: the float32 saturation, then idf * (double)sat
__device__ __forceinline__ float sim_legacy_sat(float tf, float dl, const SimParams &a) {
    return __fdiv_rn(__fmul_rn(tf, a.k1_plus_1), saturation_denominator(tf, dl, a));
}
__device__ __forceinline__ double sim_legacy(double idf, float sat) { return __dmul_rn(idf, (double)sat); }

// classic_similarity: (idf * sqrt(tf)) * (1 / sqrt(dl)), the products in float64
__device__ __forceinline__ double sim_classic(double idf, float tf, float dl) {
    const float length_norm = __fdiv_rn(1.0f, __fsqrt_rn(dl));
    return __dmul_rn(__dmul_rn(idf, (double)__fsqrt_rn(tf)), (double)length_norm);
}
#endif
