// sa_similarity.cu -- the reference's non-default similarities as device kernels (SURVEY.md 8f-3).
//
// Replaces the numpy closures of searcharray/similarity.py:41-89 (bm25_impact,
// bm25_legacy_similarity, classic_similarity).  The formulas, and how they reproduce numpy's
// dtype promotion, are in sa_sim.cuh (shared with the batched top-k of sa_view.cu).
#include <cmath>

#include "sa_sim.cuh"

struct SimArgs {
    const float *tf, *dl;
    u64 n;
    SimParams p;
    double idf;
    void *out;
};

template <int KIND>
__global__ void __launch_bounds__(256) similarity_kernel(const SimArgs a) {
    const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    const float tf = a.tf[i], dl = a.dl[i];
    if (KIND == SA_SIM_BM25_IMPACT) {
        ((float *)a.out)[i] = sim_impact(tf, dl, a.p);
    } else if (KIND == SA_SIM_BM25_LEGACY) {
        ((double *)a.out)[i] = sim_legacy(a.idf, sim_legacy_sat(tf, dl, a.p));
    } else {
        ((double *)a.out)[i] = sim_classic(a.idf, tf, dl);
    }
}

extern "C" int sa_op_similarity(int kind, const float *term_freqs, const float *doc_lens, uint64_t n,
                                double avg_doc_len, double idf, double k1, double b, int device, void *out) {
    if (n == 0) return SA_OK;
    SA_CHECK(term_freqs && doc_lens && out, "NULL argument");
    SA_CHECK(kind == SA_SIM_BM25_IMPACT || kind == SA_SIM_BM25_LEGACY || kind == SA_SIM_CLASSIC, "unknown similarity %d", kind);
    SA_CUDA(cudaSetDevice(device));
    const size_t out_bytes = n * (kind == SA_SIM_BM25_IMPACT ? sizeof(float) : sizeof(double));
    float *d_tf = nullptr, *d_dl = nullptr;
    void *d_out = nullptr;
    cudaError_t e = cudaMalloc(&d_tf, n * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&d_dl, n * sizeof(float));
    if (e == cudaSuccess) e = cudaMalloc(&d_out, out_bytes);
    if (e == cudaSuccess) e = cudaMemcpy(d_tf, term_freqs, n * sizeof(float), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(d_dl, doc_lens, n * sizeof(float), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
        SimArgs a;
        a.tf = d_tf; a.dl = d_dl; a.n = n;
        a.p = make_sim_params(avg_doc_len, k1, b);
        a.idf = idf;
        a.out = d_out;
        const unsigned blocks = (unsigned)((n + 255) / 256);
        if (kind == SA_SIM_BM25_IMPACT) similarity_kernel<SA_SIM_BM25_IMPACT><<<blocks, 256>>>(a);
        else if (kind == SA_SIM_BM25_LEGACY) similarity_kernel<SA_SIM_BM25_LEGACY><<<blocks, 256>>>(a);
        else similarity_kernel<SA_SIM_CLASSIC><<<blocks, 256>>>(a);
        e = cudaGetLastError();
        if (e == cudaSuccess) e = cudaMemcpy(out, d_out, out_bytes, cudaMemcpyDeviceToHost);
    }
    cudaFree(d_tf);
    cudaFree(d_dl);
    cudaFree(d_out);
    if (e != cudaSuccess) { sa_set_error("sa_op_similarity: %s", cudaGetErrorString(e)); return SA_ERR_CUDA; }
    return SA_OK;
}
