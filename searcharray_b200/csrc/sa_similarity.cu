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
    DevBuf d_tf, d_dl, d_out;
    int rc;
    if ((rc = d_tf.allocate(n * sizeof(float))) || (rc = d_dl.allocate(n * sizeof(float))) || (rc = d_out.allocate(out_bytes)))
        return rc;
    SA_CUDA(cudaMemcpy(d_tf.p, term_freqs, n * sizeof(float), cudaMemcpyHostToDevice));
    SA_CUDA(cudaMemcpy(d_dl.p, doc_lens, n * sizeof(float), cudaMemcpyHostToDevice));
    SimArgs a;
    a.tf = d_tf.as<float>(); a.dl = d_dl.as<float>(); a.n = n;
    a.p = make_sim_params(avg_doc_len, k1, b);
    a.idf = idf;
    a.out = d_out.p;
    const unsigned blocks = (unsigned)((n + 255) / 256);
    if (kind == SA_SIM_BM25_IMPACT) similarity_kernel<SA_SIM_BM25_IMPACT><<<blocks, 256>>>(a);
    else if (kind == SA_SIM_BM25_LEGACY) similarity_kernel<SA_SIM_BM25_LEGACY><<<blocks, 256>>>(a);
    else similarity_kernel<SA_SIM_CLASSIC><<<blocks, 256>>>(a);
    SA_CUDA(cudaGetLastError());
    SA_CUDA(cudaMemcpy(out, d_out.p, out_bytes, cudaMemcpyDeviceToHost));
    return SA_OK;
}
