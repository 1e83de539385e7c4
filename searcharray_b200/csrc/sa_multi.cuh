// sa_multi.cuh -- the multi-field handle (sa_multi) and the guard that puts a field's index on the handle's stream,
// shared by the edismax calls (sa_edismax.cu) and the multi-field boolean top-k (sa_bool.cu).
#pragma once
#include "sa_common.cuh"

#define ED_MAX_FIELDS 8
#define ED_MAX_ROWS 64                                               // phrase rows of one field in one sa_multi_phrases
// entries of one sa_multi_add_phase: pf2 on every field of a query of SA_MAX_PHRASE_TERMS tokens (T - 1 bigrams and
// the last one repeated), the most searcharray_b200.solr._Plan.device_ok admits
#define ED_MAX_PHASE_ENTRIES (ED_MAX_FIELDS * SA_MAX_PHRASE_TERMS)

struct sa_multi {
    ~sa_multi() {
        cudaSetDevice(device);          // the buffers below are freed after this body, on this device
        if (stream) { cudaStreamSynchronize(stream); cudaStreamDestroy(stream); }
    }
    std::vector<sa_index *> fields;
    int device = 0;
    u64 n_docs = 0, doc_base = 0, stride = 0;
    cudaStream_t stream = nullptr;
    DevBuf d_qf;                         // double [stride] combined scores (float32 values widened in field-centric mode)
    DevBuf d_mask;                       // unsigned char [stride] qf > 0 after the qf phase
    DevBuf d_count;                      // unsigned long long
    bool f32_mode = false, has_qf = false;
    std::vector<std::vector<u64>> filt_offs, filt_lens;   // per field: last sa_multi_filter
    std::vector<u32> phrase_rows;        // per field: rows produced by the last sa_multi_phrases
    std::vector<u64> filt_bound;         // per field: words reserved for filtered lists (0 = not computed yet)
    // per field: 1 when another field of the multi is the same index (two column names of one array).  Such a field
    // keeps its term and phrase rows in rows[f] instead of its index's dense scratch, which the other field's calls
    // overwrite before the combine / sa_multi_add_phase read them.
    std::vector<char> shared;
    std::vector<DevBuf> rows;
    float *field_rows(u32 f) const { return shared[f] ? rows[f].as<float>() : fields[f]->dense.as<float>(); }
    DevBuf cand;                         // top-k: candidate slots (then, for sa_multi_topk, their float64 scores)
    DevBuf keys;                         // top-k result: k keys, k float64 scores, the overflow flag
    std::unique_ptr<BoolState, BoolStateDelete> boolq;   // buffers of sa_multi_score_batch_topk_bool (sa_bool.cu)
    std::mutex mu;
};

// All kernels of one multi call run on the multi's stream, including the ones the per-field
// helpers launch on `ix->stream`: the field streams are swapped for the duration of the call.
struct FieldGuard {
    sa_index *ix;
    cudaStream_t saved;
    std::unique_lock<std::mutex> lk;
    FieldGuard(sa_index *ix_, cudaStream_t s) : ix(ix_), saved(ix_->stream), lk(ix_->mu) {
        cudaStreamSynchronize(saved);
        ix->stream = s;
    }
    ~FieldGuard() {
        cudaStreamSynchronize(ix->stream);
        ix->stream = saved;
    }
};
