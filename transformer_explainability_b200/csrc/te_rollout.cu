// Aggregation + rollout, composed path: one aggregation launch per layer + a chain of batched fp32
// GEMMs.  (The fused single-kernel path is selected with TE_FLAG_ROLLOUT_FUSED, te_rollout_fused.cu.)
#include "te_rollout.h"
#include "te_kernels.h"
#include "te_rollout_fused.h"
#include "te_gemm_tc.h"
#include <string.h>

int te_rollout_chain(const float* mats, int L, int B, int N, int ld, int start_layer, float* joint_a, float* joint_b,
                     const float** result, cudaStream_t st) {
    // joint = M[start] ; for i > start: joint = M[i].bmm(joint)     (ViT_LRP.py:46-48)
    const long long ms = (long long)B * N * ld;
    const float* joint = mats + (long long)start_layer * ms;
    float* bufs[2] = {joint_a, joint_b};
    int which = 0;
    for (int i = start_layer + 1; i < L; ++i) {
        TeGemm p;
        memset(&p, 0, sizeof(p));
        p.alpha = 1.f; p.nb1 = B; p.nb2 = 1;
        p.A = mats + (long long)i * ms; p.lda = ld; p.sA1 = (long long)N * ld;
        p.B = joint; p.ldb = ld; p.sB1 = (long long)N * ld;
        p.C = bufs[which]; p.ldc = ld; p.sC1 = (long long)N * ld;
        p.M = N; p.N = N; p.K = N;
        TE_TRY(te_gemm_launch(p, TE_L_K, TE_L_MN, TE_XF_NONE, TE_EPI_STORE, st));
        joint = bufs[which];
        which ^= 1;
    }
    *result = joint;
    return TE_OK;
}

int te_rollout_layers(const float* G0, const float* cam0, long long layer_stride, int L, int B, int H, int N,
                      int ld_in, int ld, int start_layer, int normalize, unsigned flags, float* mats, float* joint_a, float* joint_b,
                      float* joint_out, float* row_out, int first, int bert_fix, cudaStream_t st, float* diag) {
    if (start_layer < 0 || start_layer >= L) { te_set_last_error("rollout: start_layer out of range"); return TE_ERR_ARG; }
    const float* joint = nullptr;
    if ((flags & 2u) && !joint_out && row_out && te_rollout_fused_supported(N, ld_in, ld)) {
        // row-only consumer (generate_LRP): fused single kernel, G / cam streamed once, nothing else in HBM
        return te_rollout_fused_row(G0, cam0, layer_stride, L, B, H, N, ld_in, start_layer, normalize, row_out, first,
                                    bert_fix, st);
    } else if ((flags & 2u) && te_tc_bmm_nk_supported(N, ld) && (!normalize || diag)) {
        // dense joint on the tensor cores, residual form: J <- A_l J + d_l J with A_l = M_l without its identity part
        // (tensor cores, 3xTF32) and the identity's share d_l (1, or 1/rowsum for BERT) applied in fp32 in the epilogue
        const long long ms = (long long)B * N * ld;
        const bool one_launch = ld_in % 4 == 0 && ld % 4 == 0 && ld_in >= ((N + 3) & ~3) && layer_stride % 4 == 0 &&
                                ((reinterpret_cast<uintptr_t>(G0) | reinterpret_cast<uintptr_t>(cam0) |
                                  reinterpret_cast<uintptr_t>(mats)) & 15u) == 0;
        if (one_launch)          // every layer's aggregation in flight at once: the stream is deep enough for the copy bandwidth
            TE_TRY(te_launch_aggregate_layers(G0, cam0, layer_stride, mats, ms, B, H, N, ld_in, ld, start_layer, L - start_layer,
                                              normalize, st, normalize ? diag : nullptr));
        else
            TE_TRY(te_launch_aggregate(G0 + start_layer * layer_stride, cam0 + start_layer * layer_stride,
                                       mats + start_layer * ms, B, H, N, ld_in, ld, /*add_eye=*/1, normalize, st));
        joint = mats + start_layer * ms;
        float* bufs[2] = {joint_a, joint_b};
        int which = 0;
        for (int l = start_layer + 1; l < L; ++l) {
            float* dl = normalize ? diag + (long long)l * B * N : nullptr;
            if (!one_launch)
                TE_TRY(te_launch_aggregate(G0 + l * layer_stride, cam0 + l * layer_stride, mats + l * ms, B, H, N, ld_in, ld,
                                           /*add_eye=*/0, normalize, st, dl));
            TE_TRY(te_tc_bmm_nk_resid(mats + l * ms, joint, dl, bufs[which], B, N, ld, st));
            joint = bufs[which];
            which ^= 1;
        }
    } else {
        const long long ms = (long long)B * N * ld;
        for (int l = start_layer; l < L; ++l)
            TE_TRY(te_launch_aggregate(G0 + l * layer_stride, cam0 + l * layer_stride, mats + l * ms, B, H, N, ld_in, ld,
                                       /*add_eye=*/1, normalize, st));
        TE_TRY(te_rollout_chain(mats, L, B, N, ld, start_layer, joint_a, joint_b, &joint, st));
    }
    if (joint_out) {
        if (cudaMemcpy2DAsync(joint_out, sizeof(float) * N, joint, sizeof(float) * ld, sizeof(float) * N,
                              (size_t)B * N, cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
            te_set_last_error("rollout: joint copy failed");
            return TE_ERR_CUDA;
        }
    }
    if (row_out) TE_TRY(te_launch_extract_row(joint, row_out, B, N, ld, first, bert_fix, st));
    return TE_OK;
}
