// Host-side helpers shared by the model engines: GEMM parameter builders over packed activations.
#pragma once
#include <string.h>

#include "te_gemm.cuh"
#include "te_gemm_tc.h"
#include "te_kernels.h"

// 1 (default): the z+ rules of the top block run on the pooled-token rows only (exact); te_set_option("cls_row_top_block", 0)
// restores the all-rows form for A/B comparison
bool te_engine_cls_rows();
void te_engine_set_cls_rows(int on);
// 1 (default): with TE_FLAG_LINEAR_F16_SPLIT the fc1 GEMM's GELU epilogue emits the fp16 split of gelu(y) for the fc2 GEMM;
// te_set_option("gelu_split_fused", 0) / TE_B200_GELU_SPLIT=0 restores the stand-alone pre-pass
bool te_engine_gelu_split();
void te_engine_set_gelu_split(int on);

namespace te_util {

static inline TeGemm gemm0() {
    TeGemm p;
    memset(&p, 0, sizeof(p));
    p.nb1 = 1; p.nb2 = 1; p.alpha = 1.f;
    return p;
}

// y[M,out] = x[M,in] * W[out,in]^T  (+ epilogue);  y2 / e0 share y's row stride
static inline int linear_fwd(const float* x, int lda, const float* w, const float* bias, float* y, float* y2,
                             const float* e0, long long M, int in, int out, int epi, cudaStream_t st) {
    TeGemm p = gemm0();
    p.A = x; p.lda = lda; p.B = w; p.ldb = in; p.C = y; p.ldc = out; p.C2 = y2; p.ldc2 = out; p.E0 = e0; p.lde0 = out;
    p.bias = bias; p.M = (int)M; p.N = out; p.K = in;
    return te_gemm_launch(p, TE_L_K, TE_L_K, TE_XF_NONE, epi, st);
}
// dx[M,in] = dy[M,out] * W[out,in]
static inline int linear_bwd(const float* dy, const float* w, float* dx, const float* e0, long long M, int in, int out,
                             int epi, cudaStream_t st) {
    TeGemm p = gemm0();
    p.A = dy; p.lda = out; p.B = w; p.ldb = in; p.C = dx; p.ldc = in; p.E0 = e0; p.lde0 = in;
    p.M = (int)M; p.N = in; p.K = out;
    return te_gemm_launch(p, TE_L_K, TE_L_MN, TE_XF_NONE, epi, st);
}

// tensor-core (3xTF32) variants when the derived weight copies are supplied and the shape qualifies
// fp16-split forward Linear (TE_FLAG_LINEAR_F16_SPLIT, te_tc_wgmma.cu): where the block-scaled split of the input lives
// (M*in floats + M*ceil(in/128) floats), whether its producer already filled it (ready: te_launch_layernorm_split or the previous
// GEMM's GELU epilogue), and where the GELU epilogue puts the split of y2 for the next Linear (may be NULL)
struct F16Split { float* split; float* scale; bool ready; float* split_out; float* scale_out; };
static inline int linear_fwd_tc(const float* dw, const float* x, int lda, const float* w, const float* bias, float* y,
                                float* y2, const float* e0, long long M, int in, int out, int epi, cudaStream_t st,
                                const F16Split* fs = nullptr) {
    if (dw && fs && fs->split && epi != TE_EPI_GELU_BWD && te_tc_fwd16_supported(M, in, out, lda))
        return te_tc_linear_fwd16(fs->ready ? nullptr : x, lda, fs->split, fs->scale, dw, in, out, bias, y, y2, e0, M, epi, st,
                                  epi == TE_EPI_BIAS_GELU ? fs->split_out : nullptr, epi == TE_EPI_BIAS_GELU ? fs->scale_out : nullptr);
    if (dw && te_tc_gemm3x_supported(M, in, out, lda))
        return te_tc_linear_fwd(x, lda, dw, in, out, bias, y, y2, e0, M, epi, st);      // epilogue ids coincide
    return linear_fwd(x, lda, w, bias, y, y2, e0, M, in, out, epi, st);
}
// tf32: single-pass TF32 on the persistent CTA-pair kernel (TE_FLAG_BACKWARD_TF32) instead of the 3xTF32 split
// fs: hi-only split scratch of dy (M*out/2 floats + M*ceil(out/128)) -> single-pass fp16 kernel (TE_FLAG_BACKWARD_F16)
static inline int linear_bwd_tc(const float* dw, const float* dy, const float* w, float* dx, const float* e0, long long M,
                                int in, int out, int epi, cudaStream_t st, bool tf32 = false, const F16Split* fs = nullptr) {
    if (dw && fs && fs->split && (epi == TE_EPI_STORE || epi == TE_EPI_GELU_BWD) && te_tc_f16_single_supported(M, out, in, out))
        return te_tc_linear_bwd16(fs->ready ? nullptr : dy, out, fs->split, fs->scale, dw, in, out, dx, e0, M, epi, st);
    if (dw && tf32 && (epi == TE_EPI_STORE || epi == TE_EPI_GELU_BWD) && te_tc_pair_supported(M, out, in, out))
        return te_tc_pair_linear_bwd(dy, out, dw, in, out, dx, e0, M, epi, st);
    if (dw && te_tc_gemm3x_supported(M, out, in, out))
        return te_tc_linear_bwd(dy, dw, in, out, dx, e0, M, epi, st);
    return linear_bwd(dy, w, dx, e0, M, in, out, epi, st);
}

// one operand of a (batch, head)-batched attention-shaped GEMM
struct HeadOp { const float* ptr; int ld; long long s1, s2; };
static inline HeadOp head_rows(const float* base, int ld, int N, int dh) {        // [b, n, (h d)] slice, rows = tokens
    return {base, ld, (long long)N * ld, (long long)dh};
}
static inline HeadOp attn_map(const float* base, int H, int N, int NP) {          // [b, h, n, NP]
    return {base, NP, (long long)H * N * NP, (long long)N * NP};
}
static inline int head_gemm(int B, int H, HeadOp A, int alay, HeadOp Bm, int blay, HeadOp C, HeadOp E, int M, int N,
                            int K, float alpha, int epi, cudaStream_t st) {
    TeGemm p = gemm0();
    p.A = A.ptr; p.lda = A.ld; p.sA1 = A.s1; p.sA2 = A.s2;
    p.B = Bm.ptr; p.ldb = Bm.ld; p.sB1 = Bm.s1; p.sB2 = Bm.s2;
    p.C = const_cast<float*>(C.ptr); p.ldc = C.ld; p.sC1 = C.s1; p.sC2 = C.s2;
    p.E0 = E.ptr; p.lde0 = E.ld; p.sE1 = E.s1; p.sE2 = E.s2;
    p.M = M; p.N = N; p.K = K; p.nb1 = B; p.nb2 = H; p.alpha = alpha;
    return te_gemm_launch(p, alay, blay, TE_XF_NONE, epi, st);
}

// out[b,h,:,:] = epi(alpha * A_h B_h^T) for head slices A, B of packed [batch*N, ld] activations
// (Q K^T, dctx V^T, S2 V^T).  tc: fp32-grade 3xTF32 tensor-core kernel when the shape qualifies.
// tf32: single-pass TF32 (STORE / MUL epilogues; gradient and relevance products, never a denominator)
static inline int attn_nn(bool tc, int B, int H, int N, int NP, int dh, const float* A, int lda, const float* Bm, int ldb,
                          float* out, const float* E, float alpha, int epi, cudaStream_t st, bool tf32 = false) {
    if (tc && te_tc_attn_supported(N, dh, lda, ldb, NP)) {
        const int e = (epi == TE_EPI_STORE) ? TE_TC_ATTN_STORE : (epi == TE_EPI_MUL) ? TE_TC_ATTN_MUL : TE_TC_ATTN_SD;
        return te_tc_attn_nn(A, lda, Bm, ldb, B, H, N, dh, out, NP, E, alpha, e, st, tf32 && N <= 256 && epi != TE_EPI_SD);
    }
    const HeadOp none = {nullptr, 0, 0, 0};
    return head_gemm(B, H, head_rows(A, lda, N, dh), TE_L_K, head_rows(Bm, ldb, N, dh), TE_L_K, attn_map(out, H, N, NP),
                     E ? attn_map(E, H, N, NP) : none, N, N, dh, alpha, epi, st);
}

// P[b,h] = softmax(alpha * Q_h K_h^T): fused into the tensor-core kernel's epilogue when the key axis fits one tile
// (N <= 256), otherwise scores + row softmax
static inline int attn_probs(bool tc, int B, int H, int N, int NP, int dh, const float* Q, int ldq, const float* K, int ldk,
                             float* P, float alpha, cudaStream_t st) {
    if (tc && N <= 256 && te_tc_attn_supported(N, dh, ldq, ldk, NP))
        return te_tc_attn_nn(Q, ldq, K, ldk, B, H, N, dh, P, NP, nullptr, alpha, TE_TC_ATTN_SOFTMAX, st);
    TE_TRY(attn_nn(tc, B, H, N, NP, dh, Q, ldq, K, ldk, P, nullptr, alpha, TE_EPI_STORE, st));
    return te_launch_softmax(P, (long long)B * H * N, N, NP, st);
}

// out[b,m,h,:] = epi(alpha * sum_k A_h[m,k] X[b,k,h,:]) with A_h = map[b,h] (amn = 0) or map[b,h]^T (amn = 1)
// tf32: single-pass TF32 (activation-gradient contractions, TE_FLAG_BACKWARD_TF32)
static inline int attn_nk(bool tc, int B, int H, int N, int NP, int dh, const float* map, int amn, const float* X, int ldx,
                          float* out, int ld_out, const float* E, float alpha, int epi, cudaStream_t st, bool tf32 = false) {
    if (tc && te_tc_attn_nk_supported(N, dh, NP, ldx, ld_out)) {
        const int e = (epi == TE_EPI_STORE) ? TE_TC_ATTN_STORE : TE_TC_ATTN_MUL;
        if (epi == TE_EPI_STORE || epi == TE_EPI_MUL)
            return te_tc_attn_nk(map, NP, amn, X, ldx, B, H, N, out, ld_out, E, alpha, e, st, tf32);
    }
    const HeadOp none = {nullptr, 0, 0, 0};
    return head_gemm(B, H, attn_map(map, H, N, NP), amn ? TE_L_MN : TE_L_K, head_rows(X, ldx, N, dh), TE_L_MN,
                     head_rows(out, ld_out, N, dh), E ? head_rows(E, ld_out, N, dh) : none, N, dh, N, alpha, epi, st);
}

}  // namespace te_util
