// FP32 SIMT strided-batched GEMM with fused load transforms and epilogues.
//
// This is the fp32-exact workhorse of the engine: every contraction whose result feeds a
// safe_divide denominator or the arg-max (forward, activation-gradient backward, both attention
// matmul rules) runs here, because SURVEY.md §7b shows those paths do not tolerate TF32 inputs.
// The z+ Linear rule (97 % of the relprop flops, well conditioned) has a tensor-core (wgmma) path in
// te_tc_wgmma.cu; this kernel is its fp32 fallback and its checker.
//
//   C[m,n] = epi( alpha * sum_k xfA(A[m,k]) * xfB(B[k,n]) )
//
// Operand layouts: TE_L_K  -> reduction index contiguous   (A[m*lda+k] ; B[n*ldb+k])
//                  TE_L_MN -> m / n index contiguous        (A[k*lda+m] ; B[k*ldb+n])
// Batch index z = b1*nb2 + b2 with independent (s1, s2) strides per operand, which lets a head
// slice of the packed qkv tensor be addressed in place ('b n (qkv h d)', ViT_LRP.py:135).
#pragma once
#include "te_common.cuh"

enum { TE_L_K = 0, TE_L_MN = 1 };
// AB_POSNEG: [A+ | A-] [B+ | B-]^T (the reduction runs over both halves) ; AB_NEGPOS: [A+ | A-] [B- | B+]^T (the inhibitor
// denominator of the alpha-beta rule) ; A_POS_B_NEG / A_NEG_B_POS: the mixed-sign products of the layers_lrp inhibitor half
enum {
    TE_XF_NONE = 0, TE_XF_AB_POSNEG = 1, TE_XF_B_POS = 2, TE_XF_B_NEG = 3, TE_XF_AB_POS = 4, TE_XF_AB_NEG = 5,
    TE_XF_AB_NEGPOS = 6, TE_XF_A_POS_B_NEG = 7, TE_XF_A_NEG_B_POS = 8
};
enum {
    TE_EPI_STORE = 0,      // C = alpha*acc
    TE_EPI_BIAS = 1,       // C = acc + bias[n]
    TE_EPI_BIAS_GELU = 2,  // C = acc + bias[n] ; C2 = gelu(C)
    TE_EPI_BIAS_ADD = 3,   // C = acc + bias[n] ; C2 = E0 + C
    TE_EPI_GELU_BWD = 4,   // C = acc * gelu'(E0)
    TE_EPI_SD = 5,         // C = safe_divide(E0, alpha*acc)
    TE_EPI_MUL = 6,        // C = alpha * acc * E0
    TE_EPI_MULPOS = 7,     // C  = max(E0,0) * acc
    TE_EPI_MULNEG_ACC = 8, // C += min(E0,0) * acc
    TE_EPI_ACCUM = 9,      // C += alpha*acc
    TE_EPI_SD_SCALED = 10, // C = scale * safe_divide(E0, alpha*acc)
    TE_EPI_MULPOS_ACC = 11, // C += max(E0,0) * acc
    TE_EPI_BIAS_QUICK_GELU = 12,  // C = acc + bias[n] ; C2 = quick_gelu(C)   (CLIP's MLP activation)
    TE_EPI_QUICK_GELU_BWD = 13    // C = acc * quick_gelu'(E0)
};

struct TeGemm {
    const float* A; const float* B; float* C; float* C2; const float* E0; const float* bias;
    int M, N, K;
    int lda, ldb, ldc, ldc2, lde0;
    long long sA1, sA2, sB1, sB2, sC1, sC2, sE1, sE2, sD1, sD2;   // D = C2
    int nb1, nb2;
    float alpha;
    float scale;                          // TE_EPI_SD_SCALED only
    int vecA, vecB, vecC, vecC2, vecE;   // filled by te_gemm_launch
};

int te_gemm_launch(TeGemm p, int alay, int blay, int xf, int epi, cudaStream_t st);
