// Tensor-core (Hopper wgmma) GEMMs of the engines (te_tc_wgmma.cu): TF32 / bf16 / fp16 operands, fp32 accumulation.
#pragma once
#include <cuda_bf16.h>
#include <type_traits>

#include "te_common.cuh"
#include "te_zplus.h"

// shapes the tensor-core z+ path accepts (in/out multiples of 128, 16-byte aligned rows)
bool te_tc_zplus_supported(long long rows, int in_features, int out_features, long long ldx);

// The derived copies of one frozen weight W [out,in] in its buffer of floats(in, out) = 16 n floats (n = in*out), all K-major.
// F = float where the copies are made, const float where the kernels read them.  Offsets in floats:
//   0 .. 4n     W+, W-, W+^T, W-^T rounded to TF32: operands of the two-pass z+ S and the TF32 R kernels
//   4n .. 8n    W_hi, W_lo, W^T_hi, W^T_lo: error-compensated split (x_hi = tf32(x), x_lo = tf32(x - x_hi)) of the fp32-grade
//               3xTF32 forward / backward Linear; W^T_hi is also the operand of the single-pass TF32 backward
//   8n          tf32(|W|): operand of the single-pass S kernel
//   9n          bf16(W+^T), bf16(W-^T) [in,out]: operands of the bf16 R kernel
//   10n .. 11n  gap (unused)
//   11n         bf16(|W|): operand of the bf16 S1 kernel (TE_FLAG_ZPLUS_S1_BF16), n/2 floats
//   11n + n/2   fp16 hi, fp16 lo of W and the 2^-f of each of its out rows: the fp16-split forward Linear
//   13n         fp16(tf32(W)^T) and the 2^-f of each of its in rows: the single-pass fp16 backward Linear
//   14n         fp16(W+^T), fp16(W-^T), then their 2^-f per row (in each, from 15n): the fp16 R kernel
// What follows each fp16 group up to the next whole multiple of n is tail padding.
template <class F>
struct TeDerived {
    template <class T> using P = std::conditional_t<std::is_const<F>::value, const T*, T*>;
    F *wp, *wn, *wpt, *wnt;
    F *wh, *wl, *wth, *wtl;
    F* wabs;
    P<__nv_bfloat16> bf_wpt, bf_wnt;
    F* gap;
    P<__nv_bfloat16> bf_wabs;
    P<__half> h_w, l_w;
    F* s_w;
    P<__half> h_wt;
    F* s_wt;
    P<__half> h_wpt, h_wnt;
    F *s_wpt, *s_wnt;
    static constexpr long long floats(int in_features, int out_features) { return 16LL * in_features * out_features; }
    __host__ __device__ TeDerived(F* d, int in_features, int out_features) {
        const long long n = (long long)in_features * out_features;
        wp = d; wn = d + n; wpt = d + 2 * n; wnt = d + 3 * n;
        wh = d + 4 * n; wl = d + 5 * n; wth = d + 6 * n; wtl = d + 7 * n;
        wabs = d + 8 * n;
        bf_wpt = reinterpret_cast<P<__nv_bfloat16>>(d + 9 * n); bf_wnt = bf_wpt + n;
        gap = d + 10 * n;
        bf_wabs = reinterpret_cast<P<__nv_bfloat16>>(d + 11 * n);
        h_w = reinterpret_cast<P<__half>>(d + 11 * n + n / 2); l_w = reinterpret_cast<P<__half>>(d + 12 * n); s_w = d + 12 * n + n / 2;
        h_wt = reinterpret_cast<P<__half>>(d + 13 * n); s_wt = d + 13 * n + n / 2;
        h_wpt = reinterpret_cast<P<__half>>(d + 14 * n); h_wnt = reinterpret_cast<P<__half>>(d + 14 * n + n / 2);
        s_wpt = d + 15 * n; s_wnt = d + 15 * n + in_features;
    }
};
long long te_tc_derived_floats(int in_features, int out_features);
int te_tc_prepare_weights(const float* w, float* derived, int in_features, int out_features, cudaStream_t st);
// y / bias (optional): the Linear's saved forward output y = x W^T + bias [rows, out] (row stride ldy).  When given,
// Z is formed in ONE pass as ((y - bias) + |x| |W|^T) / 2  ==  x+ W+^T + x- W-^T  (exact identity), halving the S kernel.
// zv, ld_out, xabs: as in te_zplus_linear_relprop (te_zplus.h).
int te_tc_zplus_linear_relprop(const float* x, long long ldx, const float* derived, const float* r, long long ldr,
                               float* out, float* s_scratch, long long rows, int in_features, int out_features, cudaStream_t st,
                               const float* y, long long ldy, const float* bias, ZplusVariant zv, long long ld_out,
                               float* xabs, float alpha = 1.f);
// alpha != 1 (the alpha-beta rule of te_zplus.h): the inhibitor half follows the activator through s_scratch, the same kernels
// with the weight operands swapped, the single-pass S kernel with the |x| |W|^T term negated and the R kernel accumulating.
// Linear.relprop of the layers_lrp library (te_zplus_linear_relprop_lrp) on single-pass TF32 wgmma: for each half in turn,
// S = sd(R, x+- W+-^T) into s_scratch [rows, out], then out (+)= x+- * (S W+-).  Row strides ldx, ldr, ld_out; shapes as
// te_tc_zplus_supported.  alpha != 1: the inhibitor products x+ W-, x- W+ follow, every S scaled by alpha or -beta.
int te_tc_lrp_linear_relprop(const float* x, long long ldx, const float* derived, const float* r, long long ldr, float* out,
                             long long ld_out, float* s_scratch, long long rows, int in_features, int out_features,
                             cudaStream_t st, float alpha = 1.f);

// fp32-grade (3xTF32 split) Linear GEMMs; epilogues mirror the SIMT ones
enum { TE_TC_EPI_STORE = 0, TE_TC_EPI_BIAS = 1, TE_TC_EPI_BIAS_GELU = 2, TE_TC_EPI_BIAS_ADD = 3, TE_TC_EPI_GELU_BWD = 4,
       TE_TC_EPI_BIAS_QUICK_GELU = 12, TE_TC_EPI_QUICK_GELU_BWD = 13 };   // the ids of te_gemm.cuh
bool te_tc_gemm3x_supported(long long rows, int K, int N, long long lda);
int te_tc_linear_fwd(const float* x, long long ldx, const float* derived, int in_features, int out_features,
                     const float* bias, float* y, float* y2, const float* e0, long long rows, int epi, cudaStream_t st);
int te_tc_linear_bwd(const float* dy, const float* derived, int in_features, int out_features, float* dx, const float* e0,
                     long long rows, int epi, cudaStream_t st);

// fp32-grade forward Linear on fp16 MMAs: block-scaled fp16 (hi, lo) split of both operands, three MMAs per k-step.
// Activations: one scale per (row, 128 k) — split = [hi | lo] fp16 [rows, in] (rows*in floats), scale [rows, ceil(in/128)];
// weights: one scale per row of W (derived buffer).
bool te_tc_fwd16_supported(long long rows, int K, int N, long long lda);
int te_tc_rowsplit_f16(const float* x, long long ldx, long long rows, int cols, void* hi, void* lo, float* scale_inv,
                       cudaStream_t st);
int te_tc_blocksplit_f16(const float* x, long long ldx, long long rows, int cols, float* split, float* scale_inv, cudaStream_t st,
                         bool hi_only = false);
// x != NULL: split / scale are scratch filled by the pre-pass; x == NULL: they were filled by the producer of x
// (te_launch_layernorm_split or the split_out / scale_out of the previous call, TE_TC_EPI_BIAS_GELU / _BIAS_QUICK_GELU only:
// the split of y2)
int te_tc_linear_fwd16(const float* x, long long ldx, float* split, float* scale, const float* derived, int in_features,
                       int out_features, const float* bias, float* y, float* y2, const float* e0, long long rows, int epi,
                       cudaStream_t st, float* split_out = nullptr, float* scale_out = nullptr);
// single-pass fp16 products on the same kernel (A = hi only: fp16 keeps TF32's 11 significant bits, rounded to nearest);
// shapes: te_tc_fwd16_supported
// dx = epi(dy W): split (rows*out/2 floats) / scale ([rows, ceil(out/128)]) hold the hi-only split of dy (dy != NULL: pre-pass here)
int te_tc_linear_bwd16(const float* dy, long long lddy, float* split, float* scale, const float* derived, int in_features,
                       int out_features, float* dx, const float* e0, long long rows, int epi, cudaStream_t st);
// R_in = x+ (S W+) + x- (S W-): split / scale hold the hi-only split of S [rows, out] (s != NULL: pre-pass here)
int te_tc_zplus_r16(const float* s, float* split, float* scale, const float* derived, const float* x, long long ldx, float* out,
                    long long ld_out, long long rows, int in_features, int out_features, cudaStream_t st, bool inh = false);

// attention-shaped N x N contractions (Q K^T, dctx V^T, S2 V^T), fp32-grade 3xTF32, head slices in place
enum { TE_TC_ATTN_STORE = 0, TE_TC_ATTN_MUL = 1, TE_TC_ATTN_SD = 2, TE_TC_ATTN_SOFTMAX = 3 };   // SOFTMAX: N <= 256
bool te_tc_attn_supported(int N, int dh, long long lda, long long ldb, int ld_out);
// single_pass (STORE / MUL epilogues): one TF32 MMA per k-step on TF32-rounded operands (gradient / relevance products only)
int te_tc_attn_nn(const float* A, long long lda, const float* B, long long ldb, int batch, int H, int N, int dh,
                  float* out, int ld_out, const float* E, float alpha, int epi, cudaStream_t st, bool single_pass = false);

// attention-shaped N x d contractions with the reduction over tokens (attn v, attn^T dctx, dS k, dS^T q, S1 k, S1^T q ...)
bool te_tc_attn_nk_supported(int N, int dh, int NP, long long ldx, long long ld_out);
// single_pass (STORE / MUL epilogues): one TF32 MMA per k-step instead of the 3xTF32 split — the activation-gradient
// contractions under TE_FLAG_BACKWARD_TF32, the relevance contractions under TE_FLAG_RELPROP_TF32
int te_tc_attn_nk(const float* map, int NP, int amn, const float* X, long long ldx, int batch, int H, int N, float* out,
                  int ld_out, const float* E, float alpha, int epi, cudaStream_t st, bool single_pass = false);

// dense rollout product out[b] = A[b] * J[b] + diag(rowscale[b]) J[b] ([batch, N, ld]), fp32-grade 3xTF32
bool te_tc_bmm_nk_supported(int N, int ld);
int te_tc_bmm_nk_resid(const float* A, const float* J, const float* rowscale, float* out, int batch, int N, int ld,
                       cudaStream_t st);

// z+ rule contractions and the single-pass TF32 backward Linear (shapes: te_tc_gemm3x_supported)
// xabs: scratch [rows, in] for bf16(|x|), the A operand of the bf16 single-pass S kernel
// r / y: 16-byte-aligned bases, ldr and ldy multiples of 4 (the S kernel loads their tiles by TMA)
int te_tc_zplus_s1(const float* x, long long ldx, float* xabs, const float* derived, const float* r, long long ldr,
                   const float* y, long long ldy, const float* bias, float* s_out, long long rows, int in_features,
                   int out_features, cudaStream_t st, bool bf16 = false, float* s16 = nullptr, float* s16_scale = nullptr,
                   float s_scale = 1.f, bool inh = false);
// s16 / s16_scale: when given, S leaves as hi-only block-scaled fp16 [rows, out] (+ [rows, out/128] scales) — the A operand of
// te_tc_zplus_r16 — instead of fp32 in s_out.  s_scale: S = s_scale * sd(R, Z) ; inh: the inhibitor denominator
// ((y - bias) - |x| |W|^T) / 2 of the alpha-beta rule.
// inh (te_tc_zplus_r, te_tc_zplus_r16): the inhibitor half, out += x+ (S W-) + x- (S W+)
int te_tc_zplus_r(const float* s, const float* derived, const float* x, long long ldx, float* out, long long ld_out,
                  long long rows, int in_features, int out_features, cudaStream_t st, bool inh = false);
int te_tc_linear_bwd_tf32(const float* dy, long long lddy, const float* derived, int in_features, int out_features, float* dx,
                          const float* e0, long long rows, int epi, cudaStream_t st);
