// z+ rule of Linear.relprop (modules/layers_ours.py:207-230, alpha=1):
//   Z = x+ W+^T + x- W-^T ; S = safe_divide(R, Z) ; R_in = x+ * (S W+) + x- * (S W-)
// alpha-beta rule (alpha != 1, beta = alpha - 1): R_in = alpha * act - beta * inh, act the z+ result above and inh the same
// rule with the weight signs swapped: S_i = sd(R, x+ W-^T + x- W+^T), inh = x+ * (S_i W-) + x- * (S_i W+).  The drivers run
// the inhibitor half after the activator half through the same s_scratch, with alpha and -beta folded into S, adding into
// out.  alpha = 1 launches exactly the z+ rule.  A non-finite alpha returns TE_ERR_ARG.
#pragma once
#include "te_common.cuh"

// Reduced-precision variants of the tensor-core z+ rule, decoded from the engine flags by te_zplus_from_flags:
//   r_bf16  (TE_FLAG_ZPLUS_BF16)     S is stored as bf16 and the second contraction runs on bf16 operands
//   s1_bf16 (TE_FLAG_ZPLUS_S1_BF16)  the |x| |W|^T term of the single-pass S kernel on bf16 operands
//   r_f16   (TE_FLAG_ZPLUS_R_F16)    the second contraction on fp16 MMAs, fed a block-scaled fp16 S by the S kernel's epilogue
struct ZplusVariant { bool r_bf16, s1_bf16, r_f16; };
ZplusVariant te_zplus_from_flags(unsigned flags);

// x [rows, in] with row stride ldx ; w [out, in] ; r [rows, out] with row stride ldr (a column slice of a packed
// [rows, 3*out] relevance tensor) ; out [rows, in] ; s_scratch [rows, out].
// w_derived: the te_tc_prepare_weights() copies of w, or NULL.  When given (and the shape qualifies) both
// contractions run on wgmma tensor cores (TF32 inputs, fp32 accumulate); otherwise — and as the checker —
// the fp32 SIMT path.
// y / bias: the Linear's saved forward output and bias (optional; enables the single-pass tensor-core S kernel)
int te_zplus_linear_relprop(const float* x, long long ldx, const float* w, const float* w_derived, const float* r,
                            long long ldr, float* out, float* s_scratch, long long rows, int in_features,
                            int out_features, cudaStream_t st, const float* y = nullptr, long long ldy = 0,
                            const float* bias = nullptr, ZplusVariant zv = {}, long long ld_out = 0,
                            float* xabs = nullptr, float alpha = 1.f);
// xabs: scratch [rows, in] (the |x| operand of the single-pass S kernel); without it the tensor-core path uses the two-pass
// S kernel.
// ld_out: row stride of out (0 = in_features).  With row strides on x, r, y and out the rule runs on a strided subset of
// token rows — the CLS rows of the top block, the only rows whose relevance is non-zero there (SURVEY.md 8a).

// Linear.relprop of the layers_lrp baseline variant (modules/layers_lrp.py:187-210, alpha=1): S1 = sd(R, x+ W+^T),
// S2 = sd(R, x- W-^T) (separate denominators), R_in = x+ * (S1 W+) + x- * (S2 W-).  s_scratch [rows, out] holds S1, then S2.
// alpha != 1: R_in = alpha * act - beta * inh with inh = x+ * (sd(R, x+ W-^T) W-) + x- * (sd(R, x- W+^T) W+), its two products
// run after the activator's through the same s_scratch.
// w_derived: the te_tc_prepare_weights() copies of w, or NULL.  When given (and the shape qualifies) both halves run on
// single-pass TF32 wgmma (TE_FLAG_RULES_LRP_TC; every denominator is a sum of non-negative products); otherwise fp32 SIMT.
// ld_out: row stride of out (0 = in_features), for the strided row subsets of te_zplus_linear_relprop.
int te_zplus_linear_relprop_lrp(const float* x, long long ldx, const float* w, const float* w_derived, const float* r,
                                long long ldr, float* out, float* s_scratch, long long rows, int in_features, int out_features,
                                cudaStream_t st, long long ld_out = 0, float alpha = 1.f);

// The Linear rule of the selected rule library: lrp (TE_FLAG_RULES_LRP) runs te_zplus_linear_relprop_lrp, which does not
// read y, ldy, bias, zv or xabs; otherwise te_zplus_linear_relprop (layers_ours).  The other arguments go to either as given.
int te_linear_rule_relprop(bool lrp, const float* x, long long ldx, const float* w, const float* w_derived, const float* r,
                           long long ldr, float* out, float* s_scratch, long long rows, int in_features, int out_features,
                           cudaStream_t st, const float* y, long long ldy, const float* bias, ZplusVariant zv,
                           long long ld_out, float* xabs, float alpha);
