// z+ Linear rule driver: fp32 SIMT path (te_gemm.cu) or wgmma tensor-core path (te_tc_wgmma.cu).
#include "te_zplus.h"
#include "../../include/te_b200.h"
#include "te_gemm.cuh"
#include "te_gemm_tc.h"
#include <math.h>
#include <string.h>

ZplusVariant te_zplus_from_flags(unsigned flags) {
    return {(flags & TE_FLAG_ZPLUS_BF16) != 0, (flags & TE_FLAG_ZPLUS_S1_BF16) != 0, (flags & TE_FLAG_ZPLUS_R_F16) != 0};
}

int te_zplus_linear_relprop(const float* x, long long ldx, const float* w, const float* w_derived, const float* r,
                            long long ldr, float* out, float* s_scratch, long long rows, int in_features,
                            int out_features, cudaStream_t st, const float* y, long long ldy, const float* bias, ZplusVariant zv,
                            long long ld_out, float* xabs, float alpha) {
    if (rows <= 0) return TE_OK;
    if (ld_out == 0) ld_out = in_features;
    if (!isfinite(alpha)) { te_set_last_error("zplus: alpha must be finite"); return TE_ERR_ARG; }
    if (rows > 0x7fffffffLL || ldx > 0x7fffffffLL) { te_set_last_error("zplus: rows/ldx overflow int"); return TE_ERR_ARG; }
    if (w_derived && ldr % 4 == 0 && ld_out % 4 == 0 && te_tc_zplus_supported(rows, in_features, out_features, ldx)) {
        const int rc = te_tc_zplus_linear_relprop(x, ldx, w_derived, r, ldr, out, s_scratch, rows, in_features, out_features, st, y,
                                                  ldy, bias, zv, ld_out, xabs, alpha);
        if (rc != TE_ERR_UNSUPPORTED) return rc;
    }
    if (ld_out > 0x7fffffffLL) { te_set_last_error("zplus: ld_out overflow int"); return TE_ERR_ARG; }
    TeGemm p;
    memset(&p, 0, sizeof(p));
    p.nb1 = p.nb2 = 1; p.alpha = 1.f;
    const float beta = alpha - 1.f;
    auto s_pass = [&]() {
        p.A = x; p.lda = (int)ldx; p.B = w; p.ldb = in_features; p.C = s_scratch; p.ldc = out_features;
        p.E0 = r; p.lde0 = (int)ldr; p.M = (int)rows; p.N = out_features; p.K = in_features;
    };
    auto r_pass = [&]() {
        p.A = s_scratch; p.lda = out_features; p.B = w; p.ldb = in_features; p.C = out; p.ldc = (int)ld_out;
        p.E0 = x; p.lde0 = (int)ldx; p.M = (int)rows; p.N = in_features; p.K = out_features;
    };
    // activator: S = alpha * sd(R, x+ W+^T + x- W-^T)  (alpha = 1: the plain z+ rule, unscaled)
    s_pass();
    p.scale = alpha;
    TE_TRY(te_gemm_launch(p, TE_L_K, TE_L_K, TE_XF_AB_POSNEG, alpha == 1.f ? TE_EPI_SD : TE_EPI_SD_SCALED, st));
    // R_in = x+ * (S W+) + x- * (S W-)
    r_pass();
    TE_TRY(te_gemm_launch(p, TE_L_K, TE_L_MN, TE_XF_B_POS, TE_EPI_MULPOS, st));
    TE_TRY(te_gemm_launch(p, TE_L_K, TE_L_MN, TE_XF_B_NEG, TE_EPI_MULNEG_ACC, st));
    if (beta == 0.f) return TE_OK;
    // inhibitor, through the same S buffer: S = -beta * sd(R, x+ W-^T + x- W+^T) ; R_in += x+ * (S W-) + x- * (S W+)
    s_pass();
    p.scale = -beta;
    TE_TRY(te_gemm_launch(p, TE_L_K, TE_L_K, TE_XF_AB_NEGPOS, TE_EPI_SD_SCALED, st));
    r_pass();
    TE_TRY(te_gemm_launch(p, TE_L_K, TE_L_MN, TE_XF_B_NEG, TE_EPI_MULPOS_ACC, st));
    TE_TRY(te_gemm_launch(p, TE_L_K, TE_L_MN, TE_XF_B_POS, TE_EPI_MULNEG_ACC, st));
    return TE_OK;
}

int te_zplus_linear_relprop_lrp(const float* x, long long ldx, const float* w, const float* w_derived, const float* r,
                                long long ldr, float* out, float* s_scratch, long long rows, int in_features, int out_features,
                                cudaStream_t st, long long ld_out, float alpha) {
    if (rows <= 0) return TE_OK;
    if (ld_out == 0) ld_out = in_features;
    if (!isfinite(alpha)) { te_set_last_error("zplus_lrp: alpha must be finite"); return TE_ERR_ARG; }
    if (rows > 0x7fffffffLL || ldx > 0x7fffffffLL || ldr > 0x7fffffffLL || ld_out > 0x7fffffffLL) {
        te_set_last_error("zplus_lrp: overflow");
        return TE_ERR_ARG;
    }
    if (w_derived && te_tc_zplus_supported(rows, in_features, out_features, ldx) && ldr % 4 == 0 && ld_out % 4 == 0)
        return te_tc_lrp_linear_relprop(x, ldx, w_derived, r, ldr, out, ld_out, s_scratch, rows, in_features, out_features, st,
                                        alpha);
    TeGemm p;
    memset(&p, 0, sizeof(p));
    p.nb1 = p.nb2 = 1; p.alpha = 1.f;
    const float beta = alpha - 1.f;
    // the four products in order: activator x+ W+, x- W-, then (beta != 0) inhibitor x+ W-, x- W+; each over its own
    // denominator, S scaled by alpha (activator) or -beta (inhibitor); the first one writes out, the others add to it
    struct Half { int s_xf, r_xf, r_epi; };
    const Half halves[4] = {{TE_XF_AB_POS, TE_XF_B_POS, TE_EPI_MULPOS}, {TE_XF_AB_NEG, TE_XF_B_NEG, TE_EPI_MULNEG_ACC},
                            {TE_XF_A_POS_B_NEG, TE_XF_B_NEG, TE_EPI_MULPOS_ACC}, {TE_XF_A_NEG_B_POS, TE_XF_B_POS, TE_EPI_MULNEG_ACC}};
    for (int half = 0; half < (beta == 0.f ? 2 : 4); ++half) {
        const Half& h = halves[half];
        // S_half = scale * sd(R, x+- W+-^T)
        p.A = x; p.lda = (int)ldx; p.B = w; p.ldb = in_features; p.C = s_scratch; p.ldc = out_features;
        p.E0 = r; p.lde0 = (int)ldr; p.M = (int)rows; p.N = out_features; p.K = in_features;
        p.scale = half < 2 ? alpha : -beta;
        TE_TRY(te_gemm_launch(p, TE_L_K, TE_L_K, h.s_xf, alpha == 1.f ? TE_EPI_SD : TE_EPI_SD_SCALED, st));
        // R_in (+)= x+- * (S_half W+-)
        p.A = s_scratch; p.lda = out_features; p.B = w; p.ldb = in_features; p.C = out; p.ldc = (int)ld_out;
        p.E0 = x; p.lde0 = (int)ldx; p.M = (int)rows; p.N = in_features; p.K = out_features;
        TE_TRY(te_gemm_launch(p, TE_L_K, TE_L_MN, h.r_xf, h.r_epi, st));
    }
    return TE_OK;
}

int te_linear_rule_relprop(bool lrp, const float* x, long long ldx, const float* w, const float* w_derived, const float* r,
                           long long ldr, float* out, float* s_scratch, long long rows, int in_features, int out_features,
                           cudaStream_t st, const float* y, long long ldy, const float* bias, ZplusVariant zv,
                           long long ld_out, float* xabs, float alpha) {
    if (lrp)
        return te_zplus_linear_relprop_lrp(x, ldx, w, w_derived, r, ldr, out, s_scratch, rows, in_features, out_features, st,
                                           ld_out, alpha);
    return te_zplus_linear_relprop(x, ldx, w, w_derived, r, ldr, out, s_scratch, rows, in_features, out_features, st, y, ldy,
                                   bias, zv, ld_out, xabs, alpha);
}
