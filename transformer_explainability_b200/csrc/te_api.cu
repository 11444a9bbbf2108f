// C-ABI wrappers for the stand-alone rules and rollout entry points declared in include/te_b200.h.
#include <stdlib.h>
#include <string.h>
#include <atomic>
#include <string>

#include "../../include/te_b200.h"
#include "te_engine_util.h"
#include "te_kernels.h"
#include "te_rollout.h"
#include "te_zplus.h"
#include "te_gemm_tc.h"

static thread_local std::string g_last_error;
void te_set_last_error(const char* msg) { g_last_error = msg ? msg : ""; }

static std::atomic<long long> g_launches{0};
void te_count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
extern "C" long long te_kernel_launch_count(void) { return g_launches.load(); }

extern "C" const char* te_last_error(void) { return g_last_error.c_str(); }
extern "C" int te_version(void) { return 101; }

#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define REQ(c, msg) do { if (!(c)) { te_set_last_error(msg); return TE_ERR_ARG; } } while (0)

static TeGemm g0(int nb) {
    TeGemm p;
    memset(&p, 0, sizeof(p));
    p.nb1 = nb; p.nb2 = 1; p.alpha = 1.f;
    return p;
}

// The scratch of the stand-alone tensor-core entry points, in the layouts include/te_b200.h documents:
// [S: s_floats, rounded up to 64 | the derived copies of W [out,in] | an operand: op_floats, rounded up to 64 | block scales]
// (each entry point uses the regions it needs; an empty region takes no room).
struct TcScratch { float* s; float* derived; float* op; float* scale; };
static TcScratch tc_scratch(float* scratch, long long s_floats, int in_features, int out_features, long long op_floats) {
    TcScratch c;
    c.s = scratch;
    c.derived = scratch + ((s_floats + 63) & ~63LL);
    c.op = c.derived + te_tc_derived_floats(in_features, out_features);
    c.scale = c.op + ((op_floats + 63) & ~63LL);
    return c;
}

// The Linear entries run the family the flags name or return TE_ERR_UNSUPPORTED before anything is launched.  The derived
// weight copies start the scratch; with TE_FLAG_LINEAR_F16_SPLIT the operand region holds the fp16 hi, lo split of x
// (rows*in floats), with TE_FLAG_BACKWARD_F16 the fp16 hi part of dy (rows*out/2 floats).
extern "C" int te_linear_forward(const float* x, const float* w, const float* bias, const float* e0, float* y, float* y2,
                                 float* scratch, int rows, int in_features, int out_features, int epi, unsigned flags,
                                 void* stream) {
    REQ(x && w && y && rows > 0 && in_features > 0 && out_features > 0, "te_linear_forward: bad argument");
    REQ((epi >= TE_EPI_STORE && epi <= TE_EPI_BIAS_ADD) || epi == TE_EPI_BIAS_QUICK_GELU,
        "te_linear_forward: epilogue must be STORE, BIAS, BIAS_GELU, BIAS_ADD or BIAS_QUICK_GELU");
    REQ(y2 || (epi != TE_EPI_BIAS_GELU && epi != TE_EPI_BIAS_ADD && epi != TE_EPI_BIAS_QUICK_GELU),
        "te_linear_forward: BIAS_GELU / BIAS_ADD / BIAS_QUICK_GELU need y2");
    REQ(e0 || epi != TE_EPI_BIAS_ADD, "te_linear_forward: BIAS_ADD needs e0");
    REQ(!(flags & ~(TE_FLAG_LINEAR_TENSOR_CORES | TE_FLAG_LINEAR_F16_SPLIT)), "te_linear_forward: unknown family flags");
    const bool tc = (flags & TE_FLAG_LINEAR_TENSOR_CORES) != 0, f16 = (flags & TE_FLAG_LINEAR_F16_SPLIT) != 0;
    REQ(!f16 || tc, "te_linear_forward: TE_FLAG_LINEAR_F16_SPLIT needs TE_FLAG_LINEAR_TENSOR_CORES");
    REQ(scratch || !tc, "te_linear_forward: the tensor-core families need scratch");
    if (f16 && !te_tc_fwd16_supported(rows, in_features, out_features, in_features))
        return te_util::no_fallback("te_linear_forward: the fp16-split kernel does not take this shape");
    if (tc && !te_tc_gemm3x_supported(rows, in_features, out_features, in_features))
        return te_util::no_fallback("te_linear_forward: the 3xTF32 kernel does not take this shape");
    cudaStream_t st = ST(stream);
    if (tc) TE_TRY(te_tc_prepare_weights(w, scratch, in_features, out_features, st));
    te_util::F16Split fs = {nullptr, nullptr, false, nullptr, nullptr};
    if (f16) {
        const TcScratch c = tc_scratch(scratch, 0, in_features, out_features, (long long)rows * in_features);
        fs.split = c.op; fs.scale = c.scale;
    }
    return te_util::linear_fwd_tc(tc ? scratch : nullptr, x, in_features, w, bias, y, y2, e0, rows, in_features, out_features,
                                  epi, st, &fs);
}

extern "C" int te_linear_backward(const float* dy, const float* w, const float* e0, float* dx, float* scratch, int rows,
                                  int in_features, int out_features, int epi, unsigned flags, void* stream) {
    REQ(dy && w && dx && rows > 0 && in_features > 0 && out_features > 0, "te_linear_backward: bad argument");
    REQ(epi == TE_EPI_STORE || epi == TE_EPI_GELU_BWD || epi == TE_EPI_QUICK_GELU_BWD,
        "te_linear_backward: epilogue must be STORE, GELU_BWD or QUICK_GELU_BWD");
    REQ(e0 || (epi != TE_EPI_GELU_BWD && epi != TE_EPI_QUICK_GELU_BWD), "te_linear_backward: GELU_BWD / QUICK_GELU_BWD need e0");
    REQ(!(flags & ~(TE_FLAG_LINEAR_TENSOR_CORES | TE_FLAG_BACKWARD_TF32 | TE_FLAG_BACKWARD_F16)),
        "te_linear_backward: unknown family flags");
    const bool tc = (flags & TE_FLAG_LINEAR_TENSOR_CORES) != 0, f16 = (flags & TE_FLAG_BACKWARD_F16) != 0;
    REQ(!(flags & (TE_FLAG_BACKWARD_TF32 | TE_FLAG_BACKWARD_F16)) || tc,
        "te_linear_backward: the single-pass families need TE_FLAG_LINEAR_TENSOR_CORES");
    REQ(scratch || !tc, "te_linear_backward: the tensor-core families need scratch");
    if (f16 && !te_tc_fwd16_supported(rows, out_features, in_features, out_features))
        return te_util::no_fallback("te_linear_backward: the single-pass fp16 kernel does not take this shape");
    if (tc && !te_tc_gemm3x_supported(rows, out_features, in_features, out_features))
        return te_util::no_fallback("te_linear_backward: the 3xTF32 / single-pass TF32 kernels do not take this shape");
    cudaStream_t st = ST(stream);
    if (tc) TE_TRY(te_tc_prepare_weights(w, scratch, in_features, out_features, st));
    te_util::F16Split fs = {nullptr, nullptr, false, nullptr, nullptr};
    if (f16) {
        const TcScratch c = tc_scratch(scratch, 0, in_features, out_features, (long long)rows * out_features / 2);
        fs.split = c.op; fs.scale = c.scale;
    }
    return te_util::linear_bwd_tc(tc ? scratch : nullptr, dy, w, dx, e0, rows, in_features, out_features, epi, st,
                                  (flags & TE_FLAG_BACKWARD_TF32) != 0, &fs);
}

extern "C" int te_layernorm_split(const float* x, const float* w, const float* b, float* y, float* mean, float* rstd, void* hi,
                                  void* lo, float* scale_inv, int rows, int D, float eps, void* stream) {
    REQ(x && w && b && y && hi && lo && scale_inv && rows > 0 && D > 0 && D % 4 == 0, "te_layernorm_split: bad argument");
    REQ(reinterpret_cast<char*>(lo) == reinterpret_cast<char*>(hi) + (long long)rows * D * 2,
        "te_layernorm_split: lo must follow hi ([hi | lo] in one buffer, as the kernels lay the split out)");
    return te_launch_layernorm_split(x, w, b, y, mean, rstd, rows, D, eps, reinterpret_cast<float*>(hi), scale_inv, ST(stream));
}

static bool al16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

extern "C" int te_tc_zplus_s(const float* x, const float* w, const float* bias, const float* y, const float* r, float* s,
                             void* s16, float* s16_scale, float* scratch, int rows, int in_features, int out_features,
                             unsigned flags, void* stream) {
    REQ(x && w && y && r && scratch && rows > 0 && in_features > 0 && out_features > 0, "te_tc_zplus_s: bad argument");
    REQ((s != nullptr) != (s16 != nullptr) && (!s16 || s16_scale), "te_tc_zplus_s: give either s or s16 + s16_scale");
    REQ(!(flags & ~TE_FLAG_ZPLUS_S1_BF16), "te_tc_zplus_s: only TE_FLAG_ZPLUS_S1_BF16 selects a variant");
    if (!te_tc_zplus_supported(rows, in_features, out_features, in_features))
        return te_util::no_fallback("te_tc_zplus_s: the tensor-core S kernel needs in / out multiples of 128");
    REQ(al16(x) && al16(y) && al16(r) && al16(scratch) && (!bias || al16(bias)) && (!s || al16(s)) && (!s16 || al16(s16)),
        "te_tc_zplus_s: operands must be 16-byte aligned");
    cudaStream_t st = ST(stream);
    const TcScratch c = tc_scratch(scratch, 0, in_features, out_features, 0);    // operand: bf16(|x|)
    TE_TRY(te_tc_prepare_weights(w, c.derived, in_features, out_features, st));
    return te_tc_zplus_s1(x, in_features, c.op, c.derived, r, out_features, y, out_features, bias, s, rows, in_features,
                          out_features, st, (flags & TE_FLAG_ZPLUS_S1_BF16) != 0, reinterpret_cast<float*>(s16), s16_scale);
}

extern "C" int te_tc_attention_nn(const float* A, long long lda, const float* B, long long ldb, int batch, int heads, int n,
                                  int dh, float* out, int ld_out, const float* E, float alpha, int epi, int single_pass,
                                  void* stream) {
    REQ(A && B && out && batch > 0 && heads > 0 && n > 0 && dh > 0, "te_tc_attention_nn: bad argument");
    REQ(epi >= TE_TC_ATTN_STORE && epi <= TE_TC_ATTN_SOFTMAX, "te_tc_attention_nn: unknown epilogue");
    REQ(E || epi == TE_TC_ATTN_STORE || epi == TE_TC_ATTN_SOFTMAX, "te_tc_attention_nn: MUL / SD need E");
    if (!te_tc_attn_supported(n, dh, lda, ldb, ld_out))
        return te_util::no_fallback("te_tc_attention_nn: the tensor-core kernel needs dh in {32, 64} and lda, ldb, ld_out multiples of 4");
    if (epi == TE_TC_ATTN_SOFTMAX && n > 256)
        return te_util::no_fallback("te_tc_attention_nn: the fused softmax needs every key in one tile (n <= 256)");
    if (single_pass && (epi == TE_TC_ATTN_SD || epi == TE_TC_ATTN_SOFTMAX))
        return te_util::no_fallback("te_tc_attention_nn: the single-pass kernel has the STORE / MUL epilogues only");
    REQ(ld_out >= ((n + 3) & ~3) && lda >= (long long)heads * dh && ldb >= (long long)heads * dh,
        "te_tc_attention_nn: ld_out < round_up(n, 4) or a row stride below heads * dh");
    REQ(al16(A) && al16(B) && al16(out) && (!E || al16(E)), "te_tc_attention_nn: operands must be 16-byte aligned");
    return te_tc_attn_nn(A, lda, B, ldb, batch, heads, n, dh, out, ld_out, E, alpha, epi, ST(stream), single_pass != 0);
}

extern "C" int te_tc_attention_nk(const float* map, int np, int amn, const float* X, long long ldx, int batch, int heads, int n,
                                  float* out, int ld_out, const float* E, float alpha, int epi, int single_pass, void* stream) {
    REQ(map && X && out && batch > 0 && heads > 0 && n > 0 && (amn == 0 || amn == 1), "te_tc_attention_nk: bad argument");
    REQ(epi == TE_TC_ATTN_STORE || epi == TE_TC_ATTN_MUL, "te_tc_attention_nk: epilogue must be STORE or MUL");
    REQ(E || epi == TE_TC_ATTN_STORE, "te_tc_attention_nk: MUL needs E");
    if (!te_tc_attn_nk_supported(n, 64, np, ldx, ld_out))
        return te_util::no_fallback("te_tc_attention_nk: the tensor-core kernel needs np, ldx, ld_out multiples of 4");
    REQ(np >= n && ldx >= 64LL * heads && ld_out >= 64 * heads, "te_tc_attention_nk: np < n or a row stride below heads * 64");
    REQ(al16(map) && al16(X) && al16(out) && (!E || al16(E)), "te_tc_attention_nk: operands must be 16-byte aligned");
    return te_tc_attn_nk(map, np, amn, X, ldx, batch, heads, n, out, ld_out, E, alpha, epi, ST(stream), single_pass != 0);
}

extern "C" int te_f16_block_split(const float* x, int rows, int cols, void* hi, void* lo, float* scale_inv, void* stream) {
    REQ(x && hi && lo && scale_inv && rows > 0 && cols > 0 && cols % 4 == 0, "te_f16_block_split: bad argument");
    REQ(reinterpret_cast<char*>(lo) == reinterpret_cast<char*>(hi) + (long long)rows * cols * 2,
        "te_f16_block_split: lo must follow hi ([hi | lo] in one buffer, as the kernels lay the split out)");
    return te_tc_blocksplit_f16(x, cols, rows, cols, reinterpret_cast<float*>(hi), scale_inv, ST(stream));
}

extern "C" int te_linear_relprop(const float* x, const float* w, const float* bias, const float* y, const float* r, float* out,
                                 float* scratch, int rows, int in_features, int out_features, float alpha, unsigned flags,
                                 void* stream) {
    REQ(x && w && r && out && scratch && rows > 0 && in_features > 0 && out_features > 0, "te_linear_relprop: bad argument");
    REQ(isfinite(alpha), "te_linear_relprop: alpha must be finite");
    const bool lrp = (flags & TE_FLAG_RULES_LRP) != 0;
    const float* derived = nullptr;
    float* xabs = nullptr;
    if ((flags & (lrp ? TE_FLAG_RULES_LRP_TC : TE_FLAG_ZPLUS_TENSOR_CORES)) &&
        te_tc_zplus_supported(rows, in_features, out_features, in_features)) {
        const TcScratch c = tc_scratch(scratch, (long long)rows * out_features, in_features, out_features, 0);   // operand: |x|
        TE_TRY(te_tc_prepare_weights(w, c.derived, in_features, out_features, ST(stream)));
        derived = c.derived;
        if (y) xabs = c.op;
    }
    // without y the z+ rule runs its two-pass form, to which the bf16 / fp16 variant flags do not apply
    return te_linear_rule_relprop(lrp, x, in_features, w, derived, r, out_features, out, scratch, rows, in_features, out_features,
                                  ST(stream), y, out_features, bias, y ? te_zplus_from_flags(flags) : ZplusVariant{}, 0, xabs,
                                  alpha);
}

extern "C" int te_add_relprop(const float* x1, const float* x2, const float* r, float* r1, float* r2, void* scratch,
                              int batch, long long per_sample, void* stream) {
    REQ(x1 && x2 && r && r1 && r2 && batch > 0 && per_sample > 0, "te_add_relprop: bad argument");
    return te_launch_add_relprop(x1, x2, r, r1, r2, reinterpret_cast<double*>(scratch), batch, per_sample, ST(stream));
}

extern "C" int te_clone_relprop(const float* x, const float* r1, const float* r2, const float* r3, float* out,
                                long long n, void* stream) {
    REQ(x && r1 && r2 && out && n > 0, "te_clone_relprop: bad argument");
    return te_launch_clone_relprop(x, r1, r2, r3, out, n, ST(stream));
}

extern "C" int te_index_select_relprop(const float* x, const float* r, float* out, int batch, int n, int d,
                                       void* stream) {
    REQ(x && r && out && batch > 0 && n > 0 && d > 0, "te_index_select_relprop: bad argument");
    return te_launch_index_select_relprop(x, r, nullptr, out, batch, n, d, ST(stream));
}

extern "C" int te_matmul_av_relprop(const float* p_, const float* v, const float* r, float* rp, float* rv,
                                    float* scratch, int bh, int n, int d, void* stream) {
    REQ(p_ && v && r && rp && rv && scratch && bh > 0 && n > 0 && d > 0 && d % 4 == 0, "te_matmul_av_relprop: bad argument");
    cudaStream_t st = ST(stream);
    const long long nn = (long long)n * n, nd = (long long)n * d;
    // Z = P V
    TeGemm g = g0(bh);
    g.A = p_; g.lda = n; g.sA1 = nn; g.B = v; g.ldb = d; g.sB1 = nd; g.C = scratch; g.ldc = d; g.sC1 = nd;
    g.M = n; g.N = d; g.K = n;
    TE_TRY(te_gemm_launch(g, TE_L_K, TE_L_MN, TE_XF_NONE, TE_EPI_STORE, st));
    // S = sd(R, Z)
    TE_TRY(te_launch_sd(r, scratch, scratch, (long long)bh * nd, st));
    // R_P = P * (S V^T)
    g = g0(bh);
    g.A = scratch; g.lda = d; g.sA1 = nd; g.B = v; g.ldb = d; g.sB1 = nd; g.C = rp; g.ldc = n; g.sC1 = nn;
    g.E0 = p_; g.lde0 = n; g.sE1 = nn; g.M = n; g.N = n; g.K = d;
    TE_TRY(te_gemm_launch(g, TE_L_K, TE_L_K, TE_XF_NONE, TE_EPI_MUL, st));
    // R_V = V * (P^T S)
    g = g0(bh);
    g.A = p_; g.lda = n; g.sA1 = nn; g.B = scratch; g.ldb = d; g.sB1 = nd; g.C = rv; g.ldc = d; g.sC1 = nd;
    g.E0 = v; g.lde0 = d; g.sE1 = nd; g.M = n; g.N = d; g.K = n;
    TE_TRY(te_gemm_launch(g, TE_L_MN, TE_L_MN, TE_XF_NONE, TE_EPI_MUL, st));
    return TE_OK;
}

extern "C" int te_matmul_qk_relprop(const float* q, const float* k, const float* r, float* rq, float* rk,
                                    float* scratch, int bh, int n, int d, void* stream) {
    REQ(q && k && r && rq && rk && scratch && bh > 0 && n > 0 && d > 0, "te_matmul_qk_relprop: bad argument");
    cudaStream_t st = ST(stream);
    const long long nn = (long long)n * n, nd = (long long)n * d;
    // S = sd(R, Q K^T)
    TeGemm g = g0(bh);
    g.A = q; g.lda = d; g.sA1 = nd; g.B = k; g.ldb = d; g.sB1 = nd; g.C = scratch; g.ldc = n; g.sC1 = nn;
    g.E0 = r; g.lde0 = n; g.sE1 = nn; g.M = n; g.N = n; g.K = d;
    TE_TRY(te_gemm_launch(g, TE_L_K, TE_L_K, TE_XF_NONE, TE_EPI_SD, st));
    // R_Q = Q * (S K)
    g = g0(bh);
    g.A = scratch; g.lda = n; g.sA1 = nn; g.B = k; g.ldb = d; g.sB1 = nd; g.C = rq; g.ldc = d; g.sC1 = nd;
    g.E0 = q; g.lde0 = d; g.sE1 = nd; g.M = n; g.N = d; g.K = n;
    TE_TRY(te_gemm_launch(g, TE_L_K, TE_L_MN, TE_XF_NONE, TE_EPI_MUL, st));
    // R_K = K * (S^T Q)
    g = g0(bh);
    g.A = scratch; g.lda = n; g.sA1 = nn; g.B = q; g.ldb = d; g.sB1 = nd; g.C = rk; g.ldc = d; g.sC1 = nd;
    g.E0 = k; g.lde0 = d; g.sE1 = nd; g.M = n; g.N = d; g.K = n;
    TE_TRY(te_gemm_launch(g, TE_L_MN, TE_L_MN, TE_XF_NONE, TE_EPI_MUL, st));
    return TE_OK;
}

static int g_cls_rows = 1;
bool te_engine_cls_rows() { return g_cls_rows != 0; }
void te_engine_set_cls_rows(int on) { g_cls_rows = on ? 1 : 0; }
static int g_gelu_split = -1;
bool te_engine_gelu_split() {
    if (g_gelu_split < 0) {
        const char* e = getenv("TE_B200_GELU_SPLIT");
        g_gelu_split = (e && e[0] == '0') ? 0 : 1;
    }
    return g_gelu_split != 0;
}
void te_engine_set_gelu_split(int on) { g_gelu_split = on ? 1 : 0; }

extern "C" int te_set_option(const char* name, int value) {
    REQ(name != nullptr, "te_set_option: null name");
    if (strcmp(name, "cls_row_top_block") == 0) { te_engine_set_cls_rows(value); return TE_OK; }
    if (strcmp(name, "gelu_split_fused") == 0) { te_engine_set_gelu_split(value); return TE_OK; }
    te_set_last_error("te_set_option: unknown option");
    return TE_ERR_ARG;
}

extern "C" int te_relevance_heatmap(const float* maps, int batch, int grid, int scale, float* out, void* stream) {
    REQ(maps && out && batch > 0 && grid > 0 && scale > 0, "te_relevance_heatmap: bad argument");
    return te_launch_relevance_heatmap(maps, out, batch, grid, scale, ST(stream));
}

// ---- head reductions of the secondary methods ------------------------------------------------------------
extern "C" int te_head_reduce(const float* a, const float* g, const float* head_w, int batch, int heads, int n, int ld,
                              int mode, float* out, void* stream) {
    REQ(a && out && batch > 0 && heads > 0 && n > 0 && ld >= n && mode >= 0 && mode <= 2, "te_head_reduce: bad argument");
    return te_launch_head_reduce(a, g, head_w, out, batch, heads, n, ld, mode, ST(stream));
}
extern "C" int te_head_region_mean(const float* g, int batch, int heads, int n, int ld, int r0, int r1, int c0, int c1,
                                   float* out, void* stream) {
    REQ(g && out && batch > 0 && heads > 0 && n > 0 && ld >= n, "te_head_region_mean: bad argument");
    return te_launch_head_region_mean(g, out, batch * heads, n, ld, r0, r1, c0, c1, ST(stream));
}

// ---- rollout -------------------------------------------------------------------------------------
static long long ro_align(long long bytes) { return ((bytes + 255) / 256) * 256; }

extern "C" long long te_rollout_workspace_bytes(int layers, int batch, int n) {
    if (layers <= 0 || batch <= 0 || n <= 0) return TE_ERR_ARG;
    const long long ld = (n + 3) & ~3;
    return ro_align((long long)layers * batch * n * ld * 4) + 2 * ro_align((long long)batch * n * ld * 4) +
           ro_align((long long)layers * batch * n * 4);
}

static int ro_carve(void* workspace, long long bytes, int layers, int batch, int n, float** mats, float** ja,
                    float** jb, int* ld, float** diag = nullptr) {
    REQ(workspace && (((uintptr_t)workspace) & 255u) == 0, "rollout: workspace null or not 256-byte aligned");
    if (te_rollout_workspace_bytes(layers, batch, n) > bytes) { te_set_last_error("rollout: workspace too small"); return TE_ERR_WORKSPACE; }
    *ld = (n + 3) & ~3;
    char* b = reinterpret_cast<char*>(workspace);
    *mats = reinterpret_cast<float*>(b);
    b += ro_align((long long)layers * batch * n * (*ld) * 4);
    *ja = reinterpret_cast<float*>(b);
    b += ro_align((long long)batch * n * (*ld) * 4);
    *jb = reinterpret_cast<float*>(b);
    b += ro_align((long long)batch * n * (*ld) * 4);
    if (diag) *diag = reinterpret_cast<float*>(b);
    return TE_OK;
}

// ---- first layer: Conv2d z^B rule / PatchEmbed.relprop (layers_ours.py:242-259, ViT_LRP.py:238-242) ----------------
extern "C" long long te_patch_embed_relprop_workspace_bytes(int batch, int in_chans, int img_size, int patch_size, int dim) {
    if (batch <= 0 || in_chans <= 0 || patch_size <= 0 || img_size % patch_size != 0 || dim <= 0) return TE_ERR_ARG;
    return te_patch_relprop_scratch_floats(batch, in_chans, img_size, patch_size, dim) * 4 + 256;
}
extern "C" int te_patch_embed_relprop(const float* images, const float* weight, const float* r, int batch, int in_chans,
                                      int img_size, int patch_size, int dim, float* r_pixels, float* r_sum, void* workspace,
                                      long long workspace_bytes, void* stream) {
    REQ(images && weight && r && (r_pixels || r_sum) && batch > 0, "te_patch_embed_relprop: bad argument");
    REQ(workspace && (((uintptr_t)workspace) & 255u) == 0, "te_patch_embed_relprop: workspace null or not 256-byte aligned");
    const long long need = te_patch_embed_relprop_workspace_bytes(batch, in_chans, img_size, patch_size, dim);
    if (need < 0) { te_set_last_error("te_patch_embed_relprop: bad shape"); return TE_ERR_ARG; }
    if (need > workspace_bytes) { te_set_last_error("te_patch_embed_relprop: workspace too small"); return TE_ERR_WORKSPACE; }
    const long long np = (long long)(img_size / patch_size) * (img_size / patch_size);
    return te_patch_relprop_run(images, weight, r, np * dim, batch, in_chans, img_size, patch_size, dim,
                                reinterpret_cast<float*>(workspace), r_pixels, r_sum, ST(stream));
}

extern "C" int te_attribution_rollout(const float* grad, const float* cam, int layers, int batch, int heads, int n,
                                      int ld, int start_layer, int normalize, unsigned flags, float* joint,
                                      float* row0, void* workspace, long long workspace_bytes, void* stream) {
    REQ(grad && cam && layers > 0 && batch > 0 && heads > 0 && n > 0 && ld >= n, "te_attribution_rollout: bad argument");
    float *mats, *ja, *jb, *diag;
    int ldw;
    TE_TRY(ro_carve(workspace, workspace_bytes, layers, batch, n, &mats, &ja, &jb, &ldw, &diag));
    return te_rollout_layers(grad, cam, (long long)batch * heads * n * ld, layers, batch, heads, n, ld, ldw, start_layer,
                             normalize, flags, mats, ja, jb, joint, row0, /*first=*/0, /*bert_fix=*/0, ST(stream), diag);
}

extern "C" int te_compute_rollout_attention(const float* mats_in, int layers, int batch, int n, int start_layer,
                                            int normalize, float* joint, void* workspace, long long workspace_bytes,
                                            void* stream) {
    REQ(mats_in && joint && layers > 0 && batch > 0 && n > 0 && start_layer >= 0 && start_layer < layers,
        "te_compute_rollout_attention: bad argument");
    float *mats, *ja, *jb;
    int ldw;
    TE_TRY(ro_carve(workspace, workspace_bytes, layers, batch, n, &mats, &ja, &jb, &ldw));
    cudaStream_t st = ST(stream);
    TE_TRY(te_launch_prep_mats(mats_in, mats, (long long)layers * batch * n, n, n, ldw, normalize, st));
    const float* res = nullptr;
    TE_TRY(te_rollout_chain(mats, layers, batch, n, ldw, start_layer, ja, jb, &res, st));
    if (cudaMemcpy2DAsync(joint, sizeof(float) * n, res, sizeof(float) * ldw, sizeof(float) * n, (size_t)batch * n,
                          cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
        te_set_last_error("te_compute_rollout_attention: copy failed");
        return TE_ERR_CUDA;
    }
    return TE_OK;
}
