// Host-side helpers shared by the model engines: kernel selection from the engine flags, GEMM parameter builders over
// packed activations, the attention-block backward / relprop sequences, and workspace / weight-table boilerplate.
#pragma once
#include <string.h>
#include <string>
#include <vector>

#include "../../include/te_b200.h"
#include "te_gemm.cuh"
#include "te_gemm_tc.h"
#include "te_kernels.h"
#include "te_zplus.h"

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

// a requested kernel family that does not take the shape / epilogue is an error (TE_ERR_UNSUPPORTED), not a fall-back to the
// next family — what the diagnostic entry points need
static inline int no_fallback(const char* msg) {
    te_set_last_error(msg);
    return TE_ERR_UNSUPPORTED;
}

// tensor-core (3xTF32) variants when the derived weight copies are supplied and the shape qualifies
// fp16-split forward Linear (TE_FLAG_LINEAR_F16_SPLIT, te_tc_wgmma.cu): where the block-scaled split of the input lives
// (M*in floats + M*ceil(in/128) floats), whether its producer already filled it (ready: te_launch_layernorm_split or the previous
// GEMM's GELU epilogue), and where the GELU epilogue puts the split of y2 for the next Linear (may be NULL)
struct F16Split { float* split; float* scale; bool ready; float* split_out; float* scale_out; };
static inline int linear_fwd_tc(const float* dw, const float* x, int lda, const float* w, const float* bias, float* y,
                                float* y2, const float* e0, long long M, int in, int out, int epi, cudaStream_t st,
                                const F16Split* fs = nullptr) {
    const bool f16 = dw && fs && fs->split;
    const bool act = epi == TE_EPI_BIAS_GELU || epi == TE_EPI_BIAS_QUICK_GELU;     // epilogues that may emit the split of y2
    if (f16 && epi != TE_EPI_GELU_BWD && epi != TE_EPI_QUICK_GELU_BWD && te_tc_fwd16_supported(M, in, out, lda))
        return te_tc_linear_fwd16(fs->ready ? nullptr : x, lda, fs->split, fs->scale, dw, in, out, bias, y, y2, e0, M, epi, st,
                                  act ? fs->split_out : nullptr, act ? fs->scale_out : nullptr);
    if (dw && te_tc_gemm3x_supported(M, in, out, lda))
        return te_tc_linear_fwd(x, lda, dw, in, out, bias, y, y2, e0, M, epi, st);      // epilogue ids coincide
    return linear_fwd(x, lda, w, bias, y, y2, e0, M, in, out, epi, st);
}
// tf32: single-pass TF32 wgmma kernel (TE_FLAG_BACKWARD_TF32) instead of the 3xTF32 split
// fs: hi-only split scratch of dy (M*out/2 floats + M*ceil(out/128)) -> single-pass fp16 kernel (TE_FLAG_BACKWARD_F16)
static inline int linear_bwd_tc(const float* dw, const float* dy, const float* w, float* dx, const float* e0, long long M,
                                int in, int out, int epi, cudaStream_t st, bool tf32 = false, const F16Split* fs = nullptr) {
    const bool f16 = dw && fs && fs->split,
               single_epi = epi == TE_EPI_STORE || epi == TE_EPI_GELU_BWD || epi == TE_EPI_QUICK_GELU_BWD;
    if (f16 && single_epi && te_tc_fwd16_supported(M, out, in, out))
        return te_tc_linear_bwd16(fs->ready ? nullptr : dy, out, fs->split, fs->scale, dw, in, out, dx, e0, M, epi, st);
    if (dw && tf32 && single_epi && te_tc_gemm3x_supported(M, out, in, out))
        return te_tc_linear_bwd_tf32(dy, out, dw, in, out, dx, e0, M, epi, st);
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

// ---- kernel selection ------------------------------------------------------------------------------------------------
// What the engine flags select for one te_*_forward / te_*_attribute call.  The model-specific modes (TE_FLAG_GRADIENTS_ONLY,
// TE_FLAG_RELPROP_TO_INPUT) are read where they are used.
struct Select {
    const float* lbase;   // derived weights of the forward / backward Linears (TE_FLAG_LINEAR_TENSOR_CORES), else NULL
    const float* dbase;   // derived weights of the Linear relevance rules: the z+ rules (TE_FLAG_ZPLUS_TENSOR_CORES), or with
                          // TE_FLAG_RULES_LRP the layers_lrp rule (TE_FLAG_RULES_LRP_TC); else NULL
    bool atc;             // attention contractions on tensor cores (TE_FLAG_ATTN_TENSOR_CORES)
    bool btf;             // single-pass TF32 backward Linears and attention gradients (TE_FLAG_BACKWARD_TF32)
    bool rtf;             // single-pass TF32 relevance-side attention contractions (TE_FLAG_RELPROP_TF32)
    bool f16;             // fp16-split forward Linears requested (TE_FLAG_LINEAR_F16_SPLIT); f16_forward() checks the shapes
    F16Split bfs;         // single-pass fp16 backward Linears (TE_FLAG_BACKWARD_F16): hi-only split of dy; split NULL = off
    bool lrp;             // rule library of modules/layers_lrp.py instead of layers_ours (TE_FLAG_RULES_LRP)
    ZplusVariant zv;      // bf16 / fp16 variants of the tensor-core z+ rule
    int low;              // lowest block the relprop must reach
    bool seeded;          // the backward starts from the workspace's similarity seed (TE_FLAG_SIMILARITY_SEED)
};
// A workspace region an engine lends to a kernel while the region is idle, with the floats it holds.
struct Lent { float* ptr; long long floats; };
// The hi-only fp16 split of dy [rows, out] (TE_FLAG_BACKWARD_F16): rows*out/2 floats of fp16 values, rows*ceil(out/128)
// floats of block scales.
static inline long long bwd_split_floats(long long rows, int out) { return rows * out / 2; }
static inline long long bwd_scale_floats(long long rows, int out) { return rows * ((out + 127) / 128); }

// fn: prefix of the error message.  zplus: the call runs the z+ rules, so TE_FLAG_ZPLUS_TENSOR_CORES needs `derived` as well.
// bwd_split / bwd_scale: regions idle during the class-gradient backward, lent for the fp16 split of dy; rows / widest_out:
// the rows and the widest output of the backward Linears.  A lent region smaller than that use is an error
// (TE_ERR_WORKSPACE), never a write past its end into the next region.
static inline int decode_flags(Select& s, const char* fn, unsigned flags, const float* derived, int start_layer, bool zplus,
                               Lent bwd_split = {nullptr, 0}, Lent bwd_scale = {nullptr, 0}, long long rows = 0,
                               int widest_out = 0) {
    // the tensor-core flag of the Linear rule of the selected rule library: layers_ours (z+) or layers_lrp
    const bool lrp = (flags & TE_FLAG_RULES_LRP) != 0;
    if ((flags & TE_FLAG_SIMILARITY_SEED) && !(flags & TE_FLAG_ATTN_GRAD_ROLLOUT)) {
        te_set_last_error((std::string(fn) + ": TE_FLAG_SIMILARITY_SEED needs TE_FLAG_ATTN_GRAD_ROLLOUT (no LRP starts from a "
                           "similarity gradient)").c_str());
        return TE_ERR_ARG;
    }
    const unsigned rule_tc = lrp ? (flags & TE_FLAG_RULES_LRP_TC) : (flags & TE_FLAG_ZPLUS_TENSOR_CORES);
    if (((flags & (TE_FLAG_LINEAR_TENSOR_CORES | (zplus ? TE_FLAG_ZPLUS_TENSOR_CORES : 0u))) || (zplus && rule_tc)) && !derived) {
        te_set_last_error((std::string(fn) + ": tensor-core flags need the derived weight buffer").c_str());
        return TE_ERR_ARG;
    }
    s.lbase = (flags & TE_FLAG_LINEAR_TENSOR_CORES) ? derived : nullptr;
    s.dbase = rule_tc ? derived : nullptr;
    s.atc = (flags & TE_FLAG_ATTN_TENSOR_CORES) != 0;
    s.btf = (flags & TE_FLAG_BACKWARD_TF32) != 0;
    s.rtf = (flags & TE_FLAG_RELPROP_TF32) != 0;
    s.f16 = s.lbase && (flags & TE_FLAG_LINEAR_F16_SPLIT);
    const bool bf16 = s.lbase && (flags & TE_FLAG_BACKWARD_F16) && bwd_split.ptr;
    if (bf16 && (bwd_split.floats < bwd_split_floats(rows, widest_out) || bwd_scale.floats < bwd_scale_floats(rows, widest_out))) {
        te_set_last_error((std::string(fn) + ": the region lent for the fp16 split of the backward gradients is too small").c_str());
        return TE_ERR_WORKSPACE;
    }
    s.bfs = {bf16 ? bwd_split.ptr : nullptr, bwd_scale.ptr, false, nullptr, nullptr};
    s.lrp = lrp;
    s.zv = te_zplus_from_flags(flags);
    s.low = (flags & (TE_FLAG_KEEP_ALL_CAMS | TE_FLAG_RELPROP_TO_INPUT)) ? 0 : start_layer;
    s.seeded = (flags & TE_FLAG_SIMILARITY_SEED) != 0;
    return TE_OK;
}

// TE_FLAG_ATTN_GRAD_ROLLOUT runs no relprop: the modes that stop before it or carry it further, and the alpha-beta rule,
// have nothing to act on, so asking for them together is an error rather than a silently ignored bit
static inline int check_grad_rollout(const char* fn, unsigned flags, float alpha) {
    if (!(flags & TE_FLAG_ATTN_GRAD_ROLLOUT)) return TE_OK;
    const char* clash = (flags & TE_FLAG_GRADIENTS_ONLY) ? "TE_FLAG_GRADIENTS_ONLY"
                      : (flags & TE_FLAG_KEEP_ALL_CAMS) ? "TE_FLAG_KEEP_ALL_CAMS"
                      : (flags & TE_FLAG_RELPROP_TO_INPUT) ? "TE_FLAG_RELPROP_TO_INPUT" : nullptr;
    if (clash) {
        te_set_last_error((std::string(fn) + ": TE_FLAG_ATTN_GRAD_ROLLOUT does not combine with " + clash).c_str());
        return TE_ERR_ARG;
    }
    if (alpha != 1.f) {
        te_set_last_error((std::string(fn) + ": TE_FLAG_ATTN_GRAD_ROLLOUT runs no relprop, alpha must be 1").c_str());
        return TE_ERR_ARG;
    }
    return TE_OK;
}

// fp16-split forward Linears (te_tc_wgmma.cu) of a block with D-wide inputs and an F-wide GELU layer: the block-scaled split
// of the D-wide inputs lives in a (+ scales a_scale), that of the GELU output in b (+ b_scale), buffers the engine lends while
// they are idle.  LayerNorm emits the split of what it produces (qkv and fc1 inputs); the attention context goes through the
// pre-pass; the fc1 GELU epilogue emits the split for fc2 with te_engine_gelu_split(), else fc2 pre-passes.  When `on` is
// false every descriptor has split == NULL, which selects the 3xTF32 kernel.
struct F16Forward { bool on; F16Split qkv, proj, fc1, fc2; };
static inline F16Forward f16_forward(const Select& s, long long M, int D, int F, float* a, float* a_scale, float* b,
                                     float* b_scale) {
    F16Forward f = {};
    f.on = s.f16 && F >= D && te_tc_fwd16_supported(M, D, 3 * D, D) && te_tc_fwd16_supported(M, D, D, D) &&
           te_tc_fwd16_supported(M, D, F, D) && te_tc_fwd16_supported(M, F, D, F);
    if (!f.on) return f;
    const bool gsf = te_engine_gelu_split();
    f.qkv = {a, a_scale, true, nullptr, nullptr};
    f.proj = {a, a_scale, false, nullptr, nullptr};
    f.fc1 = {a, a_scale, true, gsf ? b : nullptr, gsf ? b_scale : nullptr};
    f.fc2 = {b, b_scale, gsf, nullptr, nullptr};
    return f;
}

// ---- attention block: qkv = packed [B*N, 3D] q | k | v, P = probabilities [B, H, N, NP] ------------------------------------
// class-gradient backward from dctx [B*N, D]: G = dctx v^T (the gradient at P); unless g_only, dV = P^T dctx,
// dS = softmax_bwd(P, G) and dQ = dS k, dK = dS^T q into dqkv [B*N, 3D]
static inline int attn_block_bwd(const Select& s, int B, int H, int N, int NP, int dh, const float* qkv, const float* P,
                                 const float* dctx, float* G, float* dS, float* dqkv, float scale, bool g_only, cudaStream_t st) {
    const int D = H * dh;
    TE_TRY(attn_nn(s.atc, B, H, N, NP, dh, dctx, D, qkv + 2 * D, 3 * D, G, nullptr, 1.f, TE_EPI_STORE, st, s.btf));
    if (g_only) return TE_OK;
    TE_TRY(attn_nk(s.atc, B, H, N, NP, dh, P, 1, dctx, D, dqkv + 2 * D, 3 * D, nullptr, 1.f, TE_EPI_STORE, st, s.btf));
    TE_TRY(te_launch_softmax_bwd(P, G, dS, (long long)B * H * N, N, NP, scale, st));
    TE_TRY(attn_nk(s.atc, B, H, N, NP, dh, dS, 0, qkv + D, 3 * D, dqkv, 3 * D, nullptr, 1.f, TE_EPI_STORE, st, s.btf));
    return attn_nk(s.atc, B, H, N, NP, dh, dS, 1, qkv, 3 * D, dqkv + D, 3 * D, nullptr, 1.f, TE_EPI_STORE, st, s.btf);
}

// relprop, upper half, from the relevance Rctx [B*N, D] of the attention context ctx = P v: matmul2 rule S = sd(Rctx, ctx)
// (the saved ctx is the reference's bit-identical recomputation), attn_cam = (P * (S v^T)) / 2; unless cam_only,
// R_v = (v * (P^T S)) / 2 into Rqkv [B*N, 3D]
static inline int attn_relprop_pv(const Select& s, int B, int H, int N, int NP, int dh, const float* qkv, const float* P,
                                  const float* Rctx, const float* ctx, float* S, float* cam, float* Rqkv, bool cam_only,
                                  cudaStream_t st) {
    const int D = H * dh;
    TE_TRY(te_launch_sd(Rctx, ctx, S, (long long)B * N * D, st));
    TE_TRY(attn_nn(s.atc, B, H, N, NP, dh, S, D, qkv + 2 * D, 3 * D, cam, P, 0.5f, TE_EPI_MUL, st, s.rtf));
    if (cam_only) return TE_OK;
    return attn_nk(s.atc, B, H, N, NP, dh, P, 1, S, D, Rqkv + 2 * D, 3 * D, qkv + 2 * D, 0.5f, TE_EPI_MUL, st, s.rtf);
}
// relprop, lower half: matmul1 rule on the unscaled Z = q k^T with the relevance E of the scores, S1 = sd(E, Z) in the
// scratch S1 [B, H, N, NP]; R_q = (q * (S1 k)) / 2 and R_k = (k * (S1^T q)) / 2 into Rqkv
static inline int attn_relprop_qk(const Select& s, int B, int H, int N, int NP, int dh, const float* qkv, const float* E,
                                  float* S1, float* Rqkv, cudaStream_t st) {
    const int D = H * dh;
    TE_TRY(attn_nn(s.atc, B, H, N, NP, dh, qkv, 3 * D, qkv + D, 3 * D, S1, E, 1.f, TE_EPI_SD, st));
    TE_TRY(attn_nk(s.atc, B, H, N, NP, dh, S1, 0, qkv + D, 3 * D, Rqkv, 3 * D, qkv, 0.5f, TE_EPI_MUL, st, s.rtf));
    return attn_nk(s.atc, B, H, N, NP, dh, S1, 1, qkv, 3 * D, Rqkv + D, 3 * D, qkv + D, 0.5f, TE_EPI_MUL, st, s.rtf);
}

// ---- workspace and weight-table boilerplate of the engines ------------------------------------------------------------------
// bump allocator over a workspace: 256-byte aligned slices; with base == NULL it only measures (off = bytes needed)
struct Bump {
    char* base;
    long long off = 0;
    float* operator()(long long nfloat) {
        float* p = base ? reinterpret_cast<float*>(base + off) : nullptr;
        off += ((nfloat * 4 + 255) / 256) * 256;
        return p;
    }
};

// the workspace checks of te_*_forward / te_*_attribute: make_dims() validates the config (and sets its own error), carve()
// lays the workspace out and returns the bytes it needs; eng prefixes the error messages
template <class MakeDims, class Carve>
static inline int check_ws(const char* eng, int batch, void* workspace, long long bytes, MakeDims make_dims, Carve carve) {
    const std::string e(eng);
    if (batch <= 0 || !workspace) { te_set_last_error((e + ": batch <= 0 or null workspace").c_str()); return TE_ERR_ARG; }
    if (!make_dims()) return TE_ERR_ARG;
    if (((uintptr_t)workspace & 255u) != 0) { te_set_last_error((e + ": workspace must be 256-byte aligned").c_str()); return TE_ERR_ARG; }
    if (carve() > bytes) { te_set_last_error((e + ": workspace too small").c_str()); return TE_ERR_WORKSPACE; }
    return TE_OK;
}

// te_*_tensor: writes a 4-d view (pointer, dims, strides) of a workspace tensor
struct View {
    float** ptr; long long* dims; long long* strides;
    int operator()(float* p, long long d0, long long d1, long long d2, long long d3, long long s0, long long s1, long long s2,
                   long long s3) const {
        *ptr = p; dims[0] = d0; dims[1] = d1; dims[2] = d2; dims[3] = d3;
        strides[0] = s0; strides[1] = s1; strides[2] = s2; strides[3] = s3;
        return TE_OK;
    }
};

// flat weight buffer: one entry per tensor, then a sentinel whose offset is the total; empty for an invalid config
struct WEntry { std::string name; long long numel; long long offset; };
using WTable = std::vector<WEntry>;
static inline int wt_count(const WTable& t) { return t.empty() ? TE_ERR_ARG : (int)t.size() - 1; }
static inline bool wt_has(const WTable& t, int i) { return i >= 0 && i + 1 < (int)t.size(); }
static inline const char* wt_name(const WTable& t, int i) {
    static thread_local std::string s;
    if (!wt_has(t, i)) return nullptr;
    s = t[i].name;
    return s.c_str();
}
static inline long long wt_numel(const WTable& t, int i) { return wt_has(t, i) ? t[i].numel : TE_ERR_ARG; }
static inline long long wt_offset(const WTable& t, int i) { return wt_has(t, i) ? t[i].offset : TE_ERR_ARG; }
static inline long long wt_total(const WTable& t) { return t.empty() ? TE_ERR_ARG : t.back().offset; }

}  // namespace te_util
