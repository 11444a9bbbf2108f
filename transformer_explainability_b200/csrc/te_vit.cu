// ViT / DeiT transformer-attribution engine: forward with saved activations, activation-gradient
// backward (attention gradients only — no dW), LRP relprop through every block, aggregation and
// rollout.  Host-side orchestration of the kernels in te_gemm.cu / te_elementwise.cu /
// te_rollout.cu; O(1) launches per block per BATCH, never per sample.
//
// Reference wiring: baselines/ViT/ViT_LRP.py (forward :305-322, relprop :324-369, Block :196-213,
// Attention :132-177, Mlp :61-74), baselines/ViT/ViT_explanation_generator.py:25-41.
#include <string.h>

#include <algorithm>

#include "../../include/te_b200.h"
#include "te_engine_util.h"
#include "te_kernels.h"
#include "te_rollout.h"
#include "te_zplus.h"
#include "te_gemm_tc.h"

namespace {

constexpr int kMaxDepth = 64;

struct Dims {
    int B, N, NP, D, H, dh, F, C, L, P, img, Cin, npatch, prefix, KP;
    long long M;
};

static bool make_dims(const te_vit_config* c, int B, Dims& d) {
    if (!c || c->depth <= 0 || c->depth > kMaxDepth || c->heads <= 0 || c->dim % c->heads != 0 || c->dim % 4 != 0 ||
        c->mlp_dim % 4 != 0 || c->patch_size <= 0 || c->img_size % c->patch_size != 0 || c->num_classes <= 0) {
        te_set_last_error("te_vit: invalid config");
        return false;
    }
    if ((c->pre_norm != 0 && c->pre_norm != 1) || (c->act != TE_VIT_ACT_GELU && c->act != TE_VIT_ACT_QUICK_GELU)) {
        te_set_last_error("te_vit: pre_norm must be 0 or 1 and act TE_VIT_ACT_GELU or TE_VIT_ACT_QUICK_GELU");
        return false;
    }
    d.B = B; d.D = c->dim; d.H = c->heads; d.dh = c->dim / c->heads; d.F = c->mlp_dim; d.C = c->num_classes;
    d.L = c->depth; d.P = c->patch_size; d.img = c->img_size; d.Cin = c->in_chans;
    d.npatch = (c->img_size / c->patch_size) * (c->img_size / c->patch_size);
    d.prefix = c->distilled ? 2 : 1;
    d.N = d.npatch + d.prefix;
    d.NP = (d.N + 3) & ~3;
    d.KP = d.Cin * d.P * d.P;
    d.M = (long long)B * d.N;
    if (d.dh % 4 != 0) { te_set_last_error("te_vit: head_dim % 4 != 0"); return false; }
    return true;
}

// ---- flat weight buffer ------------------------------------------------------------------------
using te_util::WTable;

static WTable weight_table(const te_vit_config* c) {
    Dims d;
    WTable t;
    if (!make_dims(c, 1, d)) return t;
    long long off = 0;
    auto add = [&](const std::string& n, long long numel) {
        t.push_back({n, numel, off});
        off += (numel + 31) & ~31LL;
    };
    add("patch_embed.proj.weight", (long long)d.D * d.KP);
    add("patch_embed.proj.bias", d.D);
    add("cls_token", d.D);
    if (c->distilled) add("dist_token", d.D);
    add("pos_embed", (long long)d.N * d.D);
    if (c->pre_norm) {
        add("norm_pre.weight", d.D);
        add("norm_pre.bias", d.D);
    }
    for (int i = 0; i < d.L; ++i) {
        const std::string p = "blocks." + std::to_string(i) + ".";
        add(p + "norm1.weight", d.D);
        add(p + "norm1.bias", d.D);
        add(p + "attn.qkv.weight", 3LL * d.D * d.D);
        add(p + "attn.qkv.bias", 3LL * d.D);
        add(p + "attn.proj.weight", (long long)d.D * d.D);
        add(p + "attn.proj.bias", d.D);
        add(p + "norm2.weight", d.D);
        add(p + "norm2.bias", d.D);
        add(p + "mlp.fc1.weight", (long long)d.F * d.D);
        add(p + "mlp.fc1.bias", d.F);
        add(p + "mlp.fc2.weight", (long long)d.D * d.F);
        add(p + "mlp.fc2.bias", d.D);
    }
    add("norm.weight", d.D);
    add("norm.bias", d.D);
    add("head.weight", (long long)d.C * d.D);
    add("head.bias", d.C);
    if (c->distilled) {
        add("head_dist.weight", (long long)d.C * d.D);
        add("head_dist.bias", d.C);
    }
    t.push_back({"", 0, off});   // sentinel: total
    return t;
}

struct BlockW {
    const float *n1w, *n1b, *qkvw, *qkvb, *projw, *projb, *n2w, *n2b, *fc1w, *fc1b, *fc2w, *fc2b;
};
struct Weights {
    const float *patchw, *patchb, *cls, *dist, *pos, *prew, *preb, *normw, *normb, *headw, *headb, *headdw, *headdb;
    BlockW blk[kMaxDepth];
};

static void bind_weights(const te_vit_config* c, const float* base, Weights& w) {
    const WTable t = weight_table(c);
    size_t i = 0;
    auto next = [&]() { return base + t[i++].offset; };
    w.patchw = next(); w.patchb = next(); w.cls = next();
    w.dist = c->distilled ? next() : nullptr;
    w.pos = next();
    w.prew = c->pre_norm ? next() : nullptr;
    w.preb = c->pre_norm ? next() : nullptr;
    for (int l = 0; l < c->depth; ++l) {
        BlockW& b = w.blk[l];
        b.n1w = next(); b.n1b = next(); b.qkvw = next(); b.qkvb = next(); b.projw = next(); b.projb = next();
        b.n2w = next(); b.n2b = next(); b.fc1w = next(); b.fc1b = next(); b.fc2w = next(); b.fc2b = next();
    }
    w.normw = next(); w.normb = next(); w.headw = next(); w.headb = next();
    w.headdw = c->distilled ? next() : nullptr;
    w.headdb = c->distilled ? next() : nullptr;
}

// ---- derived (tensor-core) weight copies: per block qkv | proj | fc1 | fc2, 4 copies each ---------
struct DerivedW { const float *qkv, *proj, *fc1, *fc2; };
static long long derived_block_floats(const Dims& d) {
    return te_tc_derived_floats(d.D, 3 * d.D) + te_tc_derived_floats(d.D, d.D) + te_tc_derived_floats(d.D, d.F) +
           te_tc_derived_floats(d.F, d.D);
}
static DerivedW bind_derived(const Dims& d, const float* base, int l) {
    DerivedW w = {nullptr, nullptr, nullptr, nullptr};
    if (!base) return w;
    const float* p = base + (long long)l * derived_block_floats(d);
    w.qkv = p;  p += te_tc_derived_floats(d.D, 3 * d.D);
    w.proj = p; p += te_tc_derived_floats(d.D, d.D);
    w.fc1 = p;  p += te_tc_derived_floats(d.D, d.F);
    w.fc2 = p;
    return w;
}

// ---- workspace ---------------------------------------------------------------------------------
struct LayerAct {
    float *x_in, *xn1, *mean1, *rstd1, *qkv, *P, *ctx, *attn_out, *x_mid, *xn2, *mean2, *rstd2, *h, *g, *mlp_out,
        *G, *cam;
};
struct Workspace {
    LayerAct layer[kMaxDepth];
    float *x_last, *xf, *logits, *logits2, *seed, *dpool, *rhead0, *rhead1, *shead;
    float *tD[4], *tF[2], *t3D[2], *tA;
    long long nF[2];                  // floats of tF[0], tF[1]
    float *mats, *joint[2];
    float* pix;                       // scratch of the first-layer (pixel) relprop, method="full"
    double* addpart;
    int* index_tmp;
    long long bytes;
};

static void carve(const Dims& d, char* base, Workspace& ws) {
    te_util::Bump take{base};
    const long long MD = d.M * d.D, MF = d.M * d.F, M3D = d.M * 3LL * d.D;
    const long long AT = (long long)d.B * d.H * d.N * d.NP;
    for (int l = 0; l < d.L; ++l) {
        LayerAct& a = ws.layer[l];
        a.x_in = take(MD); a.xn1 = take(MD); a.mean1 = take(d.M); a.rstd1 = take(d.M);
        a.qkv = take(M3D); a.P = take(AT); a.ctx = take(MD); a.attn_out = take(MD); a.x_mid = take(MD);
        a.xn2 = take(MD); a.mean2 = take(d.M); a.rstd2 = take(d.M); a.h = take(MF); a.g = take(MF);
        a.mlp_out = take(MD); a.G = take(AT); a.cam = take(AT);
    }
    ws.x_last = take(MD); ws.xf = take(MD);
    ws.logits = take((long long)d.B * d.C); ws.logits2 = take((long long)d.B * d.C);
    ws.seed = take((long long)d.B * d.C); ws.shead = take((long long)d.B * d.C);
    ws.dpool = take((long long)d.B * d.D); ws.rhead0 = take((long long)d.B * d.D);
    ws.rhead1 = take((long long)d.B * d.D);
    for (int i = 0; i < 4; ++i) ws.tD[i] = take(MD);
    // tF[0], tF[1] are sized by their largest use, not by F alone (with mlp_ratio < 1.5 a use is wider than M*F):
    //   tF[0]: dF / RF [M, F]; the im2col patches; the |x| scratch [M, D] of the qkv z+ rule
    //   tF[1]: SF [M, F] (and the |x| scratch of the fc2 z+ rule); the GELU-output fp16 split [M, F] of the forward; the
    //          hi-only fp16 split of dy of every backward Linear, widest for qkv [M, 3D / 2]
    const long long patches = (long long)d.B * d.npatch * d.KP;
    ws.nF[0] = std::max({MF, patches, MD});
    ws.nF[1] = std::max(MF, te_util::bwd_split_floats(d.M, 3 * d.D));
    ws.tF[0] = take(ws.nF[0]);
    ws.tF[1] = take(ws.nF[1]);
    ws.t3D[0] = take(M3D); ws.t3D[1] = take(M3D);
    ws.tA = take(AT);
    ws.mats = take((long long)d.L * d.B * d.N * d.NP);
    ws.joint[0] = take((long long)d.B * d.N * d.NP);
    ws.joint[1] = take((long long)d.B * d.N * d.NP);
    ws.pix = take(te_patch_relprop_scratch_floats(d.B, d.Cin, d.img, d.P, d.D));
    ws.addpart = reinterpret_cast<double*>(take((long long)d.B * TE_ADD_SPLIT * 3 * 2));
    ws.index_tmp = reinterpret_cast<int*>(take(d.B));
    ws.bytes = take.off;
}

// ---- GEMM parameter helpers (shared builders live in te_engine_util.h) ----------------------------
using te_util::linear_bwd;
using te_util::linear_fwd;

static int check_ws(const te_vit_config* cfg, int batch, void* workspace, long long bytes, Dims& d, Workspace& ws) {
    return te_util::check_ws("te_vit", batch, workspace, bytes, [&] { return make_dims(cfg, batch, d); },
                             [&] { carve(d, reinterpret_cast<char*>(workspace), ws); return ws.bytes; });
}

}  // namespace

// ================================================================================================
// public: weights / workspace description
// ================================================================================================
extern "C" int te_vit_num_weights(const te_vit_config* cfg) { return te_util::wt_count(weight_table(cfg)); }
extern "C" const char* te_vit_weight_name(const te_vit_config* cfg, int i) { return te_util::wt_name(weight_table(cfg), i); }
extern "C" long long te_vit_weight_numel(const te_vit_config* cfg, int i) { return te_util::wt_numel(weight_table(cfg), i); }
extern "C" long long te_vit_weight_offset(const te_vit_config* cfg, int i) { return te_util::wt_offset(weight_table(cfg), i); }
extern "C" long long te_vit_weight_total(const te_vit_config* cfg) { return te_util::wt_total(weight_table(cfg)); }
extern "C" long long te_vit_workspace_bytes(const te_vit_config* cfg, int batch) {
    Dims d;
    if (batch <= 0 || !make_dims(cfg, batch, d)) return TE_ERR_ARG;
    Workspace ws;
    carve(d, nullptr, ws);
    return ws.bytes;
}

// ================================================================================================
// forward   (ViT_LRP.py:305-322)
// ================================================================================================
extern "C" int te_vit_forward(const te_vit_config* cfg, const float* weights, const float* derived, const float* images,
                              int batch, unsigned flags, float* logits, void* workspace, long long workspace_bytes,
                              void* stream) {
    Dims d; Workspace ws;
    TE_TRY(check_ws(cfg, batch, workspace, workspace_bytes, d, ws));
    if (!weights || !images) { te_set_last_error("te_vit_forward: null pointer"); return TE_ERR_ARG; }
    te_util::Select sel;
    TE_TRY(te_util::decode_flags(sel, "te_vit_forward", flags, derived, 0, false));
    // fp16-split forward Linears: split of the D-wide inputs in tD[1] (+ scales tD[0]), of the GELU output in tF[1] (+ scales
    // tD[2]); all idle until the backward pass
    const te_util::F16Forward f16 = te_util::f16_forward(sel, d.M, d.D, d.F, ws.tD[1], ws.tD[0], ws.tF[1], ws.tD[2]);
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    auto layernorm = [&](const float* x, const float* g, const float* b, float* y, float* mean, float* rstd) {
        return f16.on ? te_launch_layernorm_split(x, g, b, y, mean, rstd, d.M, d.D, cfg->eps_block, f16.qkv.split, f16.qkv.scale, st)
                      : te_launch_layernorm(x, g, b, y, mean, rstd, d.M, d.D, cfg->eps_block, st);
    };
    Weights w;
    bind_weights(cfg, weights, w);
    const float scale = 1.0f / sqrtf((float)d.dh);

    // patch embedding: conv k=s=P  ==  im2col + GEMM   (PatchEmbed.forward :230-236)
    float* patches = ws.tF[0];
    float* patch_out = ws.tD[3];
    TE_TRY(te_launch_im2col(images, patches, d.B, d.Cin, d.img, d.img, d.P, st));
    TE_TRY(linear_fwd(patches, d.KP, w.patchw, w.patchb, patch_out, nullptr, nullptr, (long long)d.B * d.npatch, d.KP,
                      d.D, TE_EPI_BIAS, st));
    // pre-norm towers (CLIP ln_pre, timm norm_pre): the assembled tokens pass through a LayerNorm into block 0.  Its input lives
    // in tD[2], idle until block 0's fc1 epilogue; nothing reads it later (the gradients stop at block start_layer's
    // attention, and the relevance rules take the LayerNorm as the identity)
    float* tokens = cfg->pre_norm ? ws.tD[2] : ws.layer[0].x_in;
    TE_TRY(te_launch_assemble_tokens(patch_out, w.cls, w.dist, w.pos, tokens, d.B, d.N, d.D, d.prefix, st));
    if (cfg->pre_norm)
        TE_TRY(te_launch_layernorm(tokens, w.prew, w.preb, ws.layer[0].x_in, nullptr, nullptr, d.M, d.D, cfg->eps_block, st));
    const int fc1_epi = cfg->act == TE_VIT_ACT_QUICK_GELU ? TE_EPI_BIAS_QUICK_GELU : TE_EPI_BIAS_GELU;

    for (int l = 0; l < d.L; ++l) {
        LayerAct& a = ws.layer[l];
        const BlockW& bw = w.blk[l];
        float* x_next = (l + 1 < d.L) ? ws.layer[l + 1].x_in : ws.x_last;
        const DerivedW lw = bind_derived(d, sel.lbase, l);
        TE_TRY(layernorm(a.x_in, bw.n1w, bw.n1b, a.xn1, a.mean1, a.rstd1));
        TE_TRY(te_util::linear_fwd_tc(lw.qkv, a.xn1, d.D, bw.qkvw, bw.qkvb, a.qkv, nullptr, nullptr, d.M, d.D, 3 * d.D,
                                      TE_EPI_BIAS, st, &f16.qkv));
        // dots = q k^T * scale ; attn = softmax(dots)        (:139-141)
        TE_TRY(te_util::attn_probs(sel.atc, d.B, d.H, d.N, d.NP, d.dh, a.qkv, 3 * d.D, a.qkv + d.D, 3 * d.D, a.P, scale, st));
        // out = attn v -> 'b h n d -> b n (h d)'              (:147-148)
        TE_TRY(te_util::attn_nk(sel.atc, d.B, d.H, d.N, d.NP, d.dh, a.P, 0, a.qkv + 2 * d.D, 3 * d.D, a.ctx, d.D, nullptr, 1.f,
                                TE_EPI_STORE, st));
        // proj + residual add1                                  (:150, :198)
        TE_TRY(te_util::linear_fwd_tc(lw.proj, a.ctx, d.D, bw.projw, bw.projb, a.attn_out, a.x_mid, a.x_in, d.M, d.D, d.D,
                                      TE_EPI_BIAS_ADD, st, &f16.proj));
        TE_TRY(layernorm(a.x_mid, bw.n2w, bw.n2b, a.xn2, a.mean2, a.rstd2));
        TE_TRY(te_util::linear_fwd_tc(lw.fc1, a.xn2, d.D, bw.fc1w, bw.fc1b, a.h, a.g, nullptr, d.M, d.D, d.F, fc1_epi, st,
                                      &f16.fc1));
        TE_TRY(te_util::linear_fwd_tc(lw.fc2, a.g, d.F, bw.fc2w, bw.fc2b, a.mlp_out, x_next, a.x_mid, d.M, d.F, d.D,
                                      TE_EPI_BIAS_ADD, st, &f16.fc2));
    }
    // final norm, pool token 0 (and 1), head(s)                (:318-321)
    TE_TRY(te_launch_layernorm(ws.x_last, w.normw, w.normb, ws.xf, nullptr, nullptr, d.M, d.D, cfg->eps_final, st));
    TE_TRY(linear_fwd(ws.xf, d.N * d.D, w.headw, w.headb, ws.logits, nullptr, nullptr, d.B, d.D, d.C, TE_EPI_BIAS, st));
    if (cfg->distilled) {
        TE_TRY(linear_fwd(ws.xf + d.D, d.N * d.D, w.headdw, w.headdb, ws.logits2, nullptr, nullptr, d.B, d.D, d.C,
                          TE_EPI_BIAS, st));
        TE_TRY(te_launch_average2(ws.logits, ws.logits2, ws.logits, (long long)d.B * d.C, st));
    }
    if (logits) {
        if (cudaMemcpyAsync(logits, ws.logits, sizeof(float) * d.B * d.C, cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
            te_set_last_error("te_vit_forward: logits copy failed");
            return TE_ERR_CUDA;
        }
    }
    return TE_OK;
}

// ================================================================================================
// attribute = class-gradient backward + relprop + aggregation + rollout
// ================================================================================================
extern "C" long long te_vit_derived_total(const te_vit_config* cfg) {
    Dims d;
    if (!make_dims(cfg, 1, d)) return TE_ERR_ARG;
    return (long long)d.L * derived_block_floats(d);
}

extern "C" int te_vit_prepare_derived(const te_vit_config* cfg, const float* weights, float* derived, void* stream) {
    Dims d;
    if (!make_dims(cfg, 1, d)) return TE_ERR_ARG;
    if (!weights || !derived) { te_set_last_error("te_vit_prepare_derived: null pointer"); return TE_ERR_ARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    Weights w;
    bind_weights(cfg, weights, w);
    for (int l = 0; l < d.L; ++l) {
        const DerivedW dw = bind_derived(d, derived, l);
        TE_TRY(te_tc_prepare_weights(w.blk[l].qkvw, const_cast<float*>(dw.qkv), d.D, 3 * d.D, st));
        TE_TRY(te_tc_prepare_weights(w.blk[l].projw, const_cast<float*>(dw.proj), d.D, d.D, st));
        TE_TRY(te_tc_prepare_weights(w.blk[l].fc1w, const_cast<float*>(dw.fc1), d.D, d.F, st));
        TE_TRY(te_tc_prepare_weights(w.blk[l].fc2w, const_cast<float*>(dw.fc2), d.F, d.D, st));
    }
    return TE_OK;
}

extern "C" int te_vit_attribute(const te_vit_config* cfg, const float* weights, const float* derived, int batch, int* index,
                                int start_layer, float alpha, unsigned flags, float* maps, void* workspace,
                                long long workspace_bytes, void* stream) {
    Dims d; Workspace ws;
    TE_TRY(check_ws(cfg, batch, workspace, workspace_bytes, d, ws));
    if (!isfinite(alpha)) { te_set_last_error("te_vit_attribute: alpha must be finite"); return TE_ERR_ARG; }
    TE_TRY(te_util::check_grad_rollout("te_vit_attribute", flags, alpha));
    const bool grad_rollout = (flags & TE_FLAG_ATTN_GRAD_ROLLOUT) != 0;
    if (!weights || !index || (!maps && !(flags & TE_FLAG_GRADIENTS_ONLY))) { te_set_last_error("te_vit_attribute: null pointer"); return TE_ERR_ARG; }
    if (start_layer < 0 || start_layer >= d.L) { te_set_last_error("te_vit_attribute: start_layer out of range"); return TE_ERR_ARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    Weights w;
    bind_weights(cfg, weights, w);
    const float scale = 1.0f / sqrtf((float)d.dh);
    const long long MD = d.M * d.D, M3D = d.M * 3LL * d.D;
    // fp16 backward split of dy in tF[1], block scales in t3D[1] (idle until the relprop)
    te_util::Select sel;
    TE_TRY(te_util::decode_flags(sel, "te_vit_attribute", flags, derived, start_layer, !grad_rollout, {ws.tF[1], ws.nF[1]},
                                 {ws.t3D[1], M3D}, d.M, std::max(3 * d.D, d.F)));

    // ---- class index and seeds  (ViT_explanation_generator.py:28-35); TE_FLAG_SIMILARITY_SEED: te_vit_similarity_seed's ----
    if (!sel.seeded) {
        TE_TRY(te_launch_argmax(ws.logits, index, d.B, d.C, /*only_negative=*/1, st));
        const float seedv = cfg->distilled ? 0.5f : 1.0f;   // averaged heads: each gets half of the seed
        TE_TRY(te_launch_onehot(index, ws.seed, d.B, d.C, seedv, st));
    }
    const int fc2_bwd_epi = cfg->act == TE_VIT_ACT_QUICK_GELU ? TE_EPI_QUICK_GELU_BWD : TE_EPI_GELU_BWD;

    // ---- backward: d logit_c / d attn_l for every block  (what :145's hook captures) -------------
    float* dxa = ws.tD[0]; float* dxb = ws.tD[1]; float* dctx = ws.tD[2]; float* dxn = ws.tD[3];
    float* dF = ws.tF[0]; float* dqkv = ws.t3D[0]; float* dS = ws.tA;
    TE_TRY(te_launch_fill(dxa, 0.f, MD, st));
    {
        // d pooled = seed * W_head ; final LayerNorm backward touches only the pooled token rows
        TE_TRY(linear_bwd(ws.seed, w.headw, ws.dpool, nullptr, d.B, d.D, d.C, TE_EPI_STORE, st));
        TE_TRY(te_launch_layernorm_bwd_strided(ws.dpool, d.D, ws.x_last, (long long)d.N * d.D, w.normw, cfg->eps_final,
                                               dxa, (long long)d.N * d.D, d.B, d.D, st));
        if (cfg->distilled) {
            TE_TRY(linear_bwd(ws.seed, w.headdw, ws.dpool, nullptr, d.B, d.D, d.C, TE_EPI_STORE, st));
            TE_TRY(te_launch_layernorm_bwd_strided(ws.dpool, d.D, ws.x_last + d.D, (long long)d.N * d.D, w.normw,
                                                   cfg->eps_final, dxa + d.D, (long long)d.N * d.D, d.B, d.D, st));
        }
    }
    for (int l = d.L - 1; l >= start_layer; --l) {
        LayerAct& a = ws.layer[l];
        const BlockW& bw = w.blk[l];
        const DerivedW lw = bind_derived(d, sel.lbase, l);
        // mlp branch
        TE_TRY(te_util::linear_bwd_tc(lw.fc2, dxa, bw.fc2w, dF, a.h, d.M, d.F, d.D, fc2_bwd_epi, st, sel.btf, &sel.bfs));
        TE_TRY(te_util::linear_bwd_tc(lw.fc1, dF, bw.fc1w, dxn, nullptr, d.M, d.D, d.F, TE_EPI_STORE, st, sel.btf, &sel.bfs));
        TE_TRY(te_launch_layernorm_bwd(dxn, a.x_mid, bw.n2w, a.mean2, a.rstd2, dxa, dxb, d.M, d.D, st));
        // attention branch
        TE_TRY(te_util::linear_bwd_tc(lw.proj, dxb, bw.projw, dctx, nullptr, d.M, d.D, d.D, TE_EPI_STORE, st, sel.btf, &sel.bfs));
        const bool last = (l == start_layer);                                       // lower gradients are never read
        TE_TRY(te_util::attn_block_bwd(sel, d.B, d.H, d.N, d.NP, d.dh, a.qkv, a.P, dctx, a.G, dS, dqkv, scale, last, st));
        if (last) break;
        TE_TRY(te_util::linear_bwd_tc(lw.qkv, dqkv, bw.qkvw, dxn, nullptr, d.M, d.D, 3 * d.D, TE_EPI_STORE, st, sel.btf, &sel.bfs));
        TE_TRY(te_launch_layernorm_bwd(dxn, a.x_in, bw.n1w, a.mean1, a.rstd1, dxb, dxa, d.M, d.D, st));
    }

    if (flags & TE_FLAG_GRADIENTS_ONLY) return TE_OK;      // attention-GradCAM baseline: gradients are all it reads
    // P and G of a layer are carved side by side in every layer's slice, so one layer stride serves both operands
    const long long layer_stride = d.L > 1 ? (long long)(ws.layer[1].G - ws.layer[0].G) : 0;
    if (grad_rollout)       // gradient-weighted attention rollout: mean_h relu(G * P) + I chained from start_layer, no relprop
        return te_rollout_layers(ws.layer[0].G, ws.layer[0].P, layer_stride, d.L, d.B, d.H, d.N, d.NP, d.NP, start_layer,
                                 /*normalize=*/0, flags, ws.mats, ws.joint[0], ws.joint[1], nullptr, maps, d.prefix,
                                 /*bert_fix=*/0, st);

    // ---- relprop  (VisionTransformer.relprop :324-331) --------------------------------------------
    float* R = ws.tD[0]; float* R1 = ws.tD[1]; float* R2 = ws.tD[2]; float* R3 = ws.tD[3];
    float* RF = ws.tF[0]; float* SF = ws.tF[1]; float* S = ws.t3D[0]; float* Rqkv = ws.t3D[1]; float* S1 = ws.tA;
    // head.relprop (z+), pool.relprop (IndexSelect), norm.relprop (identity)
    // Linear rule / Add rule of the selected rule library (layers_ours, or layers_lrp with TE_FLAG_RULES_LRP; the derived
    // weights are then set only with TE_FLAG_RULES_LRP_TC); alpha != 1: the alpha-beta Linear rule of either library
    auto addrule = [&](const float* x1, const float* x2, const float* r, float* r1, float* r2) -> int {
        return te_launch_add_relprop(x1, x2, r, r1, r2, sel.lrp ? nullptr : ws.addpart, d.B, (long long)d.N * d.D, st);
    };
    TE_TRY(te_linear_rule_relprop(sel.lrp, ws.xf, (long long)d.N * d.D, w.headw, nullptr, ws.seed, d.C, ws.rhead0, ws.shead, d.B,
                                  d.D, d.C, st, nullptr, 0, nullptr, sel.zv, 0, nullptr, alpha));
    if (cfg->distilled)
        TE_TRY(te_linear_rule_relprop(sel.lrp, ws.xf + d.D, (long long)d.N * d.D, w.headdw, nullptr, ws.seed, d.C, ws.rhead1,
                                      ws.shead, d.B, d.D, d.C, st, nullptr, 0, nullptr, sel.zv, 0, nullptr, alpha));
    TE_TRY(te_launch_index_select_relprop(ws.xf, ws.rhead0, cfg->distilled ? ws.rhead1 : nullptr, R, d.B, d.N, d.D, st));

    for (int l = d.L - 1; l >= sel.low; --l) {
        LayerAct& a = ws.layer[l];
        const BlockW& bw = w.blk[l];
        const DerivedW dw = bind_derived(d, sel.dbase, l);
        // Block.relprop :203-213
        // In the TOP block the relevance that enters is non-zero only in the pooled token's row (IndexSelect.relprop, a7),
        // and every rule down to the proj rule is row-wise: Add / Clone map a zero row to a zero row, the z+ rule computes
        // each output row from the same input row.  So the three z+ rules of the top block run on the B pooled rows only
        // (row stride N*D / N*F) — exact (SURVEY.md 8a "structural savings"), bit-identical rows, 1/N of the work.
        const bool top = (l == d.L - 1) && !cfg->distilled && !sel.lrp && te_engine_cls_rows();
        const long long zr = top ? d.B : d.M;                          // rows the z+ rules of this block touch
        const long long sD = top ? (long long)d.N * d.D : d.D, sF = top ? (long long)d.N * d.F : d.F;
        TE_TRY(addrule(a.x_mid, a.mlp_out, R, R1, R2));                                                            // add2
        TE_TRY(te_linear_rule_relprop(sel.lrp, a.g, sF, bw.fc2w, dw.fc2, R2, sD, RF, S, zr, d.F, d.D, st, a.mlp_out, sD, bw.fc2b,
                                      sel.zv, sF, SF, alpha));                                                    // fc2 ; GELU id
        TE_TRY(te_linear_rule_relprop(sel.lrp, a.xn2, sD, bw.fc1w, dw.fc1, RF, sF, R2, SF, zr, d.D, d.F, st, a.h, sF, bw.fc1b,
                                      sel.zv, sD, S, alpha));                                                     // fc1 ; norm2 id
        TE_TRY(te_launch_clone_relprop(a.x_mid, R1, R2, nullptr, R, MD, st));                                      // clone2
        TE_TRY(addrule(a.x_in, a.attn_out, R, R1, R2));                                                            // add1
        // Attention.relprop :154-177
        if (top) TE_TRY(te_launch_fill(R3, 0.f, MD, st));                                   // rows the strided rule does not write
        TE_TRY(te_linear_rule_relprop(sel.lrp, a.ctx, sD, bw.projw, dw.proj, R2, sD, R3, S, zr, d.D, d.D, st, a.attn_out, sD,
                                      bw.projb, sel.zv, sD, S + MD, alpha));                                      // proj
        // matmul2 rule -> attn_cam (:160-165), cam_v ; matmul1 rule -> cam_q, cam_k (:170-173)
        const bool last = (l == sel.low && !(flags & TE_FLAG_RELPROP_TO_INPUT));      // nothing below attn_cam is consumed
        TE_TRY(te_util::attn_relprop_pv(sel, d.B, d.H, d.N, d.NP, d.dh, a.qkv, a.P, R3, a.ctx, S, a.cam, Rqkv, last, st));
        if (last) break;
        TE_TRY(te_util::attn_relprop_qk(sel, d.B, d.H, d.N, d.NP, d.dh, a.qkv, a.cam, S1, Rqkv, st));
        TE_TRY(te_linear_rule_relprop(sel.lrp, a.xn1, d.D, bw.qkvw, dw.qkv, Rqkv, 3 * d.D, R2, S, d.M, d.D, 3 * d.D, st, a.qkv,
                                      3 * d.D, bw.qkvb, sel.zv, 0, RF, alpha));                                   // qkv ; norm1 id
        TE_TRY(te_launch_clone_relprop(a.x_in, R1, R2, nullptr, R, MD, st));                                       // clone1
    }

    // ---- aggregation + rollout  (:357-368) ---------------------------------------------------------
    TE_TRY(te_rollout_layers(ws.layer[0].G, ws.layer[0].cam, layer_stride, d.L, d.B, d.H, d.N, d.NP, d.NP,
                             start_layer, /*normalize=*/0, flags, ws.mats, ws.joint[0], ws.joint[1], nullptr, maps,
                             d.prefix, /*bert_fix=*/0, st));
    return TE_OK;
}

// ================================================================================================
// method="full": relevance of every input pixel   (ViT_LRP.py:337-343)
//   (cam, _) = self.add.relprop(cam) ; cam = cam[:, 1:] ; cam = self.patch_embed.relprop(cam) ; cam.sum(dim=1)
// Precondition: te_vit_forward + te_vit_attribute(flags | TE_FLAG_RELPROP_TO_INPUT) on this workspace and these images.
// ================================================================================================
extern "C" int te_vit_relprop_pixels(const te_vit_config* cfg, const float* weights, const float* images, int batch,
                                     unsigned flags, float* pixel_maps, float* pixel_relevance, void* workspace,
                                     long long workspace_bytes, void* stream) {
    Dims d; Workspace ws;
    TE_TRY(check_ws(cfg, batch, workspace, workspace_bytes, d, ws));
    if (!weights || !images || (!pixel_maps && !pixel_relevance)) { te_set_last_error("te_vit_relprop_pixels: null pointer"); return TE_ERR_ARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    Weights w;
    bind_weights(cfg, weights, w);
    float* R = ws.tD[0];                       // relevance at the encoder input (clone1 of block 0)
    float* tokens = ws.tD[1];                  // cat(cls[,dist], patch_embed(x)): the first operand of self.add (:311)
    float* Rtok = ws.tD[2];
    float* patches = ws.tF[0];
    float* patch_out = ws.tD[3];
    TE_TRY(te_launch_im2col(images, patches, d.B, d.Cin, d.img, d.img, d.P, st));
    TE_TRY(linear_fwd(patches, d.KP, w.patchw, w.patchb, patch_out, nullptr, nullptr, (long long)d.B * d.npatch, d.KP,
                      d.D, TE_EPI_BIAS, st));
    TE_TRY(te_launch_assemble_tokens(patch_out, w.cls, w.dist, nullptr, tokens, d.B, d.N, d.D, d.prefix, st));
    // self.add.relprop: x2 = pos_embed, shared by every sample; only the tokens' share is consumed
    TE_TRY(te_launch_add_relprop_strided(tokens, w.pos, 0, R, Rtok, nullptr, (flags & TE_FLAG_RULES_LRP) ? nullptr : ws.addpart,
                                         d.B, (long long)d.N * d.D, st));
    // cam[:, 1:] -> PatchEmbed.relprop (:238-242) -> Conv2d z^B rule -> sum over channels
    return te_patch_relprop_run(images, w.patchw, Rtok + (long long)d.prefix * d.D, (long long)d.N * d.D, d.B, d.Cin, d.img,
                                d.P, d.D, ws.pix, pixel_relevance, pixel_maps, st);
}

// ================================================================================================
// CLIP image-text similarity and its gradient, the seed of te_vit_attribute(TE_FLAG_SIMILARITY_SEED)
// ================================================================================================
extern "C" int te_vit_similarity_seed(const te_vit_config* cfg, int batch, const float* text, float logit_scale, float* similarity,
                                      void* workspace, long long workspace_bytes, void* stream) {
    Dims d; Workspace ws;
    TE_TRY(check_ws(cfg, batch, workspace, workspace_bytes, d, ws));
    if (!text) { te_set_last_error("te_vit_similarity_seed: null pointer"); return TE_ERR_ARG; }
    if (cfg->distilled) { te_set_last_error("te_vit_similarity_seed: a distilled model has two heads, not one embedding"); return TE_ERR_ARG; }
    if (!isfinite(logit_scale)) { te_set_last_error("te_vit_similarity_seed: logit_scale must be finite"); return TE_ERR_ARG; }
    return te_launch_similarity_seed(ws.logits, text, logit_scale, similarity, ws.seed, d.B, d.C,
                                     reinterpret_cast<cudaStream_t>(stream));
}

extern "C" int te_vit_explain(const te_vit_config* cfg, const float* weights, const float* derived, const float* images,
                              int batch, int* index, int start_layer, unsigned flags, float* maps, float* logits,
                              void* workspace, long long workspace_bytes, void* stream) {
    if (flags & TE_FLAG_SIMILARITY_SEED) {      // the forward here would leave no seed: te_vit_similarity_seed runs between
        te_set_last_error("te_vit_explain: TE_FLAG_SIMILARITY_SEED needs te_vit_forward, te_vit_similarity_seed, te_vit_attribute");
        return TE_ERR_ARG;
    }
    TE_TRY(te_vit_forward(cfg, weights, derived, images, batch, flags, logits, workspace, workspace_bytes, stream));
    return te_vit_attribute(cfg, weights, derived, batch, index, start_layer, 1.f, flags, maps, workspace, workspace_bytes,
                            stream);
}

extern "C" int te_vit_tensor(const te_vit_config* cfg, int batch, void* workspace, const char* name, int layer,
                             float** ptr, long long dims[4], long long strides[4]) {
    Dims d; Workspace ws;
    if (!workspace || !name || !ptr) return TE_ERR_ARG;
    if (batch <= 0 || !make_dims(cfg, batch, d)) return TE_ERR_ARG;
    carve(d, reinterpret_cast<char*>(workspace), ws);
    const std::string n(name);
    const te_util::View set{ptr, dims, strides};
    if (n == "logits") return set(ws.logits, d.B, d.C, 1, 1, d.C, 1, 1, 1);
    if (n == "relevance_in") return set(ws.tD[0], d.B, d.N, d.D, 1, (long long)d.N * d.D, d.D, 1, 1);
    if (n == "rollout_mats") return set(ws.mats, d.L, d.B, d.N, d.N, (long long)d.B * d.N * d.NP, (long long)d.N * d.NP, d.NP, 1);
    const long long ND = (long long)d.N * d.D, NF = (long long)d.N * d.F;
    if (n == "x_last") return set(ws.x_last, d.B, d.N, d.D, 1, ND, d.D, 1, 1);
    if (n == "x_final_norm") return set(ws.xf, d.B, d.N, d.D, 1, ND, d.D, 1, 1);
    // scratch of the last attribute() call (debug / diagnostics): tmp_d0..3 [B,N,D], tmp_f0..1 [B,N,F], tmp_3d0..1 [B,N,3D]
    if (n.rfind("tmp_d", 0) == 0 && n.size() == 6 && n[5] >= '0' && n[5] <= '3')
        return set(ws.tD[n[5] - '0'], d.B, d.N, d.D, 1, (long long)d.N * d.D, d.D, 1, 1);
    if (n.rfind("tmp_f", 0) == 0 && n.size() == 6 && n[5] >= '0' && n[5] <= '1')
        return set(ws.tF[n[5] - '0'], d.B, d.N, d.F, 1, (long long)d.N * d.F, d.F, 1, 1);
    if (n.rfind("tmp_3d", 0) == 0 && n.size() == 7 && n[6] >= '0' && n[6] <= '1')
        return set(ws.t3D[n[6] - '0'], d.B, d.N, 3LL * d.D, 1, (long long)d.N * 3 * d.D, 3LL * d.D, 1, 1);
    if (layer < 0 || layer >= d.L) { te_set_last_error("te_vit_tensor: layer out of range"); return TE_ERR_ARG; }
    LayerAct& a = ws.layer[layer];
    const long long hs = (long long)d.N * d.NP, bs = hs * d.H;
    if (n == "attn") return set(a.P, d.B, d.H, d.N, d.N, bs, hs, d.NP, 1);
    if (n == "attn_grad") return set(a.G, d.B, d.H, d.N, d.N, bs, hs, d.NP, 1);
    if (n == "attn_cam") return set(a.cam, d.B, d.H, d.N, d.N, bs, hs, d.NP, 1);
    if (n == "qkv") return set(a.qkv, d.B, d.N, 3LL * d.D, 1, (long long)d.N * 3 * d.D, 3LL * d.D, 1, 1);
    if (n == "x_in") return set(a.x_in, d.B, d.N, d.D, 1, (long long)d.N * d.D, d.D, 1, 1);
    if (n == "ctx") return set(a.ctx, d.B, d.N, d.D, 1, (long long)d.N * d.D, d.D, 1, 1);
    // the rest of the saved forward activations of the block (views only: test / diagnostic taps)
    float* rowD = n == "xn1" ? a.xn1 : n == "attn_out" ? a.attn_out : n == "x_mid" ? a.x_mid : n == "xn2" ? a.xn2
                : n == "mlp_out" ? a.mlp_out : nullptr;
    if (rowD) return set(rowD, d.B, d.N, d.D, 1, ND, d.D, 1, 1);
    float* rowF = n == "h" ? a.h : n == "g" ? a.g : nullptr;
    if (rowF) return set(rowF, d.B, d.N, d.F, 1, NF, d.F, 1, 1);
    float* row1 = n == "mean1" ? a.mean1 : n == "rstd1" ? a.rstd1 : n == "mean2" ? a.mean2 : n == "rstd2" ? a.rstd2 : nullptr;
    if (row1) return set(row1, d.B, d.N, 1, 1, d.N, 1, 1, 1);
    te_set_last_error("te_vit_tensor: unknown tensor name");
    return TE_ERR_ARG;
}
