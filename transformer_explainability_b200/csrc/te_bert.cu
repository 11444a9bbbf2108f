// BERT (post-LN encoder + pooler + classifier) transformer-attribution engine.
//
// The same engine runs the RoBERTa / XLM-RoBERTa and DistilBERT sequence classifiers (te_bert_config.arch): their
// encoder layer is this one, only the embedding (position ids, token-type table, order of the sum) and the head
// (classifier.dense / out_proj, or pre_classifier -> ReLU -> classifier) differ, see include/te_b200.h.
//
// Reference wiring: BERT_explainability/modules/BERT/BERT.py (BertEmbeddings :61-85, BertSelfAttention :307-409,
// BertSelfOutput :420-434, BertIntermediate :446-456, BertOutput :467-487, BertLayer :498-530, BertPooler :169-190,
// BertModel.relprop :645-651), BertForSequenceClassification.py:23-88, ExplanationGenerator.py:7-59.
// The additive attention mask (1-mask)*-10000 and head_mask = None are transformers==3.5.1 behaviour
// (un-vendored dependency; call sites BERT.py:598,616) restated here.
//
// q/k/v Linears are packed into one [3D, D] weight so that the forward is one GEMM and the per-head slices are
// addressed in place exactly like the ViT engine; their three z+ rules stay separate (Clone(3) needs them apart).
#include <string.h>

#include <algorithm>

#include "../../include/te_b200.h"
#include "te_engine_util.h"
#include "te_gemm_tc.h"
#include "te_kernels.h"
#include "te_rollout.h"
#include "te_zplus.h"

using namespace te_util;

namespace {

constexpr int kMaxDepth = 64;

struct Dims {
    int B, N, NP, D, H, dh, F, C, L, V, P, T, arch, pad;
    long long M;
    float eps;
};

static bool make_dims(const te_bert_config* c, int B, int S, Dims& d) {
    if (!c || c->layers <= 0 || c->layers > kMaxDepth || c->heads <= 0 || c->hidden % c->heads != 0 || c->hidden % 8 != 0 ||
        c->intermediate % 4 != 0 || c->num_labels <= 0 || c->vocab_size <= 0 || c->max_position <= 0) {
        te_set_last_error("te_bert: invalid config");
        return false;
    }
    if (c->arch != TE_BERT_ARCH_BERT && c->arch != TE_BERT_ARCH_ROBERTA && c->arch != TE_BERT_ARCH_DISTILBERT) {
        te_set_last_error("te_bert: unknown arch (TE_BERT_ARCH_BERT, _ROBERTA or _DISTILBERT)");
        return false;
    }
    if (c->arch == TE_BERT_ARCH_DISTILBERT ? c->type_vocab != 0 : c->type_vocab <= 0) {
        te_set_last_error(c->arch == TE_BERT_ARCH_DISTILBERT ? "te_bert: DistilBERT has no token-type table (type_vocab must be 0)"
                                                             : "te_bert: invalid config (type_vocab must be positive)");
        return false;
    }
    if (c->arch == TE_BERT_ARCH_ROBERTA && (c->pad_token_id < 0 || c->pad_token_id >= c->vocab_size)) {
        te_set_last_error("te_bert: RoBERTa pad_token_id outside [0, vocab_size)");
        return false;
    }
    // RoBERTa positions run pad + 1 .. pad + S: the table needs S + pad + 1 rows
    const long long max_seq = c->arch == TE_BERT_ARCH_ROBERTA ? (long long)c->max_position - c->pad_token_id - 1
                                                              : c->max_position;
    if (S <= 0 || S > max_seq) {
        te_set_last_error(c->arch == TE_BERT_ARCH_ROBERTA
                              ? "te_bert: sequence length out of range (RoBERTa: seq + pad_token_id + 1 <= max_position)"
                              : "te_bert: sequence length out of range");
        return false;
    }
    d.B = B; d.N = S; d.NP = (S + 3) & ~3; d.D = c->hidden; d.H = c->heads; d.dh = c->hidden / c->heads;
    d.F = c->intermediate; d.C = c->num_labels; d.L = c->layers; d.V = c->vocab_size; d.P = c->max_position;
    d.T = c->type_vocab; d.M = (long long)B * S; d.eps = c->layer_norm_eps;
    d.arch = c->arch; d.pad = c->pad_token_id;
    if (d.dh % 4 != 0) { te_set_last_error("te_bert: head_dim % 4 != 0"); return false; }
    return true;
}

// ---- flat weight buffer (HF state_dict keys) -------------------------------------------------------
static WTable weight_table(const te_bert_config* c) {
    WTable t;
    Dims d;
    if (!make_dims(c, 1, 1, d)) return t;
    long long off = 0;
    auto add = [&](const std::string& n, long long numel, bool pad = true) {
        t.push_back({n, numel, off});
        off += pad ? ((numel + 31) & ~31LL) : numel;
    };
    // per family: the state_dict prefix, the layer's module names (in the order bind_weights reads them), the head
    const bool distil = d.arch == TE_BERT_ARCH_DISTILBERT;
    const std::string M = distil ? "distilbert." : d.arch == TE_BERT_ARCH_ROBERTA ? "roberta." : "bert.";
    // q, k, v, attention output dense, its LayerNorm, intermediate dense, output dense, its LayerNorm
    static const char* const kBertLayer[8] = {"attention.self.query", "attention.self.key", "attention.self.value",
                                              "attention.output.dense", "attention.output.LayerNorm",
                                              "intermediate.dense", "output.dense", "output.LayerNorm"};
    static const char* const kDistilLayer[8] = {"attention.q_lin", "attention.k_lin", "attention.v_lin",
                                                "attention.out_lin", "sa_layer_norm", "ffn.lin1", "ffn.lin2",
                                                "output_layer_norm"};
    const char* const* n = distil ? kDistilLayer : kBertLayer;
    const std::string E = M + "embeddings.";
    add(E + "word_embeddings.weight", (long long)d.V * d.D);
    add(E + "position_embeddings.weight", (long long)d.P * d.D);
    if (!distil) add(E + "token_type_embeddings.weight", (long long)d.T * d.D);
    add(E + "LayerNorm.weight", d.D);
    add(E + "LayerNorm.bias", d.D);
    for (int i = 0; i < d.L; ++i) {
        const std::string L = M + (distil ? "transformer.layer." : "encoder.layer.") + std::to_string(i) + ".";
        // query | key | value stored back to back (no padding): one packed [3D, D] weight, [3D] bias
        add(L + n[0] + ".weight", (long long)d.D * d.D, false);
        add(L + n[1] + ".weight", (long long)d.D * d.D, false);
        add(L + n[2] + ".weight", (long long)d.D * d.D, true);
        add(L + n[0] + ".bias", d.D, false);
        add(L + n[1] + ".bias", d.D, false);
        add(L + n[2] + ".bias", d.D, true);
        add(L + n[3] + ".weight", (long long)d.D * d.D);
        add(L + n[3] + ".bias", d.D);
        add(L + n[4] + ".weight", d.D);
        add(L + n[4] + ".bias", d.D);
        add(L + n[5] + ".weight", (long long)d.F * d.D);
        add(L + n[5] + ".bias", d.F);
        add(L + n[6] + ".weight", (long long)d.D * d.F);
        add(L + n[6] + ".bias", d.D);
        add(L + n[7] + ".weight", d.D);
        add(L + n[7] + ".bias", d.D);
    }
    // head: dense [D, D] -> tanh / ReLU -> out [C, D]
    const std::string hd = distil ? "pre_classifier." : d.arch == TE_BERT_ARCH_ROBERTA ? "classifier.dense." : "bert.pooler.dense.";
    const std::string ho = d.arch == TE_BERT_ARCH_ROBERTA ? "classifier.out_proj." : "classifier.";
    add(hd + "weight", (long long)d.D * d.D);
    add(hd + "bias", d.D);
    add(ho + "weight", (long long)d.C * d.D);
    add(ho + "bias", d.C);
    t.push_back({"", 0, off});
    return t;
}

struct LayerW {
    const float *qkvw, *qkvb, *ow, *ob, *ln1w, *ln1b, *w1, *b1, *w2, *b2, *ln2w, *ln2b;
};
struct Weights {
    const float *word, *pos, *type, *elnw, *elnb, *poolw, *poolb, *clsw, *clsb;
    LayerW layer[kMaxDepth];
};

static void bind_weights(const te_bert_config* c, const float* base, Weights& w) {
    const WTable t = weight_table(c);
    size_t i = 0;
    auto next = [&]() { return base + t[i++].offset; };
    w.word = next(); w.pos = next();
    w.type = c->arch == TE_BERT_ARCH_DISTILBERT ? nullptr : next();
    w.elnw = next(); w.elnb = next();
    for (int l = 0; l < c->layers; ++l) {
        LayerW& y = w.layer[l];
        y.qkvw = next(); next(); next();
        y.qkvb = next(); next(); next();
        y.ow = next(); y.ob = next(); y.ln1w = next(); y.ln1b = next();
        y.w1 = next(); y.b1 = next(); y.w2 = next(); y.b2 = next(); y.ln2w = next(); y.ln2b = next();
    }
    w.poolw = next(); w.poolb = next(); w.clsw = next(); w.clsb = next();
}

// ---- derived tensor-core copies: per layer q | k | v | o | w1 | w2 ---------------------------------------
// (q, k, v: operands of their three z+ rules; qkv: the packed [3D, D] weight for the forward / backward GEMMs)
struct DerivedW { const float *q, *k, *v, *o, *w1, *w2, *qkv; };
static long long derived_layer_floats(const Dims& d) {
    return 4 * te_tc_derived_floats(d.D, d.D) + te_tc_derived_floats(d.D, d.F) + te_tc_derived_floats(d.F, d.D) +
           te_tc_derived_floats(d.D, 3 * d.D);
}
static DerivedW bind_derived(const Dims& d, const float* base, int l) {
    DerivedW w = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    if (!base) return w;
    const float* p = base + (long long)l * derived_layer_floats(d);
    const long long dd = te_tc_derived_floats(d.D, d.D);
    w.q = p; w.k = p + dd; w.v = p + 2 * dd; w.o = p + 3 * dd;
    w.w1 = p + 4 * dd;
    w.w2 = w.w1 + te_tc_derived_floats(d.D, d.F);
    w.qkv = w.w2 + te_tc_derived_floats(d.F, d.D);
    return w;
}

// ---- workspace ---------------------------------------------------------------------------------------
struct LayerAct {
    float *h, *qkv, *P, *ctx, *d1, *s1, *ao, *mean1, *rstd1, *hpre, *g, *d2, *s2, *mean2, *rstd2, *G, *cam;
};
struct Workspace {
    LayerAct layer[kMaxDepth];
    float *h_last, *maskadd, *pd, *pooled, *logits, *seed, *dpool, *dpd, *dfirst, *rpool, *rfirst, *shead;
    float *tD[4], *tF[2], *t3D[2], *tA[2];
    long long nF[2];                  // floats of tF[0], tF[1]
    float *mats, *joint[2];
    double* addpart;
    long long bytes;
};

static void carve(const Dims& d, char* base, Workspace& ws) {
    Bump take{base};
    const long long MD = d.M * d.D, MF = d.M * d.F, M3D = d.M * 3LL * d.D;
    const long long AT = (long long)d.B * d.H * d.N * d.NP;
    for (int l = 0; l < d.L; ++l) {
        LayerAct& a = ws.layer[l];
        a.h = take(MD); a.qkv = take(M3D); a.P = take(AT); a.ctx = take(MD); a.d1 = take(MD); a.s1 = take(MD);
        a.ao = take(MD); a.mean1 = take(d.M); a.rstd1 = take(d.M); a.hpre = take(MF); a.g = take(MF); a.d2 = take(MD);
        a.s2 = take(MD); a.mean2 = take(d.M); a.rstd2 = take(d.M); a.G = take(AT); a.cam = take(AT);
    }
    ws.h_last = take(MD);
    ws.maskadd = take((long long)d.B * d.N);
    const long long BD = (long long)d.B * d.D, BC = (long long)d.B * d.C;
    ws.pd = take(BD); ws.pooled = take(BD); ws.dpool = take(BD); ws.dpd = take(BD); ws.dfirst = take(BD);
    ws.rpool = take(BD); ws.rfirst = take(BD);
    ws.logits = take(BC); ws.seed = take(BC); ws.shead = take(BC > BD ? BC : BD);
    for (int i = 0; i < 4; ++i) ws.tD[i] = take(MD);
    // tF[1] is sized by its largest use, not by F alone (with intermediate < 1.5 hidden a use is wider than M*F):
    //   SF [M, F] (and the |x| scratch of the output-dense z+ rule); the GELU-output fp16 split [M, F] of the forward; the
    //   3-way clone's sum [M, D]; the hi-only fp16 split of dy of every backward Linear, widest for qkv [M, 3D / 2]
    ws.nF[0] = MF;
    ws.nF[1] = std::max({MF, MD, bwd_split_floats(d.M, 3 * d.D)});
    ws.tF[0] = take(ws.nF[0]); ws.tF[1] = take(ws.nF[1]);
    ws.t3D[0] = take(M3D); ws.t3D[1] = take(M3D);
    ws.tA[0] = take(AT); ws.tA[1] = take(AT);
    ws.mats = take((long long)d.L * d.B * d.N * d.NP);
    ws.joint[0] = take((long long)d.B * d.N * d.NP);
    ws.joint[1] = take((long long)d.B * d.N * d.NP);
    ws.addpart = reinterpret_cast<double*>(take((long long)d.B * TE_ADD_SPLIT * 3 * 2));
    ws.bytes = take.off;
}

static int check_ws(const te_bert_config* cfg, int batch, int seq, void* workspace, long long bytes, Dims& d,
                    Workspace& ws) {
    return te_util::check_ws("te_bert", batch, workspace, bytes, [&] { return make_dims(cfg, batch, seq, d); },
                             [&] { carve(d, reinterpret_cast<char*>(workspace), ws); return ws.bytes; });
}

}  // namespace

// =====================================================================================================
extern "C" int te_bert_num_weights(const te_bert_config* cfg) { return wt_count(weight_table(cfg)); }
extern "C" const char* te_bert_weight_name(const te_bert_config* cfg, int i) { return wt_name(weight_table(cfg), i); }
extern "C" long long te_bert_weight_numel(const te_bert_config* cfg, int i) { return wt_numel(weight_table(cfg), i); }
extern "C" long long te_bert_weight_offset(const te_bert_config* cfg, int i) { return wt_offset(weight_table(cfg), i); }
extern "C" long long te_bert_weight_total(const te_bert_config* cfg) { return wt_total(weight_table(cfg)); }
extern "C" long long te_bert_workspace_bytes(const te_bert_config* cfg, int batch, int seq) {
    Dims d;
    if (batch <= 0 || !make_dims(cfg, batch, seq, d)) return TE_ERR_ARG;
    Workspace ws;
    carve(d, nullptr, ws);
    return ws.bytes;
}
extern "C" long long te_bert_derived_total(const te_bert_config* cfg) {
    Dims d;
    if (!make_dims(cfg, 1, 1, d)) return TE_ERR_ARG;
    return (long long)d.L * derived_layer_floats(d);
}
extern "C" int te_bert_prepare_derived(const te_bert_config* cfg, const float* weights, float* derived, void* stream) {
    Dims d;
    if (!make_dims(cfg, 1, 1, d)) return TE_ERR_ARG;
    if (!weights || !derived) { te_set_last_error("te_bert_prepare_derived: null pointer"); return TE_ERR_ARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    Weights w;
    bind_weights(cfg, weights, w);
    const long long DD = (long long)d.D * d.D;
    for (int l = 0; l < d.L; ++l) {
        const DerivedW dw = bind_derived(d, derived, l);
        TE_TRY(te_tc_prepare_weights(w.layer[l].qkvw, const_cast<float*>(dw.q), d.D, d.D, st));
        TE_TRY(te_tc_prepare_weights(w.layer[l].qkvw + DD, const_cast<float*>(dw.k), d.D, d.D, st));
        TE_TRY(te_tc_prepare_weights(w.layer[l].qkvw + 2 * DD, const_cast<float*>(dw.v), d.D, d.D, st));
        TE_TRY(te_tc_prepare_weights(w.layer[l].ow, const_cast<float*>(dw.o), d.D, d.D, st));
        TE_TRY(te_tc_prepare_weights(w.layer[l].w1, const_cast<float*>(dw.w1), d.D, d.F, st));
        TE_TRY(te_tc_prepare_weights(w.layer[l].w2, const_cast<float*>(dw.w2), d.F, d.D, st));
        TE_TRY(te_tc_prepare_weights(w.layer[l].qkvw, const_cast<float*>(dw.qkv), d.D, 3 * d.D, st));
    }
    return TE_OK;
}

// =====================================================================================================
// forward  (BertForSequenceClassification.forward -> BertModel.forward)
// =====================================================================================================
extern "C" int te_bert_forward(const te_bert_config* cfg, const float* weights, const float* derived,
                               const long long* input_ids, const long long* attention_mask,
                               const long long* token_type_ids, int batch, int seq, unsigned flags, float* logits,
                               void* workspace, long long workspace_bytes, void* stream) {
    Dims d; Workspace ws;
    TE_TRY(check_ws(cfg, batch, seq, workspace, workspace_bytes, d, ws));
    if (!weights || !input_ids || !attention_mask) { te_set_last_error("te_bert_forward: null pointer"); return TE_ERR_ARG; }
    if (token_type_ids && d.arch == TE_BERT_ARCH_DISTILBERT) {
        te_set_last_error("te_bert_forward: DistilBERT takes no token_type_ids (it has no token-type table)");
        return TE_ERR_ARG;
    }
    Select sel;
    TE_TRY(decode_flags(sel, "te_bert_forward", flags, derived, 0, false));
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    // fp16-split forward Linears: split of the D-wide inputs in tD[1] (+ scales tD[2]), of the GELU output in tF[1] (+ scales
    // tD[3]); all idle until the backward pass.  Every LayerNorm emits the split of its output (the hidden state feeds the next
    // layer's qkv).
    const F16Forward f16 = f16_forward(sel, d.M, d.D, d.F, ws.tD[1], ws.tD[2], ws.tF[1], ws.tD[3]);
    auto layernorm = [&](const float* x, const float* g, const float* b, float* y, float* mean, float* rstd) {
        return f16.on ? te_launch_layernorm_split(x, g, b, y, mean, rstd, d.M, d.D, d.eps, f16.qkv.split, f16.qkv.scale, st)
                      : te_launch_layernorm(x, g, b, y, mean, rstd, d.M, d.D, d.eps, st);
    };
    Weights w;
    bind_weights(cfg, weights, w);
    const float scale = 1.0f / sqrtf((float)d.dh);

    if (d.arch == TE_BERT_ARCH_BERT)
        TE_TRY(te_launch_bert_embed(input_ids, token_type_ids, w.word, w.pos, w.type, ws.tD[0], d.B, d.N, d.D, d.V, d.T, st));
    else      // RoBERTa: position ids counted from pad on the device; DistilBERT: arange, no token-type table
        TE_TRY(te_launch_hf_embed(input_ids, token_type_ids, w.word, w.pos, w.type, ws.tD[0], d.B, d.N, d.D, d.V, d.P, d.T,
                                  d.arch == TE_BERT_ARCH_ROBERTA ? d.pad : -1, st));
    TE_TRY(layernorm(ws.tD[0], w.elnw, w.elnb, ws.layer[0].h, nullptr, nullptr));
    TE_TRY(te_launch_bert_mask(attention_mask, ws.maskadd, (long long)d.B * d.N, st));

    for (int l = 0; l < d.L; ++l) {
        LayerAct& a = ws.layer[l];
        const LayerW& lw = w.layer[l];
        float* h_next = (l + 1 < d.L) ? ws.layer[l + 1].h : ws.h_last;
        const DerivedW tw = bind_derived(d, sel.lbase, l);
        TE_TRY(linear_fwd_tc(tw.qkv, a.h, d.D, lw.qkvw, lw.qkvb, a.qkv, nullptr, nullptr, d.M, d.D, 3 * d.D, TE_EPI_BIAS, st,
                             &f16.qkv));
        // scores = q k^T / sqrt(d) ; + extended mask ; softmax      (:338-345)
        TE_TRY(attn_nn(sel.atc, d.B, d.H, d.N, d.NP, d.dh, a.qkv, 3 * d.D, a.qkv + d.D, 3 * d.D, a.P, nullptr, scale,
                       TE_EPI_STORE, st));
        TE_TRY(te_launch_softmax_masked(a.P, (long long)d.B * d.H * d.N, d.N, d.NP, ws.maskadd, (long long)d.H * d.N, st));
        TE_TRY(attn_nk(sel.atc, d.B, d.H, d.N, d.NP, d.dh, a.P, 0, a.qkv + 2 * d.D, 3 * d.D, a.ctx, d.D, nullptr, 1.f,
                       TE_EPI_STORE, st));
        // BertSelfOutput: dense -> add([dense, input]) -> LayerNorm
        TE_TRY(linear_fwd_tc(tw.o, a.ctx, d.D, lw.ow, lw.ob, a.d1, a.s1, a.h, d.M, d.D, d.D, TE_EPI_BIAS_ADD, st, &f16.proj));
        TE_TRY(layernorm(a.s1, lw.ln1w, lw.ln1b, a.ao, a.mean1, a.rstd1));
        // BertIntermediate (dense + GELU), BertOutput (dense -> add -> LayerNorm)
        TE_TRY(linear_fwd_tc(tw.w1, a.ao, d.D, lw.w1, lw.b1, a.hpre, a.g, nullptr, d.M, d.D, d.F, TE_EPI_BIAS_GELU, st,
                             &f16.fc1));
        TE_TRY(linear_fwd_tc(tw.w2, a.g, d.F, lw.w2, lw.b2, a.d2, a.s2, a.ao, d.M, d.F, d.D, TE_EPI_BIAS_ADD, st, &f16.fc2));
        TE_TRY(layernorm(a.s2, lw.ln2w, lw.ln2b, h_next, a.mean2, a.rstd2));
    }
    // pooler (first token -> dense -> tanh; DistilBERT's pre_classifier -> ReLU), classifier
    TE_TRY(linear_fwd(ws.h_last, d.N * d.D, w.poolw, w.poolb, ws.pd, nullptr, nullptr, d.B, d.D, d.D, TE_EPI_BIAS, st));
    if (d.arch == TE_BERT_ARCH_DISTILBERT) TE_TRY(te_launch_relu(ws.pd, ws.pooled, (long long)d.B * d.D, st));
    else TE_TRY(te_launch_tanh(ws.pd, ws.pooled, (long long)d.B * d.D, st));
    TE_TRY(linear_fwd(ws.pooled, d.D, w.clsw, w.clsb, ws.logits, nullptr, nullptr, d.B, d.D, d.C, TE_EPI_BIAS, st));
    if (logits && cudaMemcpyAsync(logits, ws.logits, sizeof(float) * d.B * d.C, cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
        te_set_last_error("te_bert_forward: logits copy failed");
        return TE_ERR_CUDA;
    }
    return TE_OK;
}

// =====================================================================================================
// attribute = class-gradient backward + relprop + normalised rollout   (Generator.generate_LRP :33-59)
// =====================================================================================================
extern "C" int te_bert_attribute(const te_bert_config* cfg, const float* weights, const float* derived, int batch, int seq,
                                 int* index, int start_layer, float alpha, unsigned flags, float* maps, void* workspace,
                                 long long workspace_bytes, void* stream) {
    Dims d; Workspace ws;
    TE_TRY(check_ws(cfg, batch, seq, workspace, workspace_bytes, d, ws));
    if (!isfinite(alpha)) { te_set_last_error("te_bert_attribute: alpha must be finite"); return TE_ERR_ARG; }
    TE_TRY(te_util::check_grad_rollout("te_bert_attribute", flags, alpha));
    const bool grad_rollout = (flags & TE_FLAG_ATTN_GRAD_ROLLOUT) != 0;
    if (!weights || !index || (!maps && !(flags & TE_FLAG_GRADIENTS_ONLY))) { te_set_last_error("te_bert_attribute: null pointer"); return TE_ERR_ARG; }
    if (start_layer < 0 || start_layer >= d.L) { te_set_last_error("te_bert_attribute: start_layer out of range"); return TE_ERR_ARG; }
    // fp16 backward split of dy in tF[1], block scales in t3D[1] (idle until the relprop)
    Select sel;
    TE_TRY(decode_flags(sel, "te_bert_attribute", flags, derived, start_layer, !grad_rollout, {ws.tF[1], ws.nF[1]},
                        {ws.t3D[1], d.M * 3LL * d.D}, d.M, std::max(3 * d.D, d.F)));
    if (sel.seeded) { te_set_last_error("te_bert_attribute: TE_FLAG_SIMILARITY_SEED is a ViT (CLIP image tower) mode"); return TE_ERR_ARG; }
    cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    Weights w;
    bind_weights(cfg, weights, w);
    const float scale = 1.0f / sqrtf((float)d.dh);
    const long long MD = d.M * d.D, DD = (long long)d.D * d.D;

    TE_TRY(te_launch_argmax(ws.logits, index, d.B, d.C, 1, st));
    TE_TRY(te_launch_onehot(index, ws.seed, d.B, d.C, 1.0f, st));

    // ---- backward: d logit_c / d attention_probs of every layer --------------------------------------------
    float* dxa = ws.tD[0]; float* dsx = ws.tD[1]; float* dctx = ws.tD[2]; float* dxn = ws.tD[3];
    float* dF = ws.tF[0]; float* dqkv = ws.t3D[0]; float* dS = ws.tA[0];
    TE_TRY(linear_bwd(ws.seed, w.clsw, ws.dpool, nullptr, d.B, d.D, d.C, TE_EPI_STORE, st));         // classifier
    if (d.arch == TE_BERT_ARCH_DISTILBERT)
        TE_TRY(te_launch_relu_bwd(ws.dpool, ws.pooled, ws.dpd, (long long)d.B * d.D, st));           // head ReLU
    else
        TE_TRY(te_launch_tanh_bwd(ws.dpool, ws.pooled, ws.dpd, (long long)d.B * d.D, st));           // pooler tanh
    TE_TRY(linear_bwd(ws.dpd, w.poolw, ws.dfirst, nullptr, d.B, d.D, d.D, TE_EPI_STORE, st));        // pooler dense
    TE_TRY(te_launch_fill(dxa, 0.f, MD, st));
    if (cudaMemcpy2DAsync(dxa, sizeof(float) * d.N * d.D, ws.dfirst, sizeof(float) * d.D, sizeof(float) * d.D, d.B,
                          cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
        te_set_last_error("te_bert_attribute: scatter of the pooled-token gradient failed");
        return TE_ERR_CUDA;
    }
    for (int l = d.L - 1; l >= start_layer; --l) {
        LayerAct& a = ws.layer[l];
        const LayerW& lw = w.layer[l];
        TE_TRY(te_launch_layernorm_bwd(dxa, a.s2, lw.ln2w, a.mean2, a.rstd2, nullptr, dsx, d.M, d.D, st));    // d s2
        const DerivedW tw = bind_derived(d, sel.lbase, l);
        TE_TRY(linear_bwd_tc(tw.w2, dsx, lw.w2, dF, a.hpre, d.M, d.F, d.D, TE_EPI_GELU_BWD, st, sel.btf, &sel.bfs));
        TE_TRY(linear_bwd_tc(tw.w1, dF, lw.w1, dxn, nullptr, d.M, d.D, d.F, TE_EPI_STORE, st, sel.btf, &sel.bfs));
        TE_TRY(te_launch_add2(dxn, dsx, dxn, MD, st));                                                          // d ao
        TE_TRY(te_launch_layernorm_bwd(dxn, a.s1, lw.ln1w, a.mean1, a.rstd1, nullptr, dsx, d.M, d.D, st));    // d s1
        TE_TRY(linear_bwd_tc(tw.o, dsx, lw.ow, dctx, nullptr, d.M, d.D, d.D, TE_EPI_STORE, st, sel.btf, &sel.bfs));
        const bool last = (l == start_layer);
        TE_TRY(attn_block_bwd(sel, d.B, d.H, d.N, d.NP, d.dh, a.qkv, a.P, dctx, a.G, dS, dqkv, scale, last, st));
        if (last) break;
        TE_TRY(linear_bwd_tc(tw.qkv, dqkv, lw.qkvw, dxn, nullptr, d.M, d.D, 3 * d.D, TE_EPI_STORE, st, sel.btf, &sel.bfs));
        TE_TRY(te_launch_add2(dxn, dsx, dxa, MD, st));                                                          // d h
    }

    if (flags & TE_FLAG_GRADIENTS_ONLY) return TE_OK;      // attention-GradCAM baseline: gradients are all it reads
    // P and G of a layer are carved side by side in every layer's slice, so one layer stride serves both operands
    const long long layer_stride = d.L > 1 ? (long long)(ws.layer[1].G - ws.layer[0].G) : 0;
    if (grad_rollout) {
        // gradient-weighted attention rollout: mean_h relu(G * P) + I chained from start_layer, no relprop, no row
        // normalisation; row 0 with element 0 set to 0 (the reference's BERT comparison generators).  Padded keys have
        // P = 0 and padded queries G = 0, so padded entries come out exactly 0.
        TE_TRY(te_rollout_layers(ws.layer[0].G, ws.layer[0].P, layer_stride, d.L, d.B, d.H, d.N, d.NP, d.NP, start_layer,
                                 /*normalize=*/0, flags, ws.mats, ws.joint[0], ws.joint[1], nullptr, maps, /*first=*/0,
                                 /*bert_fix=*/0, st));
        if (cudaMemset2DAsync(maps, sizeof(float) * d.N, 0, sizeof(float), d.B, st) != cudaSuccess) {
            te_set_last_error("te_bert_attribute: clearing element 0 of the maps failed");
            return TE_ERR_CUDA;
        }
        return TE_OK;
    }

    // ---- relprop -----------------------------------------------------------------------------------------------
    float* R = ws.tD[0]; float* R1 = ws.tD[1]; float* R2 = ws.tD[2]; float* R3 = ws.tD[3];
    float* RF = ws.tF[0]; float* SF = ws.tF[1]; float* S = ws.t3D[0]; float* Rqkv = ws.t3D[1];
    // Linear / Add rules of the selected rule library: layers_ours, or with TE_FLAG_RULES_LRP layers_lrp (BERT_cls_lrp.py on
    // BERT_orig_lrp.py: Linear with separate denominators, Add = RelPropSimple, also for the attention-mask Add).  dw is set
    // for the z+ rules with TE_FLAG_ZPLUS_TENSOR_CORES, for the layers_lrp rule with TE_FLAG_RULES_LRP_TC.  alpha != 1: the
    // alpha-beta Linear rule of either library.
    double* addp = sel.lrp ? nullptr : ws.addpart;
    // classifier.relprop (X = pooled) ; dropout / Tanh identity ; pooler.dense.relprop (X = first token) ; pool
    TE_TRY(te_linear_rule_relprop(sel.lrp, ws.pooled, d.D, w.clsw, nullptr, ws.seed, d.C, ws.rpool, ws.shead, d.B, d.D, d.C, st,
                                  nullptr, 0, nullptr, sel.zv, 0, nullptr, alpha));
    TE_TRY(te_linear_rule_relprop(sel.lrp, ws.h_last, (long long)d.N * d.D, w.poolw, nullptr, ws.rpool, d.D, ws.rfirst, ws.shead,
                                  d.B, d.D, d.D, st, nullptr, 0, nullptr, sel.zv, 0, nullptr, alpha));
    TE_TRY(te_launch_index_select_relprop(ws.h_last, ws.rfirst, nullptr, R, d.B, d.N, d.D, st));

    for (int l = d.L - 1; l >= sel.low; --l) {
        LayerAct& a = ws.layer[l];
        const LayerW& lw = w.layer[l];
        const DerivedW dw = bind_derived(d, sel.dbase, l);
        // BertOutput.relprop :474-487 ; BertIntermediate.relprop :451-456 ; BertLayer.clone
        // top layer: relevance is non-zero only in the first token's row (pooler, BERT.py:181-190) and every rule down
        // to the attention-output dense rule is row-wise (both libraries) -> its three Linear rules run on the B
        // first-token rows only (exact)
        const bool top = (l == d.L - 1) && te_engine_cls_rows();
        const long long zr = top ? d.B : d.M;
        const long long sD = top ? (long long)d.N * d.D : d.D, sF = top ? (long long)d.N * d.F : d.F;
        TE_TRY(te_launch_add_relprop(a.d2, a.ao, R, R1, R2, addp, d.B, (long long)d.N * d.D, st));
        TE_TRY(te_linear_rule_relprop(sel.lrp, a.g, sF, lw.w2, dw.w2, R1, sD, RF, S, zr, d.F, d.D, st, a.d2, sD, lw.b2, sel.zv, sF,
                                      SF, alpha));
        TE_TRY(te_linear_rule_relprop(sel.lrp, a.ao, sD, lw.w1, dw.w1, RF, sF, R1, SF, zr, d.D, d.F, st, a.hpre, sF, lw.b1, sel.zv,
                                      sD, S, alpha));
        TE_TRY(te_launch_clone_relprop(a.ao, R1, R2, nullptr, R, MD, st));
        // BertSelfOutput.relprop :427-434
        TE_TRY(te_launch_add_relprop(a.d1, a.h, R, R1, R2, addp, d.B, (long long)d.N * d.D, st));
        if (top) TE_TRY(te_launch_fill(R3, 0.f, MD, st));
        TE_TRY(te_linear_rule_relprop(sel.lrp, a.ctx, sD, lw.ow, dw.o, R1, sD, R3, S, zr, d.D, d.D, st, a.d1, sD, lw.ob, sel.zv, sD,
                                      S + MD, alpha));
        // BertSelfAttention.relprop :367-409: matmul2 rule -> attn_cam (:380), cam_v
        const bool last = (l == sel.low && !(flags & TE_FLAG_RELPROP_TO_INPUT));
        TE_TRY(attn_relprop_pv(sel, d.B, d.H, d.N, d.NP, d.dh, a.qkv, a.P, R3, a.ctx, S, a.cam, Rqkv, last, st));
        if (last) break;
        // add([scores, mask]).relprop : scores = q k^T / sqrt(d) recomputed ; relevance renormalised (layers_ours)  :386-388
        TE_TRY(attn_nn(sel.atc, d.B, d.H, d.N, d.NP, d.dh, a.qkv, 3 * d.D, a.qkv + d.D, 3 * d.D, ws.tA[0], nullptr, scale,
                       TE_EPI_STORE, st));
        TE_TRY(te_launch_add_relprop_keymask(ws.tA[0], ws.maskadd, a.cam, ws.tA[1], addp, d.B, d.H, d.N, d.NP, st));
        // matmul1 rule on the unscaled product -> cam_q, cam_k
        TE_TRY(attn_relprop_qk(sel, d.B, d.H, d.N, d.NP, d.dh, a.qkv, ws.tA[1], ws.tA[0], Rqkv, st));
        // query / key / value Linear rules (separate Linears), Clone(3), Clone(2)
        TE_TRY(te_linear_rule_relprop(sel.lrp, a.h, d.D, lw.qkvw, dw.q, Rqkv, 3 * d.D, R, S, d.M, d.D, d.D, st, a.qkv, 3 * d.D,
                                      lw.qkvb, sel.zv, 0, S + MD, alpha));
        TE_TRY(te_linear_rule_relprop(sel.lrp, a.h, d.D, lw.qkvw + DD, dw.k, Rqkv + d.D, 3 * d.D, R1, S, d.M, d.D, d.D, st,
                                      a.qkv + d.D, 3 * d.D, lw.qkvb + d.D, sel.zv, 0, S + MD, alpha));
        TE_TRY(te_linear_rule_relprop(sel.lrp, a.h, d.D, lw.qkvw + 2 * DD, dw.v, Rqkv + 2 * d.D, 3 * d.D, R3, S, d.M, d.D, d.D, st,
                                      a.qkv + 2 * d.D, 3 * d.D, lw.qkvb + 2 * d.D, sel.zv, 0, S + MD, alpha));
        TE_TRY(te_launch_clone_relprop(a.h, R, R1, R3, SF, MD, st));                      // self.clone (3-way)
        TE_TRY(te_launch_clone_relprop(a.h, SF, R2, nullptr, R, MD, st));                 // attention.clone
    }

    // ---- aggregation + normalised rollout, row 0 with [0] = min   (ExplanationGenerator.py:47-59) ---------------
    TE_TRY(te_rollout_layers(ws.layer[0].G, ws.layer[0].cam, layer_stride, d.L, d.B, d.H, d.N, d.NP, d.NP, start_layer,
                             /*normalize=*/1, flags, ws.mats, ws.joint[0], ws.joint[1], nullptr, maps, /*first=*/0,
                             /*bert_fix=*/1, st));
    return TE_OK;
}

extern "C" int te_bert_explain(const te_bert_config* cfg, const float* weights, const float* derived,
                               const long long* input_ids, const long long* attention_mask,
                               const long long* token_type_ids, int batch, int seq, int* index, int start_layer,
                               unsigned flags, float* maps, float* logits, void* workspace, long long workspace_bytes,
                               void* stream) {
    TE_TRY(te_bert_forward(cfg, weights, derived, input_ids, attention_mask, token_type_ids, batch, seq, flags, logits,
                           workspace, workspace_bytes, stream));
    return te_bert_attribute(cfg, weights, derived, batch, seq, index, start_layer, 1.f, flags, maps, workspace, workspace_bytes,
                             stream);
}

extern "C" int te_bert_tensor(const te_bert_config* cfg, int batch, int seq, void* workspace, const char* name, int layer,
                              float** ptr, long long dims[4], long long strides[4]) {
    Dims d; Workspace ws;
    if (!workspace || !name || !ptr) return TE_ERR_ARG;
    if (batch <= 0 || !make_dims(cfg, batch, seq, d)) return TE_ERR_ARG;
    carve(d, reinterpret_cast<char*>(workspace), ws);
    const std::string n(name);
    const View set{ptr, dims, strides};
    if (n == "logits") return set(ws.logits, d.B, d.C, 1, 1, d.C, 1, 1, 1);
    if (n == "relevance_in") return set(ws.tD[0], d.B, d.N, d.D, 1, (long long)d.N * d.D, d.D, 1, 1);
    // scratch of the last attribute() call (debug / diagnostics): tmp_d0..3 [B,N,D], tmp_f0..1 [B,N,F], tmp_3d0..1 [B,N,3D]
    if (n.rfind("tmp_d", 0) == 0 && n.size() == 6 && n[5] >= '0' && n[5] <= '3')
        return set(ws.tD[n[5] - '0'], d.B, d.N, d.D, 1, (long long)d.N * d.D, d.D, 1, 1);
    if (n.rfind("tmp_f", 0) == 0 && n.size() == 6 && n[5] >= '0' && n[5] <= '1')
        return set(ws.tF[n[5] - '0'], d.B, d.N, d.F, 1, (long long)d.N * d.F, d.F, 1, 1);
    if (n.rfind("tmp_3d", 0) == 0 && n.size() == 7 && n[6] >= '0' && n[6] <= '1')
        return set(ws.t3D[n[6] - '0'], d.B, d.N, 3LL * d.D, 1, (long long)d.N * 3 * d.D, 3LL * d.D, 1, 1);
    const long long ND = (long long)d.N * d.D, NF = (long long)d.N * d.F;
    if (n == "h_last") return set(ws.h_last, d.B, d.N, d.D, 1, ND, d.D, 1, 1);
    if (n == "pooled") return set(ws.pooled, d.B, d.D, 1, 1, d.D, 1, 1, 1);
    if (layer < 0 || layer >= d.L) { te_set_last_error("te_bert_tensor: layer out of range"); return TE_ERR_ARG; }
    LayerAct& a = ws.layer[layer];
    const long long hs = (long long)d.N * d.NP, bs = hs * d.H;
    if (n == "attn") return set(a.P, d.B, d.H, d.N, d.N, bs, hs, d.NP, 1);
    if (n == "attn_grad") return set(a.G, d.B, d.H, d.N, d.N, bs, hs, d.NP, 1);
    if (n == "attn_cam") return set(a.cam, d.B, d.H, d.N, d.N, bs, hs, d.NP, 1);
    if (n == "hidden") return set(a.h, d.B, d.N, d.D, 1, (long long)d.N * d.D, d.D, 1, 1);
    // the rest of the saved forward activations of the layer (views only: test / diagnostic taps)
    if (n == "qkv") return set(a.qkv, d.B, d.N, 3LL * d.D, 1, 3 * ND, 3LL * d.D, 1, 1);
    float* rowD = n == "ctx" ? a.ctx : n == "d1" ? a.d1 : n == "s1" ? a.s1 : n == "ao" ? a.ao : n == "d2" ? a.d2
                : n == "s2" ? a.s2 : nullptr;
    if (rowD) return set(rowD, d.B, d.N, d.D, 1, ND, d.D, 1, 1);
    float* rowF = n == "hpre" ? a.hpre : n == "g" ? a.g : nullptr;
    if (rowF) return set(rowF, d.B, d.N, d.F, 1, NF, d.F, 1, 1);
    float* row1 = n == "mean1" ? a.mean1 : n == "rstd1" ? a.rstd1 : n == "mean2" ? a.mean2 : n == "rstd2" ? a.rstd2 : nullptr;
    if (row1) return set(row1, d.B, d.N, 1, 1, d.N, 1, 1, 1);
    te_set_last_error("te_bert_tensor: unknown tensor name");
    return TE_ERR_ARG;
}
