/* te_b200 — C ABI of the transformer-attribution engine (CUDA, sm_90a / H100).
 *
 * Drop-in boundary for the `transformer_attribution` path of hila-chefer/Transformer-Explainability.
 * The reference has no FFI: its interface for this path is a Python "relprop protocol"
 * (every layer has forward()/relprop(R, alpha); generators call model(x) -> backward -> model.relprop()).
 * Each entry point below names the reference interface (file:line under /root/reference) it replaces.
 *
 * Conventions
 *  - all tensors are contiguous row-major fp32 in DEVICE memory, borrowed from the caller
 *    (the library never allocates or frees caller memory; scratch comes from a caller `workspace`
 *    whose size is queried with the matching *_workspace_bytes function);
 *  - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, nothing synchronises;
 *  - return value: 0 = ok, negative = error (TE_ERR_*); te_last_error() returns a message.
 *    No exceptions cross the boundary; there is NO CPU fallback: a missing GPU is an error;
 *  - a "batch" is a set of INDEPENDENT B=1 explanations: every reduction the reference does over
 *    a whole B=1 tensor (Add.relprop's sums) is done per sample.
 */
#ifndef TE_B200_H
#define TE_B200_H

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define TE_API __attribute__((visibility("default")))
#else
#define TE_API
#endif

#define TE_OK 0
#define TE_ERR_ARG (-1)
#define TE_ERR_WORKSPACE (-2)
#define TE_ERR_CUDA (-3)
#define TE_ERR_UNSUPPORTED (-4)

/* te_vit_attribute / te_vit_explain flags */
#define TE_FLAG_ZPLUS_TENSOR_CORES 1u /* z+ Linear-rule GEMMs on wgmma tensor cores (TF32 in, fp32 acc) instead of fp32 SIMT */
#define TE_FLAG_ROLLOUT_FUSED 2u      /* single fused aggregation+rollout kernel instead of aggregate + bmm chain */
#define TE_FLAG_KEEP_ALL_CAMS 4u      /* run the relprop below start_layer too (accessor parity with the reference) */
#define TE_FLAG_LINEAR_TENSOR_CORES 16u /* forward / backward Linear GEMMs on wgmma with the fp32-grade 3xTF32 split */
#define TE_FLAG_ATTN_TENSOR_CORES 32u  /* the N x N attention contractions (QK^T, dctx V^T, S2 V^T) on wgmma, 3xTF32 */
#define TE_FLAG_ZPLUS_BF16 64u          /* with TE_FLAG_ZPLUS_TENSOR_CORES: S = R/Z stored as bf16 and the second z+ contraction
                                         (R_in = x+ (S W+) + x- (S W-)) on bf16 wgmma */
#define TE_FLAG_GRADIENTS_ONLY 128u    /* te_*_attribute stops after the class-gradient backward: only "attn_grad" of the layers
                                         >= start_layer is produced (maps may be NULL) — the attention-GradCAM baselines */
#define TE_FLAG_BACKWARD_TF32 256u     /* with TE_FLAG_LINEAR_TENSOR_CORES: the activation-gradient backward Linears run as
                                         single-pass TF32 GEMMs instead of the 3xTF32 split.  The gradients only enter the
                                         result linearly (relu(G * cam)), never a safe_divide denominator
                                         (tests/test_gpu_parity_full.py bounds the effect) */
#define TE_FLAG_RELPROP_TF32 1024u     /* with TE_FLAG_ATTN_TENSOR_CORES: the attention-shaped contractions of the relprop whose
                                         result is relevance (attn_cam = P * (S V^T) / 2, P^T S, S1 K, S1^T Q) run single-pass
                                         TF32 like the z+ rule does; the denominator Q K^T keeps the 3xTF32 split */
#define TE_FLAG_ZPLUS_S1_BF16 2048u    /* with TE_FLAG_ZPLUS_TENSOR_CORES: the |x| |W|^T term of the single-pass z+ denominator with bf16
                                         operands (a sum of K non-negative products: rounding errors average to ~2^-9 / sqrt(K)) */
#define TE_FLAG_LINEAR_F16_SPLIT 4096u  /* with TE_FLAG_LINEAR_TENSOR_CORES: the forward Linears on fp16 wgmma with a block-scaled
                                         * fp16 (hi, lo) split of both operands (3 MMAs per k-step, same 22-bit operand precision
                                         * as the 3xTF32 split, fp16 MMAs run at twice the TF32 rate) */
#define TE_FLAG_ZPLUS_R_F16 8192u        /* with TE_FLAG_ZPLUS_TENSOR_CORES: the second contraction of the z+ rule, x+ (S W+) + x- (S W-), on
                                         * fp16 wgmma: S as block-scaled fp16 (one power of two per row and 128 columns),
                                         * W+^T / W-^T as row-scaled fp16 — the 11 significant bits of the TF32 form, at twice
                                         * the tensor rate */
#define TE_FLAG_BACKWARD_F16 16384u      /* with TE_FLAG_LINEAR_TENSOR_CORES: the activation-gradient backward Linears as ONE fp16 MMA per
                                         * k-step (block-scaled fp16 gradients, row-scaled fp16 weights) instead of one TF32 MMA
                                         * (TE_FLAG_BACKWARD_TF32): same 11 significant bits, twice the tensor rate */
#define TE_FLAG_RULES_LRP 512u         /* the rule library of modules/layers_lrp.py (baselines/ViT/ViT_orig_LRP.py) instead of
                                         modules/layers_ours.py: Linear divides its two halves by their OWN denominators
                                         (layers_lrp.py:199-200), Add has no ratio normalisation (:98-100).  fp32 SIMT rules
                                         unless TE_FLAG_RULES_LRP_TC.  te_vit_attribute (ViT_orig_LRP) and te_bert_attribute
                                         (BERT_cls_lrp.py on BERT_orig_lrp.py; also the attention-mask Add) */
#define TE_FLAG_RULES_LRP_TC 32768u      /* with TE_FLAG_RULES_LRP (read only together with it): both halves of its Linear rule,
                                          * S = sd(R, x+- W+-^T) and x+- * (S W+-), as single-pass TF32 wgmma GEMMs (needs
                                          * `derived`).  Each denominator is a sum of non-negative products, so TF32 operands
                                          * cost no cancellation; an exact zero stays exactly zero.  The bf16 / fp16 flags
                                          * (TE_FLAG_ZPLUS_BF16, _S1_BF16, _R_F16) do not apply to this rule. */
#define TE_FLAG_RELPROP_TO_INPUT 8u   /* finish the lowest block as well: relevance at the encoder input (what
                                         model.relprop() returns in the reference) is left in tensor "relevance_in" */

TE_API const char* te_last_error(void);
/* Process-wide tuning switches (not part of the reference surface).
 * name = "cls_row_top_block": 1 (default) runs the three z+ rules of the top block on the pooled-token rows only (exact:
 * the relevance entering the top block is zero in every other row), 0 on all rows.
 * name = "gelu_split_fused": 1 (default) lets the fp16-split forward Linears reuse the fp16 split of the LayerNorm / GELU
 * outputs written next to them, 0 splits every Linear input in a stand-alone pre-pass.
 * Returns TE_OK, or a negative status for an unknown name. */
TE_API int te_set_option(const char* name, int value);
TE_API int te_version(void);
/* number of kernels this library has launched in this process (bench.py reports the delta as gpu_launches) */
TE_API long long te_kernel_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * ViT / DeiT model description  (baselines/ViT/ViT_LRP.py:247-303 VisionTransformer.__init__)
 * ---------------------------------------------------------------------------------------------- */
typedef struct te_vit_config {
    int img_size;     /* 224 */
    int patch_size;   /* 16  */
    int in_chans;     /* 3   */
    int num_classes;  /* 1000 */
    int dim;          /* embed_dim */
    int depth;        /* number of blocks */
    int heads;
    int mlp_dim;      /* int(dim*mlp_ratio) */
    int distilled;    /* 1: extra dist_token + head_dist, logits averaged (DeiT-distilled extension) */
    float eps_block;  /* 1e-6, ViT_LRP.py:184,187 */
    float eps_final;  /* 1e-5, ViT_LRP.py:266 */
} te_vit_config;

/* Frozen weights live in ONE flat fp32 device buffer (also the unit of the NCCL broadcast).
 * Tensor i has the reference state_dict key te_vit_weight_name(i), te_vit_weight_numel(i) floats,
 * and starts at float offset te_vit_weight_offset(i) (every offset is a multiple of 32 floats). */
TE_API int te_vit_num_weights(const te_vit_config* cfg);
TE_API const char* te_vit_weight_name(const te_vit_config* cfg, int i);
TE_API long long te_vit_weight_numel(const te_vit_config* cfg, int i);
TE_API long long te_vit_weight_offset(const te_vit_config* cfg, int i);
TE_API long long te_vit_weight_total(const te_vit_config* cfg); /* floats */

/* Tensor-core operand copies of the frozen Linear weights (TF32, bf16 and row-scaled fp16 forms of W, W^T, their positive /
 * negative parts and |W|), read by the tensor-core Linear GEMMs and z+ rule kernels that TE_FLAG_LINEAR_TENSOR_CORES,
 * TE_FLAG_ZPLUS_TENSOR_CORES and the precision flags select: te_vit_derived_total() floats, filled once per weight load by
 * te_vit_prepare_derived().  `derived` may be NULL when no such flag is used. */
TE_API long long te_vit_derived_total(const te_vit_config* cfg);
TE_API int te_vit_prepare_derived(const te_vit_config* cfg, const float* weights, float* derived, void* stream);

/* Scratch for `batch` samples processed together (activations of every block are kept for the
 * relprop, like the reference's forward hooks, modules/layers_ours.py:16-27). */
TE_API long long te_vit_workspace_bytes(const te_vit_config* cfg, int batch);

/* model(x): VisionTransformer.forward (ViT_LRP.py:305-322).  images [batch,in_chans,img,img];
 * logits [batch,num_classes] (may be NULL).  Leaves every saved activation in `workspace`. */
TE_API int te_vit_forward(const te_vit_config* cfg, const float* weights, const float* derived, const float* images,
                   int batch, unsigned flags, float* logits, void* workspace, long long workspace_bytes, void* stream);

/* The rest of LRP.generate_LRP (ViT_explanation_generator.py:27-41) + VisionTransformer.relprop with
 * method="transformer_attribution" (ViT_LRP.py:324-369) on the activations te_vit_forward left behind:
 * arg-max (where index[b] < 0), one-hot, class gradient of every attention map, LRP relprop through
 * every block >= start_layer, relu(grad*cam) head-mean, +I, rollout, row 0 without the prefix token(s).
 * index [batch] int32 in/out (device); maps [batch, tokens-prefix] (device).
 * alpha: model.relprop(cam, alpha=alpha) (ViT_LRP.py:324, any method): every Linear.relprop of the rule library applies
 * the LRP-alpha-beta rule with beta = alpha - 1 (layers_ours.py:207-230, layers_lrp.py:187-210), R_in = alpha * act -
 * beta * inh, the inhibitor half running after the activator through the same scratch (the workspace size does not depend
 * on alpha).  alpha = 1 is the z+ rule every generator uses.  The other rules do not depend on alpha.  A non-finite alpha
 * returns TE_ERR_ARG. */
TE_API int te_vit_attribute(const te_vit_config* cfg, const float* weights, const float* derived, int batch, int* index,
                            int start_layer, float alpha, unsigned flags, float* maps, void* workspace,
                            long long workspace_bytes, void* stream);

/* te_vit_forward + te_vit_attribute (alpha = 1): one call per batch = LRP.generate_LRP for `batch` independent inputs. */
TE_API int te_vit_explain(const te_vit_config* cfg, const float* weights, const float* derived, const float* images,
                   int batch, int* index, int start_layer, unsigned flags, float* maps, float* logits, void* workspace,
                   long long workspace_bytes, void* stream);

/* Accessors into the workspace — get_attn / get_attn_gradients / get_attn_cam / get_v ...
 * (ViT_LRP.py:102-130).  name in {"attn","attn_grad","attn_cam","qkv","x_in","ctx","logits","rollout_mats"}, and the
 * scratch regions of the last attribute call, "tmp_d0".."tmp_d3" [B,N,D], "tmp_f0","tmp_f1" [B,N,F], "tmp_3d0","tmp_3d1"
 * [B,N,3D] (diagnostics; a region may be larger than its view).
 * Test / diagnostic taps, views of the saved forward activations (named after the oracle's cache keys), per layer:
 * "xn1","attn_out","x_mid","xn2","mlp_out" [B,N,D], "h" (fc1 output before the GELU), "g" [B,N,F], "mean1","rstd1",
 * "mean2","rstd2" [B,N]; per model: "x_last" (the last block's output), "x_final_norm" [B,N,D].  attribute() leaves
 * every saved forward activation as the forward wrote it.
 * Returns a device pointer, 4 dims and 4 element strides (unused dims are 1).  Host-only address arithmetic: nothing on
 * the device is read. */
TE_API int te_vit_tensor(const te_vit_config* cfg, int batch, void* workspace, const char* name, int layer,
                  float** ptr, long long dims[4], long long strides[4]);
/* method="full" (ViT_LRP.py:337-343): relevance carried through ``self.add`` (tokens + pos_embed), ``[:, 1:]``,
 * PatchEmbed.relprop (:238-242) and the z^B rule of the patch convolution (layers_ours.py:242-259).
 * Call after te_vit_forward + te_vit_attribute(flags | TE_FLAG_RELPROP_TO_INPUT) on the same workspace and images.
 * flags: those of that te_vit_attribute call; TE_FLAG_RULES_LRP selects the layers_lrp Add rule for self.add.relprop
 * (baselines/ViT/ViT_orig_LRP.py, method="full").
 * pixel_maps [batch, img, img] (channels summed — what relprop returns) and / or pixel_relevance
 * [batch, in_chans, img, img] (Conv2d.relprop's own output) are written when non-NULL. */
TE_API int te_vit_relprop_pixels(const te_vit_config* cfg, const float* weights, const float* images, int batch,
                                 unsigned flags, float* pixel_maps, float* pixel_relevance, void* workspace,
                                 long long workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * BERT sequence classifier  (BERT_explainability/modules/BERT/BertForSequenceClassification.py:12-88,
 * BERT.py:533-651; transformers.BertConfig fields)
 * ---------------------------------------------------------------------------------------------- */
typedef struct te_bert_config {
    int vocab_size;       /* 30522 */
    int max_position;     /* 512 */
    int type_vocab;       /* 2 */
    int hidden;           /* 768 */
    int layers;           /* 12 */
    int heads;            /* 12 */
    int intermediate;     /* 3072 */
    int num_labels;       /* 2 */
    float layer_norm_eps; /* 1e-12 */
} te_bert_config;

/* flat fp32 weight buffer keyed by the HF state_dict names (query|key|value of a layer are adjacent and are
 * used as one packed [3*hidden, hidden] weight); derived = tensor-core copies as for ViT. */
TE_API int te_bert_num_weights(const te_bert_config* cfg);
TE_API const char* te_bert_weight_name(const te_bert_config* cfg, int i);
TE_API long long te_bert_weight_numel(const te_bert_config* cfg, int i);
TE_API long long te_bert_weight_offset(const te_bert_config* cfg, int i);
TE_API long long te_bert_weight_total(const te_bert_config* cfg);
TE_API long long te_bert_derived_total(const te_bert_config* cfg);
TE_API int te_bert_prepare_derived(const te_bert_config* cfg, const float* weights, float* derived, void* stream);
TE_API long long te_bert_workspace_bytes(const te_bert_config* cfg, int batch, int seq);

/* model(input_ids, attention_mask)[0]: ids / mask are int64 [batch, seq] (device); token_type_ids = 0,
 * position_ids = arange(seq) as in BERT.py:69-75; logits [batch, num_labels] (may be NULL). */
TE_API int te_bert_forward(const te_bert_config* cfg, const float* weights, const float* derived,
                    const long long* input_ids, const long long* attention_mask, int batch, int seq, unsigned flags,
                    float* logits, void* workspace, long long workspace_bytes, void* stream);
/* The rest of Generator.generate_LRP (ExplanationGenerator.py:33-59): arg-max (index[b] < 0), one-hot, class
 * gradient of every attention_probs, relprop (BertForSequenceClassification.relprop), relu(grad*cam) head mean,
 * +I, row-normalised rollout from start_layer, row 0 with element 0 replaced by the row minimum.
 * maps [batch, seq].  alpha: model.relprop(cam, alpha=alpha) (BertForSequenceClassification.py:83-88), the LRP-alpha-beta
 * Linear rule as for te_vit_attribute; a non-finite alpha returns TE_ERR_ARG. */
TE_API int te_bert_attribute(const te_bert_config* cfg, const float* weights, const float* derived, int batch, int seq,
                             int* index, int start_layer, float alpha, unsigned flags, float* maps, void* workspace,
                             long long workspace_bytes, void* stream);
/* te_bert_forward + te_bert_attribute (alpha = 1). */
TE_API int te_bert_explain(const te_bert_config* cfg, const float* weights, const float* derived,
                    const long long* input_ids, const long long* attention_mask, int batch, int seq, int* index,
                    int start_layer, unsigned flags, float* maps, float* logits, void* workspace,
                    long long workspace_bytes, void* stream);
/* get_attn / get_attn_gradients / get_attn_cam of BertSelfAttention (BERT.py:281-297):
 * name in {"attn","attn_grad","attn_cam","hidden","logits","relevance_in"} and the scratch regions "tmp_d0".."tmp_d3",
 * "tmp_f0","tmp_f1", "tmp_3d0","tmp_3d1" as for te_vit_tensor.
 * Test / diagnostic taps, views of the saved forward activations, per layer: "qkv" [B,S,3D], "ctx", "d1" (attention
 * output dense), "s1" (= d1 + hidden, the input of the attention-output LayerNorm), "ao" (its output), "d2" (output
 * dense), "s2" (= d2 + ao) [B,S,D], "hpre" (intermediate dense before the GELU), "g" [B,S,F], "mean1","rstd1","mean2",
 * "rstd2" [B,S]; per model: "h_last" [B,S,D], "pooled" [B,D]. */
TE_API int te_bert_tensor(const te_bert_config* cfg, int batch, int seq, void* workspace, const char* name, int layer,
                   float** ptr, long long dims[4], long long strides[4]);

/* ------------------------------------------------------------------------------------------------
 * Stand-alone LRP rules (modules/layers_ours.py) — the same kernels the engine chains, exported so
 * that each rule can be parity-tested against the reference layer class it replaces.
 * ---------------------------------------------------------------------------------------------- */
/* Linear.relprop(R, alpha) (layers_ours.py:207-230): x [rows,in], w [out,in], r [rows,out] -> out [rows,in].
 * alpha: the LRP-alpha-beta rule for any finite alpha, beta = alpha - 1, R_in = alpha * act - beta * inh; inh is act with the
 * weight signs swapped: x+ * (S_i W-) + x- * (S_i W+) with S_i = sd(R, x+ W-^T + x- W+^T).  alpha = 1 is the z+ rule; a
 * non-finite alpha returns TE_ERR_ARG.
 * y / bias: the Linear's saved forward output y = x W^T + bias [rows,out] (what the engines do; bias may be NULL, no bias),
 * or y = NULL.  With y and TE_FLAG_ZPLUS_TENSOR_CORES the denominator is formed in ONE tensor-core pass through the exact
 * identity x+ W+^T + x- W-^T == ((y - bias) + |x| |W|^T) / 2, and the variant flags TE_FLAG_ZPLUS_BF16, _S1_BF16 and _R_F16
 * apply; without y the denominator takes two passes and those flags are not read.
 * flags & TE_FLAG_RULES_LRP: the layers_lrp variant (modules/layers_lrp.py:187-210, separate denominators: each of the
 * four products over its own), which does not read y / bias; on the tensor cores with TE_FLAG_RULES_LRP_TC as well (in, out
 * multiples of 128; other shapes run the fp32 SIMT rule).
 * scratch: rows*out floats; with TE_FLAG_ZPLUS_TENSOR_CORES (layers_ours) or TE_FLAG_RULES_LRP | TE_FLAG_RULES_LRP_TC:
 * round_up(rows*out,64) + 16*in*out floats (S, the derived weight copies), + rows*in floats with y (the tf32(|x|) operand of
 * the single-pass kernel). */
TE_API int te_linear_relprop(const float* x, const float* w, const float* bias, const float* y, const float* r, float* out,
                             float* scratch, int rows, int in_features, int out_features, float alpha, unsigned flags,
                             void* stream);
/* Add.relprop (layers_ours.py:97-120) per sample: x1,x2,r [batch,per_sample] -> r1,r2.
 * scratch: batch*48 doubles; scratch == NULL selects the layers_lrp variant (modules/layers_lrp.py:48-60,98-100:
 * r1 = x1*sd(r, x1+x2), r2 = x2*sd(r, x1+x2), no ratio normalisation). */
TE_API int te_add_relprop(const float* x1, const float* x2, const float* r, float* r1, float* r2, void* scratch,
                   int batch, long long per_sample, void* stream);
/* Clone.relprop (layers_ours.py:151-169): out = x * (sd(r1,x)+sd(r2,x)[+sd(r3,x)]); r3 may be NULL. */
TE_API int te_clone_relprop(const float* x, const float* r1, const float* r2, const float* r3, float* out, long long n,
                     void* stream);
/* einsum('bhij,bhjd->bhid').relprop (layers_ours.py:48-60,122-127): p [bh,n,n], v [bh,n,d], r [bh,n,d]
 * -> rp [bh,n,n], rv [bh,n,d]  (UN-halved).  scratch: bh*n*d floats. */
TE_API int te_matmul_av_relprop(const float* p, const float* v, const float* r, float* rp, float* rv, float* scratch,
                         int bh, int n, int d, void* stream);
/* einsum('bhid,bhjd->bhij').relprop: q,k [bh,n,d], r [bh,n,n] -> rq, rk [bh,n,d] (UN-halved).
 * scratch: bh*n*n floats. */
TE_API int te_matmul_qk_relprop(const float* q, const float* k, const float* r, float* rq, float* rk, float* scratch,
                         int bh, int n, int d, void* stream);
/* IndexSelect.relprop for token 0 (layers_ours.py:129-147): x [b,n,d], r [b,d] -> out [b,n,d]. */
TE_API int te_index_select_relprop(const float* x, const float* r, float* out, int batch, int n, int d, void* stream);
/* Conv2d.relprop, 3-channel-input (z^B) branch (layers_ours.py:242-259) for a kernel == stride patch convolution, as
 * called by PatchEmbed.relprop (ViT_LRP.py:238-242).  images [batch, in_chans, img, img]; weight [dim, in_chans*patch*patch];
 * r [batch, (img/patch)^2, dim] (token-major: the ``cam`` PatchEmbed.relprop receives).  r_pixels [batch,in_chans,img,img]
 * and / or r_sum [batch,img,img] (channel sum) are written when non-NULL.  Min / max are taken per sample. */
TE_API long long te_patch_embed_relprop_workspace_bytes(int batch, int in_chans, int img_size, int patch_size, int dim);
TE_API int te_patch_embed_relprop(const float* images, const float* weight, const float* r, int batch, int in_chans,
                           int img_size, int patch_size, int dim, float* r_pixels, float* r_sum, void* workspace,
                           long long workspace_bytes, void* stream);

/* generate_visualization's tensor part (example.ipynb:57-60): maps [batch, grid*grid] -> reshape grid x grid -> bilinear
 * x scale (align_corners=False) -> per-sample min-max normalisation -> out [batch, grid*scale, grid*scale].  As with the
 * notebook's t.min() / t.max(), a NaN in a sample's map makes all of that sample NaN, and a constant map gives 0 / 0 = NaN. */
TE_API int te_relevance_heatmap(const float* maps, int batch, int grid, int scale, float* out, void* stream);
/* The notebooks' JET overlay (Transformer_explainability.ipynb: generate_visualization, show_cam_on_image), bit for bit the
 * numpy / cv2 sequence per sample: images [batch, 3, h, w] fp32 (the normalised input), heat [batch, h, w] fp32 (min-max
 * normalised, e.g. te_relevance_heatmap's output) -> out [batch, h, w, 3] uint8 BGR:
 *   img = (x - min) / (max - min) over the sample;  u = (uint8)(255.f * heat) (truncation, NaN -> 0);
 *   otsu: t = cv2's THRESH_OTSU value of u (fp64, getThreshVal_Otsu_8u), thresholds[b] = t when thresholds is not NULL,
 *         u = u > t ? 255 : 0;
 *   cam = JET_BGR[u] / 255.f + img (BGR colour channel k plus RGB image channel k, as the notebook adds them);
 *   out[y, x, 2 - k] = (uint8)(255.f * (cam_k / max(cam))) (truncation, NaN -> 0: a constant image renders as 0).
 * batch >= 1, h, w >= 1 (3 h w < 2^31), images / heat / out non-NULL and otsu 0 or 1, else TE_ERR_ARG before anything is
 * launched.  One launch, no workspace. */
TE_API int te_render_overlay(const float* images, const float* heat, int batch, int h, int w, int otsu, unsigned char* out,
                             int* thresholds, void* stream);
/* Head reductions of attention-shaped tensors [batch, heads, n, ld] -> out [batch, n, n] (contiguous), the building
 * block of the secondary methods (ViT_LRP.py:345-398; ViT_explanation_generator.py:51-83; BERT
 * ExplanationGenerator.py:61-155):   v_h = a_h (* g_h if g) (* head_w[b,h] if head_w);
 *   mode 0: mean_h v_h          mode 1: mean_h relu(v_h)  ("clamp(min=0).mean")      mode 2: relu(mean_h v_h).
 * g has a's layout (row stride ld), head_w is [batch, heads]; the pad columns [n, ld) are never read. */
TE_API int te_head_reduce(const float* a, const float* g, const float* head_w, int batch, int heads, int n, int ld, int mode,
                   float* out, void* stream);
/* out[b,h] = mean of g[b,h, r0:r1, c0:c1]  (``grad.mean(dim=[1,2])`` of the GradCAM baselines); the region must satisfy
 * 0 <= r0 < r1 <= n and 0 <= c0 < c1 <= n, else TE_ERR_ARG before anything is launched. */
TE_API int te_head_region_mean(const float* g, int batch, int heads, int n, int ld, int r0, int r1, int c0, int c1, float* out,
                        void* stream);

/* ------------------------------------------------------------------------------------------------
 * Aggregation + rollout  (ViT_LRP.py:357-368, :38-49 ; ExplanationGenerator.py:47-59, :7-18)
 * ---------------------------------------------------------------------------------------------- */
/* grad, cam: [layers, batch, heads, n, ld] (ld >= n row stride).  Computes
 * M_l = mean_h relu(grad_l*cam_l) + I (rows normalised if normalize), J = M_{L-1}...M_{start};
 * joint [batch,n,n] (may be NULL) receives J, row0 [batch,n] (may be NULL) receives J[:,0,:]. */
TE_API long long te_rollout_workspace_bytes(int layers, int batch, int n);
TE_API int te_attribution_rollout(const float* grad, const float* cam, int layers, int batch, int heads, int n, int ld,
                           int start_layer, int normalize, unsigned flags, float* joint, float* row0,
                           void* workspace, long long workspace_bytes, void* stream);
/* compute_rollout_attention(all_layer_matrices, start_layer): mats [layers,batch,n,n] -> joint [batch,n,n]. */
TE_API int te_compute_rollout_attention(const float* mats, int layers, int batch, int n, int start_layer, int normalize,
                                 float* joint, void* workspace, long long workspace_bytes, void* stream);

/* The operand format of the fp16-split forward Linear (TE_FLAG_LINEAR_F16_SPLIT) — exported for unit tests of the format: x [rows, cols]
 * -> hi, lo fp16 [rows, cols] (hi = fp16(2^e x), lo = fp16(2^e x - hi)) and scale_inv [rows, ceil(cols / 128)] = 2^-e, one e per row
 * and 128 columns chosen so that 2^e max|x| lies in [2^14, 2^15) (e = 0 for an all-zero or non-finite block).  cols % 4 == 0. */
TE_API int te_f16_block_split(const float* x, int rows, int cols, void* hi, void* lo, float* scale_inv, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Diagnostic entry points — exported for kernel unit tests only.  Each runs the named tensor-core kernel (or kernel family)
 * directly: a shape or epilogue that kernel does not take returns TE_ERR_UNSUPPORTED with a te_last_error() message, never a
 * fall-back to another kernel, so a call that succeeds has run the kernel it asked for.
 * ---------------------------------------------------------------------------------------------- */
/* Linear GEMMs with their fused epilogues, through the engines' own kernel selection: forward y = x W^T, x [rows,in],
 * w [out,in]; backward dx = dy W, dy [rows,out].  epi: 0 STORE (y = x W^T), 1 BIAS (+ bias), 2 BIAS_GELU (y2 = erf-GELU(y)
 * as well), 3 BIAS_ADD (y2 = e0 + y as well); backward 0 STORE (dx = dy W), 4 GELU_BWD (dx = (dy W) * GELU'(e0)).  e0 / y2
 * share the row stride of y (dx).  flags select the family: 0 fp32 SIMT; TE_FLAG_LINEAR_TENSOR_CORES 3xTF32;
 * + TE_FLAG_LINEAR_F16_SPLIT (forward) fp16 split; + TE_FLAG_BACKWARD_TF32 / TE_FLAG_BACKWARD_F16 (backward) single-pass
 * TF32 / fp16.  scratch (may be NULL for SIMT): 16*in*out floats for the derived weight copies; with the fp16 split
 * + round_up(rows*in,64) + rows*ceil(in/128) floats; with TE_FLAG_BACKWARD_F16 + round_up(rows*out/2,64) + rows*ceil(out/128)
 * floats. */
TE_API int te_linear_forward(const float* x, const float* w, const float* bias, const float* e0, float* y, float* y2,
                             float* scratch, int rows, int in_features, int out_features, int epi, unsigned flags,
                             void* stream);
TE_API int te_linear_backward(const float* dy, const float* w, const float* e0, float* dx, float* scratch, int rows,
                              int in_features, int out_features, int epi, unsigned flags, void* stream);
/* LayerNorm over the last dimension of x [rows, D] (D % 4 == 0) that also emits the fp16-split operand of y in the format of
 * te_f16_block_split: y [rows, D], mean / rstd [rows] (each may be NULL), hi, lo fp16 [rows, D] with lo == hi + rows*D,
 * scale_inv [rows, ceil(D / 128)]. */
TE_API int te_layernorm_split(const float* x, const float* w, const float* b, float* y, float* mean, float* rstd, void* hi,
                              void* lo, float* scale_inv, int rows, int D, float eps, void* stream);
/* S = safe_divide(r, Z) of the z+ Linear rule on the single-pass tensor-core S kernel, Z formed from the saved forward output
 * y = x W^T + bias [rows, out] (bias may be NULL).  Either s (S TF32-rounded, fp32 [rows, out]) or s16 + s16_scale (S as
 * hi-only block-scaled fp16 [rows, out], scale_inv [rows, out / 128] chosen as in te_f16_block_split: the operand of the fp16
 * second contraction, TE_FLAG_ZPLUS_R_F16).  flags: 0 or TE_FLAG_ZPLUS_S1_BF16.  in, out multiples of 128.
 * scratch: 16*in*out + rows*in floats. */
TE_API int te_tc_zplus_s(const float* x, const float* w, const float* bias, const float* y, const float* r, float* s, void* s16,
                         float* s16_scale, float* scratch, int rows, int in_features, int out_features, unsigned flags,
                         void* stream);
/* Attention-shaped N x N contraction on head slices of packed activations:
 * out[b,h,i,j] = epi(alpha * sum_d A[b*n+i, h*dh+d] B[b*n+j, h*dh+d]), out / E [batch, heads, n, ld_out].
 * epi: 0 STORE, 1 MUL (* E), 2 SD (safe_divide(E, .)), 3 SOFTMAX (over j; n <= 256).  Columns n .. round_up(n,4)-1 are written as
 * zeros; the columns from round_up(n,4) to ld_out are not touched.  dh in {32, 64}; single_pass (STORE / MUL): one TF32 MMA per
 * k-step instead of the 3xTF32 split. */
TE_API int te_tc_attention_nn(const float* A, long long lda, const float* B, long long ldb, int batch, int heads, int n, int dh,
                              float* out, int ld_out, const float* E, float alpha, int epi, int single_pass, void* stream);
/* Attention-shaped N x 64 contraction reduced over tokens: out[b*n+m, h*64+d] = epi(alpha * sum_k M_h[m,k] X[b*n+k, h*64+d]) with
 * M_h = map[b,h] (amn 0) or its transpose (amn 1); map [batch, heads, n, np] (np % 4 == 0, np >= n; its padding columns are
 * never read), X / out / E packed rows of stride ldx / ld_out.  epi: 0 STORE, 1 MUL (* E). */
TE_API int te_tc_attention_nk(const float* map, int np, int amn, const float* X, long long ldx, int batch, int heads, int n,
                              float* out, int ld_out, const float* E, float alpha, int epi, int single_pass, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Perturbation evaluation  (baselines/ViT/pertubation_eval_from_hdf5.py:17-23,57-68,88-118)
 * ---------------------------------------------------------------------------------------------- */
#define TE_PERTURB_MAX_STEPS 64
#define TE_PERTURB_MAX_CHANNELS 16
/* Workspace of te_perturb_images for `batch` samples of `pixels` pixels (one threshold pair per sample and step). */
TE_API long long te_perturb_workspace_bytes(int batch, long long pixels);
/* Every perturbed, normalised input of a batch in one call: images [batch, channels, pixels] (raw, in [0, 1]), saliency
 * [batch, pixels], host ks[steps] non-decreasing pixel counts in [0, pixels], host mean / std [channels] ->
 * out [steps, batch, channels, pixels] (step-major: step i is one contiguous forward batch).
 * Order key v = negate ? -s : s; pixels are ordered NaN first, then by descending v, then by ascending pixel index (-0 == +0).
 * Pixel p is removed at step i iff its position in that order is < ks[i], and
 *   out[i,b,c,p] = ((removed ? 0 : images[b,c,p]) - mean[c]) / std[c]    (fp32 subtract, then IEEE division)
 * = normalize(data.clone().scatter_(-1, topk(v, ks[i]).indices, 0)) of the reference with its choice among tied values fixed.
 * steps <= TE_PERTURB_MAX_STEPS, channels <= TE_PERTURB_MAX_CHANNELS. */
TE_API int te_perturb_images(const float* images, const float* saliency, int batch, int channels, long long pixels,
                             const int* ks, int steps, int negate, const float* mean, const float* std, float* out,
                             void* workspace, long long workspace_bytes, void* stream);
/* Per row of logits [rows, classes] (classes >= 2) with target [rows] (int32, device): pred = first index of the maximum,
 * max_logit, max_prob = the largest fp32 softmax probability, dissim = log(p_target / p_second) with p_second the
 * second-largest probability counting duplicates (topk(2)[0][:, 1]), in fp32 as the reference writes it (an underflowed
 * p_target gives -inf, an underflowed p_second +inf; a target outside [0, classes) gives NaN). */
TE_API int te_logit_stats(const float* logits, const int* target, int rows, int classes, int* pred, float* max_logit,
                          float* max_prob, float* dissim, void* stream);
/* Per row of logits [rows, classes] (classes >= 1): probs = the fp32 softmax, with torch.softmax's arithmetic (the row
 * maximum subtracted, expf, the sum, one division per entry).  A row holding a NaN gives a NaN row. */
TE_API int te_class_probs(const float* logits, int rows, int classes, float* probs, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Segmentation evaluation  (baselines/ViT/imagenet_seg_eval.py:212-277,312-314; utils/metrices.py)
 * A sort key is bits(score) << 1 | is_positive for a score >= 0 (-0 is mapped to +0): ascending keys are ascending scores,
 * and bit-equal scores form one contiguous run.
 * ---------------------------------------------------------------------------------------------- */
/* Workspace of te_sort_keys_u32 for n keys in `segments` equal segments (n % segments == 0, n / segments < 2^31). */
TE_API long long te_sort_workspace_bytes(long long n, int segments);
/* Stable LSD radix sort of uint32 keys, ascending, each of the `segments` equal segments of keys_in [n] on its own ->
 * keys_out [n] (keys_out == keys_in is allowed).  Bit-exact: the output is numpy's stable sort of each segment. */
TE_API int te_sort_keys_u32(const unsigned* keys_in, unsigned* keys_out, long long n, int segments, void* workspace,
                            long long workspace_bytes, void* stream);
/* Workspace of te_seg_metrics. */
TE_API long long te_seg_workspace_bytes(int batch, int grid, int scale);
/* Per sample of maps [batch, grid*grid] and labels [batch, P] (int32, 0 / 1), P = (grid*scale)^2:
 *   Res = bilinear x scale of the map (the arithmetic of te_relevance_heatmap; scale 1: the map as given), min-max
 *   normalised in fp32; mean[b] = the mean of Res (fp64 accumulation, one rounding to fp32); a pixel is foreground iff
 *   Res > mean.  counts[b] = (TP, FP, FN, TN) of that mask against label 1, row_counts [batch, grid*scale, 3] = (TP, FP, FN)
 *   of each image row (the reference's F1 is taken per row, utils/metrices.py:26-38); ap[b] = sklearn's average_precision_score of the
 *   2P scores (1 - Res, Res) against the one-hot label, in fp64; pr_keys [batch, P] (may be NULL) = the keys of
 *   clamp(Res, min=thr) / max(Res), positive on label 1.
 *   A degenerate map (max == min, or NaN in it) sets degenerate[b] = 1: every pixel is background, every AP and PR score 0.
 *   invalid[b] = the number of labels other than 0 / 1 (the results of such a sample are meaningless).
 * Needs 4 * grid^2 (scale > 1 only) + 12 * grid * scale <= 45056 (shared memory). */
TE_API int te_seg_metrics(const float* maps, const int* labels, int batch, int grid, int scale, float thr, float* mean,
                          long long* counts, int* row_counts, double* ap, int* degenerate, long long* invalid, unsigned* pr_keys,
                          void* workspace, long long workspace_bytes, void* stream);
/* Workspace of te_pr_curve for n keys. */
TE_API long long te_pr_curve_workspace_bytes(long long n);
/* sklearn's _binary_clf_curve over n keys sorted ascending (te_sort_keys_u32): one entry per distinct score, in descending
 * score order: thresholds (fp32), tps = positives with score >= threshold, fps = negatives with score >= threshold (int64).
 * The outputs need room for n entries; *count (device) receives the number written. */
TE_API int te_pr_curve(const unsigned* keys, long long n, float* thresholds, long long* tps, long long* fps, long long* count,
                       void* workspace, long long workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * ERASER rationale evaluation  (BERT_rationale_benchmark/models/pipeline/bert_pipeline.py:96-138,547-582;
 * BERT_rationale_benchmark/metrics.py:111-215)
 * ---------------------------------------------------------------------------------------------- */
#define TE_ERASER_MAX_WORDS 1024
#define TE_ERASER_MAX_KS 64
#define TE_ERASER_MAX_THRESHOLDS 8
/* Workspace of te_eraser_rationales for `words` word ranges and `spans` truth spans over `batch` documents. */
TE_API long long te_eraser_workspace_bytes(int batch, long long words, long long spans);
/* Per document b of maps [batch, seq] (device, padded rows), over its W = word_offsets[b+1] - word_offsets[b] words
 * (W <= TE_ERASER_MAX_WORDS) and its truth spans [span_offsets[b], span_offsets[b+1]):
 *   word_scores[w] = max over the word's pieces p in [first, last] (piece_ranges [words, 2]) of clamp(maps[b, p], min=0); a
 *     NaN piece makes the word NaN (np.max);
 *   the words are ranked NaN first, then by descending score, then by ascending word index (-0 == +0: the order key of
 *     te_perturb_images); order[b, r] = the word at rank r for r < min(kmax, W), -1 up to kmax = ks[nk-1];
 *   counts [batch, nk, 3 + nthr] (int32), over the first n = min(ks[i], W) ranks: n, tok_hits = words inside any truth
 *     span (start <= w < end), span_hits = words whose one-word span [w, w+1) is a truth span, and per threshold t
 *     iou_hits = words whose best IoU (1 / len of the shortest truth span holding w, 0 if none; fp64) is >= thresholds[t].
 * word_offsets, piece_ranges, span_offsets, spans [.., 2], ks (non-decreasing, nk <= TE_ERASER_MAX_KS) and thresholds
 * (fp64, nthr <= TE_ERASER_MAX_THRESHOLDS) are host arrays, validated before anything is launched: every piece range must
 * satisfy 0 <= first <= last < seq and every span 0 <= start <= end, else TE_ERR_ARG. */
TE_API int te_eraser_rationales(const float* maps, int batch, int seq, const int* word_offsets, const int* piece_ranges,
                                const int* span_offsets, const int* spans, const int* ks, int nk, const double* thresholds,
                                int nthr, float* word_scores, int* order, int* counts, void* workspace,
                                long long workspace_bytes, void* stream);

/* ERASER faithfulness inputs (metrics.py:284-364: comprehensiveness, sufficiency and their AOPC bins) */
#define TE_ERASER_MAX_SELECTIONS 64
#define TE_ERASER_MAX_SEQ 8192
/* Workspace of te_eraser_reduce_inputs for `words` word ranges over `batch` documents and `selections` sizes. */
TE_API long long te_eraser_reduce_workspace_bytes(int batch, long long words, int selections);
/* Per document b of maps [batch, seq] (device, padded rows) and input_ids [batch, seq] (int64, device), with its length
 * lengths[b] (the row is [CLS] p_1 ... p_n [SEP] at positions 0 .. lengths[b] - 1) and its W words (piece ranges as for
 * te_eraser_rationales): the words are ranked exactly as te_eraser_rationales ranks them, each inner piece carries the
 * smallest rank of the words whose range holds it, and for each selection size n = n_select[b, j] (0 <= n <= W):
 *   out_ids[b, j, 0] (comprehensiveness) = [CLS], every inner piece (positions 1 .. lengths[b] - 2) of rank >= n, [SEP];
 *   out_ids[b, j, 1] (sufficiency)       = [CLS], every inner piece of rank < n, [SEP];
 * both in position order and zero past their lengths out_len[b, j, 0 / 1] (int32; the two sum to lengths[b] + 2).
 * lengths, word_offsets, piece_ranges and n_select [batch, selections] are host arrays, validated before anything is
 * launched: 2 <= lengths[b] <= seq, every range 1 <= first <= last <= lengths[b] - 2, W <= TE_ERASER_MAX_WORDS,
 * 0 <= n <= W, selections <= TE_ERASER_MAX_SELECTIONS and seq <= TE_ERASER_MAX_SEQ, else TE_ERR_ARG. */
TE_API int te_eraser_reduce_inputs(const float* maps, const long long* input_ids, int batch, int seq, const int* lengths,
                                   const int* word_offsets, const int* piece_ranges, const int* n_select, int selections,
                                   long long* out_ids, int* out_len, void* workspace, long long workspace_bytes,
                                   void* stream);

/* ERASER soft-token scores (metrics.py:217-253: score_soft_tokens) */
/* Workspace of te_eraser_soft_scores for `spans` truth spans over `batch` documents. */
TE_API long long te_eraser_soft_workspace_bytes(int batch, long long spans);
/* Per document b, over its W = word_offsets[b+1] - word_offsets[b] word scores word_scores[word_offsets[b] ..] (device,
 * the layout te_eraser_rationales writes; W <= TE_ERASER_MAX_WORDS), its truth spans [span_offsets[b], span_offsets[b+1])
 * (word w < W is positive iff some span has start <= w < end) and its tail tail_counts[b] = (positives, negatives) of
 * the words past truncation, which score 0:
 *   the soft prediction is the W scores followed by the tail's zeros; the words are ranked as te_eraser_rationales ranks
 *   them, bit-equal scores (-0 == +0) form one tie group, and the tail joins the group of score 0 (or follows the last
 *   group when no word scores 0).  With P positives and N negatives in all and each group's cumulative (tps, fps) in
 *   descending score order (sklearn's _binary_clf_curve), in fp64:
 *   scores[b, 0] = auc(recall, precision) of precision_recall_curve (recall tps / P, or 1 when P = 0; precision
 *     tps / (tps + fps); the point (0, 1) first), the trapezoid area;
 *   scores[b, 1] = average_precision_score: the sum over groups of (recall step) * precision;
 *   scores[b, 2] = roc_auc_score: the trapezoid area under (fps / N, tps / P) from (0, 0), from an integer sum
 *     (roc_curve's dropped collinear points change only its rounding); NaN when P = 0 or N = 0;
 *   flags[b, 0] = 1 when P = 0 or N = 0 (a single-class document), flags[b, 1] = 1 when a word score is NaN or
 *     negative: then all three scores are NaN and only flags[b, 0] is meaningful besides.
 * word_offsets, span_offsets, spans [.., 2] and tail_counts [batch, 2] are host arrays, validated before anything is
 * launched: offsets from 0, W <= TE_ERASER_MAX_WORDS, every span 0 <= start <= end, tail counts >= 0 with sum <= 2^30, and
 * W + the tail >= 1 per document, else TE_ERR_ARG. */
TE_API int te_eraser_soft_scores(const float* word_scores, int batch, const int* word_offsets, const int* span_offsets,
                                 const int* spans, const int* tail_counts, double* scores, int* flags, void* workspace,
                                 long long workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Input preparation  (baselines/ViT/generate_visualizations.py:194-199: Resize((224, 224)) + ToTensor() on PIL images)
 * Pillow's 8-bit bilinear resize (ImagingResample, support 1): per axis scale = in / out, fs = max(scale, 1), and for output
 * index i, center = (i + 0.5) scale, xmin = max((int)(center - fs + 0.5), 0), n = min((int)(center + fs + 0.5), in) - xmin,
 * weights tri((j + xmin - center + 0.5) * (1 / fs)) divided by their (double) sum, as int32 (int)(+-0.5 + w 2^22).  Each pass starts
 * an int32 accumulator at 2^21, sums u8 * k and clips to uint8 (>= 255 << 22: 255, <= 0: 0, else >> 22); the first pass's
 * uint8 result feeds the second.  The horizontal pass runs first, except when h > 100 w and out_h < h (Pillow 12's
 * Image.resize then resizes vertically first).
 * ---------------------------------------------------------------------------------------------- */
#define TE_PREPARE_MAX_SIDE 16384
#define TE_PREPARE_MAX_OUT 4096
/* Host only: the table of one axis resized from in_size (1..TE_PREPARE_MAX_SIDE) to out_size (1..TE_PREPARE_MAX_OUT)
 * samples.  Returns ksize = 2 ceil(max(in / out, 1)) + 1 (or TE_ERR_ARG); when k and bounds are given, k [out_size, ksize]
 * receives the int32 weights (zero past n) and bounds [out_size, 2] the pairs (xmin, n). */
TE_API int te_resize_coeffs(int in_size, int out_size, int* k, int* bounds);
/* Workspace of te_prepare_images for `batch` images no taller than max_in_h and no wider than max_in_w. */
TE_API long long te_prepare_images_workspace_bytes(int batch, int max_in_h, int max_in_w, int out_h, int out_w);
/* A ragged batch of RGB uint8 images, each HWC and contiguous at byte offsets[b] of packed (device, packed_bytes long),
 * of sizes [batch, 2] = (h, w) (host; sides 1..TE_PREPARE_MAX_SIDE), resized to out_h x out_w (1..TE_PREPARE_MAX_OUT) as
 * Pillow's Image.resize((out_w, out_h), BILINEAR) does, bit for bit:
 *   out01 [batch, 3, out_h, out_w]    = u8 / 255.f (IEEE division): ToTensor() of the resized image;
 *   out_norm [batch, 3, out_h, out_w] = (out01 - mean[c]) / std[c] in fp32 (host mean / std [3], finite, std != 0).
 * Either output may be NULL (not both).  sizes and offsets are validated before anything is launched: every image must lie
 * inside packed, else TE_ERR_ARG.  One host-to-device copy (image descriptors and the tables of te_resize_coeffs) and two
 * launches per batch, whatever the image sizes. */
TE_API int te_prepare_images(const unsigned char* packed, long long packed_bytes, int batch, const int* sizes,
                             const long long* offsets, int out_h, int out_w, const float* mean, const float* std,
                             float* out01, float* out_norm, void* workspace, long long workspace_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TE_B200_H */
