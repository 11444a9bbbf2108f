// Internal launcher prototypes (C++ side).  The public C ABI lives in include/te_b200.h.
#pragma once
#include "te_common.cuh"
#include "te_gemm.cuh"

// ---- embedding -------------------------------------------------------------------------------
int te_launch_im2col(const float* img, float* patches, int B, int C, int H, int W, int P, cudaStream_t st);
int te_launch_assemble_tokens(const float* patch_out, const float* cls, const float* dist, const float* pos,
                              float* x, int B, int N, int D, int n_prefix, cudaStream_t st);
// ---- normalisation ---------------------------------------------------------------------------
int te_launch_layernorm(const float* x, const float* w, const float* b, float* y, float* mean, float* rstd,
                        long long rows, int D, float eps, cudaStream_t st);
// same, also emitting the block-scaled fp16 (hi, lo) split of y for the fp16-split Linear that consumes it (te_tc_wgmma.cu):
// split = [hi | lo] fp16 [rows, D] (rows*D floats), scale [rows, ceil(D/128)]
int te_launch_layernorm_split(const float* x, const float* w, const float* b, float* y, float* mean, float* rstd,
                              long long rows, int D, float eps, float* split, float* scale, cudaStream_t st);
int te_launch_layernorm_bwd(const float* dy, const float* x, const float* w, const float* mean, const float* rstd,
                            const float* dres, float* dx, long long rows, int D, cudaStream_t st);
// rows of dy / x / dx addressed as base + row*row_stride (used for the CLS-only final norm)
int te_launch_layernorm_bwd_strided(const float* dy, long long dy_stride, const float* x, long long x_stride,
                                    const float* w, float eps, float* dx, long long dx_stride, int rows, int D,
                                    cudaStream_t st);
// ---- softmax ---------------------------------------------------------------------------------
int te_launch_softmax(float* s, long long rows, int N, int ld, cudaStream_t st);
int te_launch_softmax_bwd(const float* p, const float* dp, float* ds, long long rows, int N, int ld, float scale,
                          cudaStream_t st);
// ---- head / seed -----------------------------------------------------------------------------
// only_negative: overwrite index[b] only where it is < 0 (caller-supplied class indices are kept)
int te_launch_argmax(const float* logits, int* index, int B, int C, int only_negative, cudaStream_t st);
int te_launch_average2(const float* a, const float* b, float* out, long long n, cudaStream_t st);
int te_launch_onehot(const int* index, float* seed, int B, int C, float value, cudaStream_t st);
// sim[b] = ls cos(x_b, t_b) (sim may be NULL), seed[b] = ls (t^_b - cos x^_b) / |x_b|; x, t, seed [B, E]
int te_launch_similarity_seed(const float* x, const float* t, float logit_scale, float* sim, float* seed, int B, int E,
                              cudaStream_t st);
// ---- LRP elementwise rules ---------------------------------------------------------------------
int te_launch_sd(const float* a, const float* b, float* out, long long n, cudaStream_t st);
int te_launch_clone_relprop(const float* x, const float* r1, const float* r2, const float* r3, float* out,
                            long long n, cudaStream_t st);
// Add rule with per-sample reductions; partial must hold B*TE_ADD_SPLIT*3 doubles.
#define TE_ADD_SPLIT 16
int te_launch_add_relprop(const float* x1, const float* x2, const float* r, float* r1, float* r2, double* partial,
                          int B, long long per_sample, cudaStream_t st);
// partial == NULL selects the layers_lrp variant (modules/layers_lrp.py:48-60,98-100): r1 = x1*sd(r,x1+x2), r2 = x2*sd(...)
// same with x2 addressed as x2 + b*x2_sample_stride (0: one tensor shared by every sample, e.g. pos_embed); r2 may be null
int te_launch_add_relprop_strided(const float* x1, const float* x2, long long x2_sample_stride, const float* r, float* r1,
                                  float* r2, double* partial, int B, long long per_sample, cudaStream_t st);
// ---- first layer: Conv2d z^B rule behind PatchEmbed.relprop (te_patch_relprop.cu) ------------------
long long te_patch_relprop_scratch_floats(int B, int C, int img, int P, int D);
// r: relevance of the patch tokens, row (b, p) at r + b*r_sample_stride + p*D.  r_pixels [B,C,img,img] and / or
// r_sum [B,img,img] (channels summed) are written when non-null.
int te_patch_relprop_run(const float* images, const float* weight, const float* r, long long r_sample_stride, int B,
                         int C, int img, int P, int D, float* scratch, float* r_pixels, float* r_sum, cudaStream_t st);
// IndexSelect rule: out[b,tok,:] = x*sd(r,x), zero elsewhere.  r is [B,D] per token slot.
int te_launch_index_select_relprop(const float* x, const float* r_tok0, const float* r_tok1, float* out, int B,
                                   int N, int D, cudaStream_t st);
// ---- aggregation / rollout ---------------------------------------------------------------------
// M[b] = mean_h relu(G*cam) (+I) (row-normalised if normalize) ; G, cam [B,H,N,ld_in] ; M [B,N,ld_out]
// diag (with add_eye = 0, normalize = 1): identity kept out of M, its normalised weight 1/rowsum written to diag [B*N]
int te_launch_aggregate(const float* G, const float* cam, float* M, int B, int H, int N, int ld_in, int ld_out,
                        int add_eye, int normalize, cudaStream_t st, float* diag = nullptr);
// every layer first_layer .. first_layer+num_layers-1 in one launch (vectorised layouts only): layer first_layer keeps its
// identity inside M, the others are written in the residual form (identity left out, its normalised weight in diag)
int te_launch_aggregate_layers(const float* G0, const float* cam0, long long in_layer_stride, float* M0, long long m_layer_stride,
                               int B, int H, int N, int ld_in, int ld_out, int first_layer, int num_layers, int normalize,
                               cudaStream_t st, float* diag0 = nullptr);
// generate_visualization: [B, g*g] -> bilinear x scale -> per-sample min-max -> [B, g*scale, g*scale]
int te_launch_relevance_heatmap(const float* maps, float* out, int B, int g, int scale, cudaStream_t st);
// secondary methods: out[b,i,j] = reduce_h( a (* g) (* hw[b,h]) ); mode 0 mean, 1 mean of relu, 2 relu of mean
int te_launch_head_reduce(const float* a, const float* g, const float* hw, float* out, int B, int H, int N, int ld,
                          int mode, cudaStream_t st);
int te_launch_head_region_mean(const float* g, float* out, int BH, int N, int ld, int r0, int r1, int c0, int c1,
                               cudaStream_t st);
int te_launch_prep_mats(const float* in, float* out, long long rows, int N, int ld_in, int ld_out, int normalize,
                        cudaStream_t st);
int te_launch_extract_row(const float* joint, float* out, int B, int N, int ld, int first, int bert_fix,
                          cudaStream_t st);
int te_launch_fill(float* p, float v, long long n, cudaStream_t st);
// ---- BERT extras -------------------------------------------------------------------------------
int te_launch_softmax_masked(float* s, long long rows, int N, int ld, const float* keymask, long long rows_per_batch,
                             cudaStream_t st);
// ids outside [0, vocab) and token types outside [0, type_vocab) never index a table: their rows are written as NaN.
// token_type_ids == NULL: every token is segment 0.
int te_launch_bert_embed(const long long* ids, const long long* token_type_ids, const float* word, const float* pos,
                         const float* type, float* out, int B, int S, int D, int vocab, int type_vocab, cudaStream_t st);
// RoBERTa / DistilBERT embeddings, one launch.  pad >= 0: RoBERTa position ids (pad + running count of ids != pad for
// non-pad tokens, pad for pad tokens) and (word + type) + position; pad < 0: arange and, with type == NULL (DistilBERT),
// word + position.  token_type_ids == NULL: segment 0.  An id, token type or position outside its table gives a NaN row.
int te_launch_hf_embed(const long long* ids, const long long* token_type_ids, const float* word, const float* pos,
                       const float* type, float* out, int B, int S, int D, int vocab, int max_position, int type_vocab,
                       int pad, cudaStream_t st);
int te_launch_bert_mask(const long long* mask, float* out, long long n, cudaStream_t st);
int te_launch_tanh(const float* x, float* y, long long n, cudaStream_t st);
int te_launch_tanh_bwd(const float* dy, const float* y, float* dx, long long n, cudaStream_t st);
// DistilBERT's head activation: y = relu(x) (NaN stays NaN, as torch.relu); dx = dy where y > 0, else 0
int te_launch_relu(const float* x, float* y, long long n, cudaStream_t st);
int te_launch_relu_bwd(const float* dy, const float* y, float* dx, long long n, cudaStream_t st);
int te_launch_add2(const float* a, const float* b, float* out, long long n, cudaStream_t st);
// Add.relprop for add([scores, key-broadcast mask]); only the scores' relevance is produced.
// partial == NULL selects the layers_lrp variant: r1 = x1 * sd(r, x1 + mask), no ratio normalisation.
int te_launch_add_relprop_keymask(const float* x1, const float* keymask, const float* r, float* r1, double* partial,
                                  int B, int H, int N, int ld, cudaStream_t st);
