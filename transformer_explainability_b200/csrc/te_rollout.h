// Aggregation + rollout:  M_l = mean_h relu(G_l * cam_l) + I  (/rowsum) ;  J = M_{L-1} ... M_{start}
// (ViT_LRP.py:357-368, :38-49 ; BERT ExplanationGenerator.py:47-59, :7-18)
#pragma once
#include "te_common.cuh"

// G0 / cam0: layer-0 tensors [B,H,N,ld_in]; layer l lives at +l*layer_stride floats.
// mats [L,B,N,ld], joint_a / joint_b [B,N,ld] scratch.  joint_out [B,N,N] and row_out [B,N-first] optional.
// flags & 2: row-only consumers get the fused streaming kernel; a dense joint is chained on the tensor cores (diag [L,B,N] scratch
// is needed for that when normalize != 0).
int te_rollout_layers(const float* G0, const float* cam0, long long layer_stride, int L, int B, int H, int N,
                      int ld_in, int ld, int start_layer, int normalize, unsigned flags, float* mats, float* joint_a, float* joint_b,
                      float* joint_out, float* row_out, int first, int bert_fix, cudaStream_t st, float* diag = nullptr);
// chain only: mats [L,B,N,ld] already hold the (+I, normalised) matrices
int te_rollout_chain(const float* mats, int L, int B, int N, int ld, int start_layer, float* joint_a, float* joint_b,
                     const float** result, cudaStream_t st);
