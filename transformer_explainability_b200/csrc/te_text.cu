// Word importance of the BERT notebook (BERT_explainability.ipynb): token_kernel, one block per row, the row's NaN-aware
// min / max over its first L tokens by a block reduction, then (a - min) / (max - min) and the sign of the explained class
// with one explicit IEEE fp32 rounding per operation.
#include "../../include/te_b200.h"
#include "te_kernels.h"

namespace {

constexpr int kTokenThreads = 256;

// row b: a = maps[b, :L]; mn / mx = min / max of a, NaN when any entry is NaN (torch.min / torch.max); w = 0 for a constant
// row (mx == mn, false for NaN), else ((a - mn) / (mx - mn)) * sign[b]; zeros past L.
__global__ void __launch_bounds__(kTokenThreads) token_kernel(const float* __restrict__ maps, const int* __restrict__ lengths,
                                                              const float* __restrict__ sign, int seq,
                                                              float* __restrict__ out) {
    __shared__ float smn[kTokenThreads / 32], smx[kTokenThreads / 32];
    __shared__ int snan[kTokenThreads / 32];
    const int b = blockIdx.x;
    const int L = min(max(lengths[b], 0), seq);
    const float* row = maps + (long long)b * seq;
    float* o = out + (long long)b * seq;
    const float inf = __int_as_float(0x7f800000);
    float mn = inf, mx = -inf;
    int nan = 0;
    for (int p = threadIdx.x; p < L; p += kTokenThreads) {
        const float v = row[p];
        if (v != v) nan = 1;
        else { mn = fminf(mn, v); mx = fmaxf(mx, v); }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int s = 16; s; s >>= 1) {
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, s));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, s));
        nan |= __shfl_xor_sync(0xffffffffu, nan, s);
    }
    if (lane == 0) { smn[warp] = mn; smx[warp] = mx; snan[warp] = nan; }
    __syncthreads();
    mn = smn[0]; mx = smx[0]; nan = snan[0];
    for (int u = 1; u < kTokenThreads / 32; ++u) {
        mn = fminf(mn, smn[u]);
        mx = fmaxf(mx, smx[u]);
        nan |= snan[u];
    }
    if (nan) mn = mx = __int_as_float(0x7fc00000);
    const float range = __fsub_rn(mx, mn);
    const float sg = sign[b];
    for (int p = threadIdx.x; p < seq; p += kTokenThreads) {
        float w = 0.f;
        if (p < L && !(mx == mn)) w = __fmul_rn(__fdiv_rn(__fsub_rn(row[p], mn), range), sg);
        o[p] = w;
    }
}

}  // namespace

extern "C" int te_token_importance(const float* maps, const int* lengths, const float* sign, int batch, int seq, float* out,
                                   void* stream) {
    if (!maps || !lengths || !sign || !out) {
        te_set_last_error("te_token_importance: null argument");
        return TE_ERR_ARG;
    }
    if (batch <= 0 || batch > 65535 || seq <= 0) {
        te_set_last_error("te_token_importance: batch must lie in 1..65535 and seq be positive");
        return TE_ERR_ARG;
    }
    token_kernel<<<batch, kTokenThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(maps, lengths, sign, seq, out);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
