// Fused aggregation + rollout (row-only).  HBM-bound by construction: per explanation it reads
// 2*(L-start)*H*N*ld*4 bytes (G and cam, once) and writes N floats.
//
// Mapping: a cluster of K CTAs (K in {1,2,4,8}, chosen so that B*K covers the 132 SMs about twice) owns one
// sample; warp w of CTA c owns rows i = c + K*w, + K*nwarps, ...  For its row a warp issues 2*6 independent
// 128-bit loads per lane (6 heads of G and cam) before consuming them, keeps the head-mean of the row in
// registers, and accumulates r[i] * (m_i + e_i) into a per-warp register accumulator.  Per layer: one
// shared-memory reduction over the warps of a CTA and one distributed-shared-memory reduction over the cluster.
#include <cooperative_groups.h>

#include "te_rollout_fused.h"

namespace cg = cooperative_groups;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kHeadGroup = 6;

template <int NCHUNK>
__global__ void __launch_bounds__(kThreads, 2)
rollout_row_kernel(const float* __restrict__ G0, const float* __restrict__ cam0, long long layer_stride, int L, int H,
                   int N, int ld, int start, int normalize, int first, int bert_fix, float* __restrict__ out) {
    constexpr int NPAD = NCHUNK * 128;
    cg::cluster_group cluster = cg::this_cluster();
    const int K = (int)cluster.num_blocks();
    const int crank = (int)cluster.block_rank();
    const int b = blockIdx.x / K;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    __shared__ __align__(16) float r[NPAD];              // current row vector
    __shared__ __align__(16) float part[NPAD];           // this CTA's partial of the next row vector
    __shared__ __align__(16) float wacc[kWarps][NPAD];   // per-warp partials

    for (int j = threadIdx.x; j < NPAD; j += kThreads) r[j] = (j == 0) ? 1.f : 0.f;
    __syncthreads();

    const float invH = 1.0f / (float)H;
    for (int l = L - 1; l >= start; --l) {
        const float* Gl = G0 + l * layer_stride + (long long)b * H * N * ld;
        const float* Cl = cam0 + l * layer_stride + (long long)b * H * N * ld;
        float acc[NCHUNK][4];
#pragma unroll
        for (int c = 0; c < NCHUNK; ++c) { acc[c][0] = acc[c][1] = acc[c][2] = acc[c][3] = 0.f; }

        for (int i = crank + K * warp; i < N; i += K * kWarps) {
            float m[NCHUNK][4];
#pragma unroll
            for (int c = 0; c < NCHUNK; ++c) { m[c][0] = m[c][1] = m[c][2] = m[c][3] = 0.f; }
            for (int h0 = 0; h0 < H; h0 += kHeadGroup) {
#pragma unroll
                for (int c = 0; c < NCHUNK; ++c) {
                    const int col = c * 128 + lane * 4;
                    float4 g[kHeadGroup], q[kHeadGroup];
#pragma unroll
                    for (int hh = 0; hh < kHeadGroup; ++hh) {
                        g[hh] = make_float4(0.f, 0.f, 0.f, 0.f);
                        q[hh] = g[hh];
                        if (h0 + hh < H && col < ld) {
                            const long long o = ((long long)(h0 + hh) * N + i) * ld + col;
                            g[hh] = __ldcs(reinterpret_cast<const float4*>(Gl + o));      // streamed once: evict-first
                            q[hh] = __ldcs(reinterpret_cast<const float4*>(Cl + o));
                        }
                    }
#pragma unroll
                    for (int hh = 0; hh < kHeadGroup; ++hh) {
                        m[c][0] += fmaxf(g[hh].x * q[hh].x, 0.f);
                        m[c][1] += fmaxf(g[hh].y * q[hh].y, 0.f);
                        m[c][2] += fmaxf(g[hh].z * q[hh].z, 0.f);
                        m[c][3] += fmaxf(g[hh].w * q[hh].w, 0.f);
                    }
                }
            }
            float rs = 0.f;
#pragma unroll
            for (int c = 0; c < NCHUNK; ++c)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int col = c * 128 + lane * 4 + e;
                    m[c][e] = (col < N) ? m[c][e] * invH : 0.f;      // pad columns hold garbage: select, not multiply
                    rs += m[c][e];
                }
            float wgt = r[i];
            if (normalize) {
                rs = te_warp_sum(rs) + 1.0f;                         // row sum of (M + I)
                wgt = wgt / rs;
            }
#pragma unroll
            for (int c = 0; c < NCHUNK; ++c)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int col = c * 128 + lane * 4 + e;
                    acc[c][e] = fmaf(wgt, m[c][e] + ((col == i) ? 1.0f : 0.0f), acc[c][e]);
                }
        }
#pragma unroll
        for (int c = 0; c < NCHUNK; ++c)
            *reinterpret_cast<float4*>(&wacc[warp][c * 128 + lane * 4]) = make_float4(acc[c][0], acc[c][1], acc[c][2], acc[c][3]);
        __syncthreads();
        for (int j = threadIdx.x; j < NPAD; j += kThreads) {
            float s = 0.f;
#pragma unroll
            for (int w = 0; w < kWarps; ++w) s += wacc[w][j];
            part[j] = s;
        }
        cluster.sync();                                              // partials of every CTA of the sample are ready
        for (int j = threadIdx.x; j < NPAD; j += kThreads) {
            float s = 0.f;
            for (int k = 0; k < K; ++k) s += cluster.map_shared_rank(part, k)[j];
            r[j] = s;
        }
        cluster.sync();                                              // nobody still reads `part` / everyone has r
    }
    if (crank == 0) {
        __shared__ float mn_s;
        if (bert_fix) {
            if (warp == 0) {
                float mn = INFINITY;
                for (int j = lane; j < N; j += 32) mn = fminf(mn, r[j]);
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
                if (lane == 0) mn_s = mn;
            }
            __syncthreads();
        }
        float* o = out + (long long)b * (N - first);
        for (int j = first + threadIdx.x; j < N; j += kThreads) o[j - first] = (bert_fix && j == 0) ? mn_s : r[j];
    }
}

template <int NCHUNK>
int launch(const float* G0, const float* cam0, long long layer_stride, int L, int B, int H, int N, int ld, int start,
           int normalize, float* out, int first, int bert_fix, int K, cudaStream_t st) {
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(B * K);
    cfg.blockDim = dim3(kThreads);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = K;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    cudaError_t e = cudaLaunchKernelEx(&cfg, rollout_row_kernel<NCHUNK>, G0, cam0, layer_stride, L, H, N, ld, start,
                                       normalize, first, bert_fix, out);
    te_count_launch();
    if (e != cudaSuccess) { te_set_last_error(cudaGetErrorString(e)); return TE_ERR_CUDA; }
    return TE_OK;
}

}  // namespace

bool te_rollout_fused_supported(int N, int ld_in, int) {
    return N >= 1 && ld_in >= N && ld_in <= 512 && (ld_in % 4) == 0;
}

int te_rollout_fused_row(const float* G0, const float* cam0, long long layer_stride, int L, int B, int H, int N,
                         int ld_in, int start_layer, int normalize, float* row_out, int first, int bert_fix,
                         cudaStream_t st) {
    if (!te_rollout_fused_supported(N, ld_in, ld_in) || (((uintptr_t)G0 | (uintptr_t)cam0) & 15u) || (layer_stride % 4)) {
        te_set_last_error("fused rollout: unsupported shape or alignment");
        return TE_ERR_UNSUPPORTED;
    }
    int K = 1;
    while (K < 8 && B * K < 264) K *= 2;                            // ~2 CTAs per SM over 132 SMs
    if (ld_in <= 128) return launch<1>(G0, cam0, layer_stride, L, B, H, N, ld_in, start_layer, normalize, row_out, first, bert_fix, K, st);
    if (ld_in <= 256) return launch<2>(G0, cam0, layer_stride, L, B, H, N, ld_in, start_layer, normalize, row_out, first, bert_fix, K, st);
    return launch<4>(G0, cam0, layer_stride, L, B, H, N, ld_in, start_layer, normalize, row_out, first, bert_fix, K, st);
}
