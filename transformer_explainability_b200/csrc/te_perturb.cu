// Positive / negative perturbation evaluation (baselines/ViT/pertubation_eval_from_hdf5.py:17-23,57-68,88-118):
//   * te_perturb_images: every perturbed, normalised input of a batch.  Per sample a radix select over order-preserving
//     uint32 keys of the saliency finds, for every step, the key threshold T and the index cut among the keys equal to T
//     (ties broken by ascending pixel index); a grid-wide stream then writes out[S,B,C,P] from one read of x and s.
//   * te_logit_stats: arg-max / max logit / max softmax probability / log(p_target / p_second), one warp per row.
//   * te_class_probs: the fp32 softmax of each row, one warp per row.
#include "../../include/te_b200.h"
#include "te_kernels.h"

namespace {

constexpr int kSelThreads = 512;
constexpr int kSelUnroll = 4;
constexpr int kThreads = 256;

struct PerturbSteps {
    int n;
    int k[TE_PERTURB_MAX_STEPS];
};
struct PerturbNorm {
    float mean[TE_PERTURB_MAX_CHANNELS];
    float std[TE_PERTURB_MAX_CHANNELS];
};

// Order key of a saliency value: larger key = removed earlier.  v = negate ? -s : s; -0 == +0; every NaN maps to the top key
// (torch.sort(descending=True) puts NaN first).  For non-NaN v the map float -> uint32 is strictly increasing.
__device__ __forceinline__ uint32_t perturb_key(float s, bool negate) {
    float v = negate ? -s : s;
    if (v != v) return 0xffffffffu;
    if (v == 0.f) v = 0.f;                                   // canonical +0
    const uint32_t b = __float_as_uint(v);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);      // at most 0xff800000 (+inf): NaN stays strictly on top
}

template <int W> __device__ __forceinline__ void load_w(const float* p, float* v) {
    if constexpr (W == 4) {
        const float4 a = *reinterpret_cast<const float4*>(p);
        v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    } else {
        v[0] = *p;
    }
}
template <int W> __device__ __forceinline__ void store_w(float* p, const float* v) {
    if constexpr (W == 4) __stcs(reinterpret_cast<float4*>(p), make_float4(v[0], v[1], v[2], v[3]));
    else __stcs(p, v[0]);
}

// grid (steps, batch): the k-th largest key T of one sample (4 passes of 8-bit digits, histograms over the keys that share
// the digits chosen so far), then the index cut: pixel p with key == T is removed iff p < cut.  k = 0 removes nothing
// (T = 0xffffffff, cut = 0).  sel[b * MAX_STEPS + i] = (T, cut).
__global__ void __launch_bounds__(kSelThreads) perturb_select_kernel(const float* __restrict__ sal, int P, int B, bool negate,
                                                                     PerturbSteps steps, uint2* __restrict__ sel) {
    const int i = blockIdx.x, b = blockIdx.y;
    const int k = steps.k[i];
    const float* s = sal + (long long)b * P;
    __shared__ uint32_t hist[256];
    __shared__ uint32_t sh_prefix, sh_rem, sh_cut, sh_run;
    __shared__ uint32_t warp_cnt[kSelThreads / 32];
    if (k == 0) {
        if (threadIdx.x == 0) sel[(long long)b * TE_PERTURB_MAX_STEPS + i] = make_uint2(0xffffffffu, 0u);
        return;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t prefix = 0, mask = 0, rem = (uint32_t)k;
    for (int shift = 24; shift >= 0; shift -= 8) {
        for (int j = threadIdx.x; j < 256; j += blockDim.x) hist[j] = 0;
        __syncthreads();
        for (int p0 = 0; p0 < P; p0 += kSelUnroll * blockDim.x) {
            float v[kSelUnroll];
#pragma unroll
            for (int u = 0; u < kSelUnroll; ++u) {                  // kSelUnroll independent loads in flight per thread
                const int p = p0 + u * blockDim.x + threadIdx.x;
                v[u] = p < P ? s[p] : 0.f;
            }
#pragma unroll
            for (int u = 0; u < kSelUnroll; ++u) {
                const bool in = p0 + u * (int)blockDim.x + (int)threadIdx.x < P;
                const uint32_t key = perturb_key(v[u], negate);
                const bool match = in && (key & mask) == prefix;
                const uint32_t digit = match ? (key >> shift) & 255u : 256u + lane;  // non-matching lanes form singleton groups
                const uint32_t peers = __match_any_sync(0xffffffffu, digit);
                if (match && lane == __ffs(peers) - 1) atomicAdd(&hist[digit], (uint32_t)__popc(peers));
            }
        }
        __syncthreads();
        if (warp == 0) {
            // lane l owns the digits 255 - 8l ... 248 - 8l, scanned from the top
            uint32_t c[8], sum = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) { c[j] = hist[255 - 8 * lane - j]; sum += c[j]; }
            uint32_t incl = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            const uint32_t excl = incl - sum;
            if (excl < rem && rem <= incl) {
                uint32_t run = excl;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    if (run < rem && rem <= run + c[j]) {
                        sh_prefix = prefix | ((uint32_t)(255 - 8 * lane - j) << shift);
                        sh_rem = rem - run;
                    }
                    run += c[j];
                }
            }
        }
        __syncthreads();
        prefix = sh_prefix;
        rem = sh_rem;
        mask |= 255u << shift;
        __syncthreads();
    }
    // prefix = T; rem = how many of the keys equal to T are removed, in ascending index order: find the rem-th of them
    if (threadIdx.x == 0) { sh_run = 0; sh_cut = 0xffffffffu; }
    __syncthreads();
    for (int p1 = 0; p1 < P; p1 += kSelUnroll * blockDim.x) {
        float v[kSelUnroll];
#pragma unroll
        for (int u = 0; u < kSelUnroll; ++u) {
            const int p = p1 + u * blockDim.x + threadIdx.x;
            v[u] = p < P ? s[p] : 0.f;
        }
        bool done = false;
#pragma unroll
        for (int u = 0; u < kSelUnroll; ++u) {                      // sub-chunks in index order
            if (done) break;
            const int p = p1 + u * blockDim.x + threadIdx.x;
            const bool eq = p < P && perturb_key(v[u], negate) == prefix;
            const uint32_t bal = __ballot_sync(0xffffffffu, eq);
            if (lane == 0) warp_cnt[warp] = __popc(bal);
            __syncthreads();
            uint32_t before = sh_run;
            for (int w = 0; w < warp; ++w) before += warp_cnt[w];
            before += __popc(bal & ((1u << lane) - 1u));
            if (eq && before + 1 == rem) sh_cut = (uint32_t)p + 1u;
            __syncthreads();
            if (threadIdx.x == 0) {
                uint32_t tot = 0;
                for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += warp_cnt[w];
                sh_run += tot;
            }
            __syncthreads();
            done = sh_cut != 0xffffffffu;
        }
        if (done) break;
    }
    if (threadIdx.x == 0) sel[(long long)b * TE_PERTURB_MAX_STEPS + i] = make_uint2(prefix, sh_cut);
}

// out[i,b,c,p] = ((removed_i(p) ? 0 : x[b,c,p]) - mean[c]) / std[c]: one thread per (sample, W pixels), W = 4 (float4) or 1;
// x and s are read once, every step's threshold pair is a broadcast load
template <int W>
__global__ void perturb_write_kernel(const float* __restrict__ x, const float* __restrict__ sal, int B, int C, int P, bool negate,
                                     int S, PerturbNorm nrm, const uint2* __restrict__ sel, float* __restrict__ out) {
    const int per = P / W;
    const long long total = (long long)B * per;
    const long long sample_stride = (long long)C * P;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(t / per);
        const int p = (int)(t - (long long)b * per) * W;
        float v[W];
        uint32_t key[W];
        load_w<W>(sal + (long long)b * P + p, v);
#pragma unroll
        for (int j = 0; j < W; ++j) key[j] = perturb_key(v[j], negate);
        const uint2* th = sel + (long long)b * TE_PERTURB_MAX_STEPS;
#pragma unroll
        for (int c = 0; c < TE_PERTURB_MAX_CHANNELS; ++c) {           // unrolled: mean / std indexed statically (no stack copy)
            if (c >= C) break;
            load_w<W>(x + b * sample_stride + (long long)c * P + p, v);
            float* o = out + b * sample_stride + (long long)c * P + p;
            for (int i = 0; i < S; ++i) {
                const uint2 tc = th[i];
                float r[W];
#pragma unroll
                for (int j = 0; j < W; ++j) {
                    const bool rm = key[j] > tc.x || (key[j] == tc.x && (uint32_t)(p + j) < tc.y);
                    r[j] = __fdiv_rn(__fsub_rn(rm ? 0.f : v[j], nrm.mean[c]), nrm.std[c]);
                }
                store_w<W>(o + (long long)i * B * sample_stride, r);
            }
        }
    }
}

// one warp per row of logits [R, K]: pred = first arg-max (as argmax_kernel), max logit, softmax maximum 1 / sum exp(l - m1),
// dissim = log(p_target / p_second) with p_second the probability of the second-largest logit counting duplicates
__global__ void logit_stats_kernel(const float* __restrict__ logits, const int* __restrict__ target, int R, int K,
                                   int* __restrict__ pred, float* __restrict__ max_logit, float* __restrict__ max_prob,
                                   float* __restrict__ dissim) {
    const int lane = threadIdx.x & 31;
    const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (r >= R) return;
    const float* l = logits + (long long)r * K;
    // the two largest values m1 >= m2 (a repeated maximum gives m2 = m1) and the first index of m1
    float m1 = -INFINITY, m2 = -INFINITY;
    int i1 = 0x7fffffff;
    for (int j = lane; j < K; j += 32) {
        const float v = l[j];
        if (v > m1) { m2 = m1; m1 = v; i1 = j; }
        else if (v > m2) m2 = v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float a1 = __shfl_xor_sync(0xffffffffu, m1, o);
        const float a2 = __shfl_xor_sync(0xffffffffu, m2, o);
        const int ai = __shfl_xor_sync(0xffffffffu, i1, o);
        if (a1 > m1) { m2 = fmaxf(m1, a2); m1 = a1; i1 = ai; }
        else if (a1 < m1) { m2 = fmaxf(m2, a1); }
        else { m2 = m1; i1 = min(i1, ai); }                  // the maximum occurs in both halves
    }
    float sum = 0.f;
    for (int j = lane; j < K; j += 32) sum += expf(l[j] - m1);
    sum = te_warp_sum(sum);
    if (lane == 0) {
        const int t = target[r];
        const float pt = (t >= 0 && t < K) ? expf(l[t] - m1) / sum : NAN;
        const float p2 = expf(m2 - m1) / sum;
        pred[r] = (i1 == 0x7fffffff) ? 0 : i1;
        max_logit[r] = m1;
        max_prob[r] = 1.f / sum;
        dissim[r] = logf(pt / p2);
    }
}

// one warp per row of logits [R, K]: torch.softmax (maximum subtracted, expf, sum, divide); fmaxf skips a NaN, whose
// expf term then makes the sum and every probability of the row NaN
__global__ void class_probs_kernel(const float* __restrict__ logits, int R, int K, float* __restrict__ probs) {
    const int lane = threadIdx.x & 31;
    const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (r >= R) return;
    const float* l = logits + (long long)r * K;
    float m = -INFINITY;
    for (int j = lane; j < K; j += 32) m = fmaxf(m, l[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float sum = 0.f;
    for (int j = lane; j < K; j += 32) sum += expf(l[j] - m);
    sum = te_warp_sum(sum);
    for (int j = lane; j < K; j += 32) probs[(long long)r * K + j] = expf(l[j] - m) / sum;
}

}  // namespace

#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define REQ(c, msg) do { if (!(c)) { te_set_last_error(msg); return TE_ERR_ARG; } } while (0)

extern "C" long long te_perturb_workspace_bytes(int batch, long long pixels) {
    if (batch <= 0 || pixels <= 0 || pixels > 0x7fffffffLL) return TE_ERR_ARG;
    return ((long long)batch * TE_PERTURB_MAX_STEPS * 8 + 255) / 256 * 256;
}

extern "C" int te_perturb_images(const float* images, const float* saliency, int batch, int channels, long long pixels,
                                 const int* ks, int steps, int negate, const float* mean, const float* std, float* out,
                                 void* workspace, long long workspace_bytes, void* stream) {
    REQ(images && saliency && out && ks && mean && std, "te_perturb_images: null argument");
    REQ(batch > 0 && pixels > 0 && pixels <= 0x7fffffffLL, "te_perturb_images: batch and pixels must be positive");
    REQ(channels > 0 && channels <= TE_PERTURB_MAX_CHANNELS, "te_perturb_images: channels outside 1..TE_PERTURB_MAX_CHANNELS");
    REQ(steps > 0 && steps <= TE_PERTURB_MAX_STEPS, "te_perturb_images: steps outside 1..TE_PERTURB_MAX_STEPS");
    const int P = (int)pixels;
    PerturbSteps st;
    st.n = steps;
    for (int i = 0; i < steps; ++i) {
        REQ(ks[i] >= 0 && ks[i] <= P, "te_perturb_images: every k must lie in [0, pixels]");
        REQ(i == 0 || ks[i] >= ks[i - 1], "te_perturb_images: ks must be non-decreasing");
        st.k[i] = ks[i];
    }
    PerturbNorm nrm;
    for (int c = 0; c < TE_PERTURB_MAX_CHANNELS; ++c) {
        nrm.mean[c] = c < channels ? mean[c] : 0.f;
        nrm.std[c] = c < channels ? std[c] : 1.f;
    }
    REQ(workspace && (((uintptr_t)workspace) & 255u) == 0, "te_perturb_images: workspace null or not 256-byte aligned");
    if (te_perturb_workspace_bytes(batch, pixels) > workspace_bytes) {
        te_set_last_error("te_perturb_images: workspace too small");
        return TE_ERR_WORKSPACE;
    }
    uint2* sel = reinterpret_cast<uint2*>(workspace);
    perturb_select_kernel<<<dim3(steps, batch), kSelThreads, 0, ST(stream)>>>(saliency, P, batch, negate != 0, st, sel);
    TE_CUDA_CHECK_LAUNCH();
    const bool vec = (P % 4 == 0) && ((((uintptr_t)images) | ((uintptr_t)saliency) | ((uintptr_t)out)) & 15u) == 0;
    const long long units = (long long)batch * (vec ? P / 4 : P);
    const long long blocks = (units + kThreads - 1) / kThreads;
    const int grid = (int)(blocks < 132LL * 16 ? blocks : 132LL * 16);
    if (vec)
        perturb_write_kernel<4><<<grid, kThreads, 0, ST(stream)>>>(images, saliency, batch, channels, P, negate != 0, steps, nrm,
                                                                   sel, out);
    else
        perturb_write_kernel<1><<<grid, kThreads, 0, ST(stream)>>>(images, saliency, batch, channels, P, negate != 0, steps, nrm,
                                                                   sel, out);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}

extern "C" int te_logit_stats(const float* logits, const int* target, int rows, int classes, int* pred, float* max_logit,
                              float* max_prob, float* dissim, void* stream) {
    REQ(logits && target && pred && max_logit && max_prob && dissim, "te_logit_stats: null argument");
    REQ(rows > 0 && classes >= 2, "te_logit_stats: rows > 0 and classes >= 2 expected");
    const int warps = kThreads / 32;
    logit_stats_kernel<<<(rows + warps - 1) / warps, kThreads, 0, ST(stream)>>>(logits, target, rows, classes, pred, max_logit,
                                                                                 max_prob, dissim);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}

extern "C" int te_class_probs(const float* logits, int rows, int classes, float* probs, void* stream) {
    REQ(logits && probs, "te_class_probs: null argument");
    REQ(rows > 0 && classes >= 1, "te_class_probs: rows > 0 and classes >= 1 expected");
    const int warps = kThreads / 32;
    class_probs_kernel<<<(rows + warps - 1) / warps, kThreads, 0, ST(stream)>>>(logits, rows, classes, probs);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
