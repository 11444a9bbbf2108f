// The notebooks' relevance overlay (Transformer_explainability.ipynb: generate_visualization + show_cam_on_image), bit for
// bit the numpy / cv2 sequence on the host:
//   img = (x - min) / (max - min)                  over the 3 h w values of the sample, fp32, IEEE division
//   u   = (uint8)(255.f * heat)                    truncation, NaN -> 0 (a constant relevance map is NaN after min-max)
//   otsu: t = cv2's THRESH_OTSU value of u (getThreshVal_Otsu_8u, fp64), u = u > t ? 255 : 0
//   cam = JET_BGR[u] / 255.f + img                 channel k of the BGR colour plus channel k of the RGB image
//   out[y, x, 2 - k] = (uint8)(255.f * (cam_k / max(cam)))            cv2.cvtColor(RGB2BGR) of np.uint8(255 * vis)
// render_overlay_kernel: one block of kThreads per sample and no workspace.  Passes: image min / max (and the histogram of u
// in shared memory when thresholding), Otsu's loop on one thread, max(cam), then the write pass; cam is recomputed rather
// than stored.  Per pixel 16 bytes are needed (12 of image, 4 of heat) and 3 written; the image is read three times and the
// heat two or three times, the rereads mostly from L2.  This file is compiled without fast math and every rounding step
// is spelled out: the fp32 divisions are IEEE, and the Otsu loop uses __dmul_rn / __dadd_rn so that no FMA is contracted.
#include <cfloat>

#include "../../include/te_b200.h"
#include "te_kernels.h"

namespace {

constexpr int kThreads = 1024;

// cv2.COLORMAP_JET as uint8 BGR.  JET is piecewise linear: channel c (1 = blue, 2 = green, 3 = red) of level u is
// clip(1.5 - |4 u / 255 - c|, 0, 1); times 255 that is k2 / 2 with the integer k2 = clip(765 - 2 |4 u - 255 c|, 0, 510).
// cv2 rounds its fp32 samples of the curve to nearest, so the half-way values (k2 odd) go to the even neighbour; the one
// exception is u = 159 in blue (k2 = 3), where cv2's table holds 1, not 2 (tests/test_render.py checks all 256 entries).
__device__ __forceinline__ int jet_bgr(int u, int k) {
    const int c = k + 1;
    const int d = 4 * u - 255 * c;
    int k2 = 765 - 2 * (d < 0 ? -d : d);
    k2 = k2 < 0 ? 0 : (k2 > 510 ? 510 : k2);
    if (u == 159 && k == 0) return 1;
    const int lo = k2 >> 1;
    return (k2 & 1) ? lo + (lo & 1) : lo;
}

// numpy's float32 -> uint8 cast on x86-64 for values in [0, 256): truncation, NaN -> 0
__device__ __forceinline__ int to_u8(float v) { return v != v ? 0 : (__float2int_rz(v) & 255); }

// np.min / np.max: a NaN anywhere makes the result NaN
__device__ __forceinline__ float nan_min(float a, float b) { return a != a ? a : (b != b || b < a ? b : a); }
__device__ __forceinline__ float nan_max(float a, float b) { return a != a ? a : (b != b || b > a ? b : a); }

template <bool kMax>
__device__ float block_reduce(float v, float* red) {
    for (int o = 16; o > 0; o >>= 1) {
        const float w = __shfl_xor_sync(0xffffffffu, v, o);
        v = kMax ? nan_max(v, w) : nan_min(v, w);
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    __syncthreads();                                     // red may still be read by a previous reduction
    if (lane == 0) red[warp] = v;
    __syncthreads();
    v = red[0];
    for (int i = 1; i < kThreads / 32; ++i) v = kMax ? nan_max(v, red[i]) : nan_min(v, red[i]);
    return v;
}

// OpenCV's getThreshVal_Otsu_8u over the 256-bin histogram of `total` pixels, every step rounded as the host's SSE2 code
__device__ int otsu_threshold(const int* h, int total) {
    const double scale = 1.0 / (double)total;
    double mu = 0.0;
    for (int i = 0; i < 256; ++i) mu = __dadd_rn(mu, __dmul_rn((double)i, (double)h[i]));
    mu = __dmul_rn(mu, scale);
    double mu1 = 0.0, q1 = 0.0, max_sigma = 0.0;
    int max_val = 0;
    for (int i = 0; i < 256; ++i) {
        const double p_i = __dmul_rn((double)h[i], scale);
        mu1 = __dmul_rn(mu1, q1);
        q1 = __dadd_rn(q1, p_i);
        const double q2 = __dadd_rn(1.0, -q1);
        if (fmin(q1, q2) < (double)FLT_EPSILON || fmax(q1, q2) > 1.0 - (double)FLT_EPSILON) continue;
        mu1 = __ddiv_rn(__dadd_rn(mu1, __dmul_rn((double)i, p_i)), q1);
        const double mu2 = __ddiv_rn(__dadd_rn(mu, -__dmul_rn(q1, mu1)), q2);
        const double d = __dadd_rn(mu1, -mu2);
        const double sigma = __dmul_rn(__dmul_rn(__dmul_rn(q1, q2), d), d);
        if (sigma > max_sigma) {
            max_sigma = sigma;
            max_val = i;
        }
    }
    return max_val;
}

__global__ void __launch_bounds__(kThreads) render_overlay_kernel(const float* __restrict__ images,
                                                                  const float* __restrict__ heat, int hw, int otsu,
                                                                  unsigned char* __restrict__ out, int* __restrict__ thresholds) {
    __shared__ float jet[256 * 3];
    __shared__ int hist[256];
    __shared__ float red[kThreads / 32];
    __shared__ int s_thr;
    const long long b = blockIdx.x;
    const float* img = images + b * 3 * hw;
    const float* ht = heat + b * hw;
    for (int i = threadIdx.x; i < 256 * 3; i += kThreads) jet[i] = (float)jet_bgr(i / 3, i % 3) / 255.f;
    for (int i = threadIdx.x; i < 256; i += kThreads) hist[i] = 0;
    __syncthreads();

    float mn = INFINITY, mx = -INFINITY;
    for (int i = threadIdx.x; i < 3 * hw; i += kThreads) {
        const float v = img[i];
        mn = nan_min(mn, v);
        mx = nan_max(mx, v);
    }
    if (otsu)
        for (int p = threadIdx.x; p < hw; p += kThreads) atomicAdd(&hist[to_u8(255.f * ht[p])], 1);
    mn = block_reduce<false>(mn, red);
    mx = block_reduce<true>(mx, red);
    if (otsu && threadIdx.x == 0) {
        s_thr = otsu_threshold(hist, hw);
        if (thresholds) thresholds[b] = s_thr;
    }
    __syncthreads();
    const int thr = otsu ? s_thr : 0;
    const float den = mx - mn;

    float cmax = -INFINITY;
    for (int p = threadIdx.x; p < hw; p += kThreads) {
        int u = to_u8(255.f * ht[p]);
        if (otsu) u = u > thr ? 255 : 0;
#pragma unroll
        for (int k = 0; k < 3; ++k) cmax = nan_max(cmax, __fadd_rn(jet[u * 3 + k], __fdiv_rn(img[k * hw + p] - mn, den)));
    }
    cmax = block_reduce<true>(cmax, red);

    unsigned char* o = out + b * 3 * hw;
    for (int p = threadIdx.x; p < hw; p += kThreads) {
        int u = to_u8(255.f * ht[p]);
        if (otsu) u = u > thr ? 255 : 0;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float cam = __fadd_rn(jet[u * 3 + k], __fdiv_rn(img[k * hw + p] - mn, den));
            o[3LL * p + 2 - k] = (unsigned char)to_u8(__fmul_rn(255.f, __fdiv_rn(cam, cmax)));
        }
    }
}

}  // namespace

#define REQ(c, msg) do { if (!(c)) { te_set_last_error(msg); return TE_ERR_ARG; } } while (0)

extern "C" int te_render_overlay(const float* images, const float* heat, int batch, int h, int w, int otsu,
                                 unsigned char* out, int* thresholds, void* stream) {
    REQ(images && heat && out, "te_render_overlay: null argument");
    REQ(batch >= 1, "te_render_overlay: batch must be at least 1");
    REQ(h >= 1 && w >= 1, "te_render_overlay: h and w must be at least 1");
    REQ(3LL * h * w <= 0x7fffffffLL, "te_render_overlay: 3 h w must fit in int32");
    REQ(otsu == 0 || otsu == 1, "te_render_overlay: otsu must be 0 or 1");
    render_overlay_kernel<<<batch, kThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(images, heat, h * w, otsu, out,
                                                                                          thresholds);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
