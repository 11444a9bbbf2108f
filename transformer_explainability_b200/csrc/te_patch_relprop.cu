// z^B ("box") rule of the first layer: Conv2d.relprop for a 3-channel image (modules/layers_ours.py:242-259) behind
// PatchEmbed.relprop (baselines/ViT/ViT_LRP.py:238-242) — the last step of method="full" (ViT_LRP.py:337-343).
//
// The patch-embedding conv has kernel == stride and no padding, so every conv / conv_transpose of the rule is a GEMM
// over the im2col'd patches X_p [B*np, K] (K = C*P*P) with the flattened weight W [D, K]:
//     conv(x, W)      = X_p W^T                      conv(L, W+) = l_b * rowsum(W+)   (L, H are per-sample constants)
//     convT(S, W)     = S W     (S [B*np, D])        conv(H, W-) = h_b * rowsum(W-)
//     Za = ((X_p W^T - l_b rowsum(W+)) - h_b rowsum(W-)) + 1e-9 ;  S = R / Za
//     C  = x * (S W) - l_b * (S W+) - h_b * (S W-)    scattered back to [B, C, H, W] (and summed over channels)
#include "te_kernels.h"
#include "te_engine_util.h"

#define TE_REQ(c, msg) do { if (!(c)) { te_set_last_error(msg); return TE_ERR_ARG; } } while (0)

namespace {
constexpr int kThreads = 256;

// per-sample min / max of the image (torch.min/max over dims 1,2,3 — layers_ours.py:247-252)
__global__ void image_minmax_kernel(const float* __restrict__ img, float* __restrict__ lo, float* __restrict__ hi,
                                    long long per4) {
    const int b = blockIdx.x;
    const float4* p = reinterpret_cast<const float4*>(img) + b * per4;
    float mn = INFINITY, mx = -INFINITY;
    for (long long t = threadIdx.x; t < per4; t += blockDim.x) {
        const float4 v = p[t];
        mn = fminf(fminf(mn, v.x), fminf(fminf(v.y, v.z), v.w));
        mx = fmaxf(fmaxf(mx, v.x), fmaxf(fmaxf(v.y, v.z), v.w));
    }
    __shared__ float smn[kThreads / 32], smx[kThreads / 32];
    for (int o = 16; o > 0; o >>= 1) {
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    if ((threadIdx.x & 31) == 0) { smn[threadIdx.x >> 5] = mn; smx[threadIdx.x >> 5] = mx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < kThreads / 32; ++i) { mn = fminf(mn, smn[i]); mx = fmaxf(mx, smx[i]); }
        lo[b] = mn; hi[b] = mx;
    }
}

// rowsum(W+), rowsum(W-): one warp per output channel
__global__ void weight_posneg_rowsum_kernel(const float* __restrict__ w, float* __restrict__ spw, float* __restrict__ snw,
                                            int D, int K) {
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= D) return;
    const int lane = threadIdx.x & 31;
    float sp = 0.f, sn = 0.f;
    for (int k = lane; k < K; k += 32) {
        const float v = w[(long long)row * K + k];
        sp += fmaxf(v, 0.f); sn += fminf(v, 0.f);
    }
    sp = te_warp_sum(sp); sn = te_warp_sum(sn);
    if (lane == 0) { spw[row] = sp; snw[row] = sn; }
}

// S = R / Za, in place over z [B*np, D]; r rows addressed as r + b*r_sample_stride + p*D
__global__ void zb_divide_kernel(float* __restrict__ z, const float* __restrict__ r, long long r_sample_stride,
                                 const float* __restrict__ lo, const float* __restrict__ hi,
                                 const float* __restrict__ spw, const float* __restrict__ snw, long long rows, int np,
                                 int D) {
    const long long total = rows * D;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        const int o = (int)(t % D);
        const long long row = t / D;
        const int b = (int)(row / np), p = (int)(row % np);
        const float za = ((z[t] - lo[b] * spw[o]) - hi[b] * snw[o]) + 1e-9f;
        z[t] = r[b * r_sample_stride + (long long)p * D + o] / za;
    }
}

// C = x*T0 - l*T1 - h*T2 scattered from patch layout to the image; one thread per 4 pixels of one channel row
__global__ void zb_combine_kernel(const float* __restrict__ img, const float* __restrict__ t0, const float* __restrict__ t1,
                                  const float* __restrict__ t2, const float* __restrict__ lo, const float* __restrict__ hi,
                                  float* __restrict__ r_pixels, float* __restrict__ r_sum, int B, int C, int H, int W,
                                  int P) {
    const int gw = W / P, gh = H / P, wq = W / 4;
    const long long total = (long long)B * H * wq;
    const long long K = (long long)C * P * P;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        const int xq = (int)(t % wq);
        const long long rt = t / wq;
        const int y = (int)(rt % H);
        const int b = (int)(rt / H);
        const int x = xq * 4, px = x / P, ix = x % P, py = y / P, iy = y % P;
        const long long prow = ((long long)b * gh + py) * gw + px;
        const float l = lo[b], h = hi[b];
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int c = 0; c < C; ++c) {
            const long long po = prow * K + ((long long)c * P + iy) * P + ix;
            const long long io = (((long long)b * C + c) * H + y) * W + x;
            const float4 xv = *reinterpret_cast<const float4*>(img + io);
            const float4 a = *reinterpret_cast<const float4*>(t0 + po);
            const float4 p1 = *reinterpret_cast<const float4*>(t1 + po);
            const float4 p2 = *reinterpret_cast<const float4*>(t2 + po);
            float4 o;
            o.x = (xv.x * a.x - l * p1.x) - h * p2.x;
            o.y = (xv.y * a.y - l * p1.y) - h * p2.y;
            o.z = (xv.z * a.z - l * p1.z) - h * p2.z;
            o.w = (xv.w * a.w - l * p1.w) - h * p2.w;
            if (r_pixels) *reinterpret_cast<float4*>(r_pixels + io) = o;
            acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w;
        }
        if (r_sum) *reinterpret_cast<float4*>(r_sum + ((long long)b * H + y) * W + x) = acc;
    }
}

// the same one pixel at a time, for patches that are not a multiple of 4 wide (four adjacent pixels may span two patches)
__global__ void zb_combine_scalar_kernel(const float* __restrict__ img, const float* __restrict__ t0, const float* __restrict__ t1,
                                         const float* __restrict__ t2, const float* __restrict__ lo, const float* __restrict__ hi,
                                         float* __restrict__ r_pixels, float* __restrict__ r_sum, int B, int C, int H, int W,
                                         int P) {
    const int gw = W / P, gh = H / P;
    const long long total = (long long)B * H * W;
    const long long K = (long long)C * P * P;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        const int x = (int)(t % W);
        const long long rt = t / W;
        const int y = (int)(rt % H);
        const int b = (int)(rt / H);
        const int px = x / P, ix = x % P, py = y / P, iy = y % P;
        const long long prow = ((long long)b * gh + py) * gw + px;
        const float l = lo[b], h = hi[b];
        float acc = 0.f;
        for (int c = 0; c < C; ++c) {
            const long long po = prow * K + ((long long)c * P + iy) * P + ix;
            const long long io = (((long long)b * C + c) * H + y) * W + x;
            const float o = (img[io] * t0[po] - l * t1[po]) - h * t2[po];
            if (r_pixels) r_pixels[io] = o;
            acc += o;
        }
        if (r_sum) r_sum[t] = acc;
    }
}

inline int flat_grid(long long n) {
    long long g = (n + kThreads - 1) / kThreads;
    return (int)(g < 1 ? 1 : (g > 132LL * 16 ? 132LL * 16 : g));
}
}  // namespace

long long te_patch_relprop_scratch_floats(int B, int C, int img, int P, int D) {
    const long long np = (long long)(img / P) * (img / P), K = (long long)C * P * P;
    auto al = [](long long n) { return (n + 63) & ~63LL; };
    return 4 * al(B * np * K) + al(B * np * D) + al(2LL * B) + al(2LL * D);
}

int te_patch_relprop_run(const float* images, const float* weight, const float* r, long long r_sample_stride, int B,
                         int C, int img, int P, int D, float* scratch, float* r_pixels, float* r_sum, cudaStream_t st) {
    TE_REQ(P > 0 && img % P == 0, "patch_relprop: patch must divide the image");
    TE_REQ(((long long)C * img * img) % 4 == 0, "patch_relprop: in_chans * img_size^2 must be a multiple of 4");
    const long long np = (long long)(img / P) * (img / P), K = (long long)C * P * P, rows = (long long)B * np;
    auto al = [](long long n) { return (n + 63) & ~63LL; };
    float* patches = scratch;
    float* t0 = patches + al(rows * K);
    float* t1 = t0 + al(rows * K);
    float* t2 = t1 + al(rows * K);
    float* z = t2 + al(rows * K);
    float* lo = z + al(rows * D);
    float* hi = lo + B;
    float* spw = lo + al(2LL * B);
    float* snw = spw + D;

    TE_TRY(te_launch_im2col(images, patches, B, C, img, img, P, st));
    image_minmax_kernel<<<B, kThreads, 0, st>>>(images, lo, hi, (long long)C * img * img / 4);
    TE_CUDA_CHECK_LAUNCH();
    weight_posneg_rowsum_kernel<<<(D + 7) / 8, kThreads, 0, st>>>(weight, spw, snw, D, (int)K);
    TE_CUDA_CHECK_LAUNCH();
    // Z0 = X_p W^T (bias = None, layers_ours.py:253)
    TE_TRY(te_util::linear_fwd(patches, (int)K, weight, nullptr, z, nullptr, nullptr, rows, (int)K, D, TE_EPI_STORE, st));
    zb_divide_kernel<<<flat_grid(rows * D), kThreads, 0, st>>>(z, r, r_sample_stride, lo, hi, spw, snw, rows, (int)np, D);
    TE_CUDA_CHECK_LAUNCH();
    // gradprop2(S, W), gradprop2(S, W+), gradprop2(S, W-)      (:257)
    for (int which = 0; which < 3; ++which) {
        TeGemm p = te_util::gemm0();
        p.A = z; p.lda = D; p.B = weight; p.ldb = (int)K; p.C = which == 0 ? t0 : (which == 1 ? t1 : t2); p.ldc = (int)K;
        p.M = (int)rows; p.N = (int)K; p.K = D;
        TE_TRY(te_gemm_launch(p, TE_L_K, TE_L_MN, which == 0 ? TE_XF_NONE : (which == 1 ? TE_XF_B_POS : TE_XF_B_NEG),
                              TE_EPI_STORE, st));
    }
    if (P % 4 == 0)
        zb_combine_kernel<<<flat_grid((long long)B * img * (img / 4)), kThreads, 0, st>>>(images, t0, t1, t2, lo, hi, r_pixels,
                                                                                       r_sum, B, C, img, img, P);
    else
        zb_combine_scalar_kernel<<<flat_grid((long long)B * img * img), kThreads, 0, st>>>(images, t0, t1, t2, lo, hi, r_pixels,
                                                                                        r_sum, B, C, img, img, P);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
