// Input preparation of the ViT evaluation commands (baselines/ViT/generate_visualizations.py:194-199: Resize((224, 224)) +
// ToTensor() on PIL images): a ragged batch of decoded RGB uint8 images, packed HWC one after another in one device buffer,
// resized with Pillow's 8-bit bilinear filter (ImagingResample, support 1, 22-bit fixed point, the intermediate image
// rounded to uint8) and written as planar fp32 in [0, 1] and / or normalised.  The horizontal pass runs first, except for
// an image taller than 100 times its width that shrinks vertically: Pillow 12's Image.resize runs that one as a vertical
// resize followed by a horizontal one, and the order changes the rounding of the intermediate.
//   * resize_first_kernel: grid (ceil(rows / kRows), batch), 256 threads, rows = the largest first-pass output height of the
//     batch; a block takes kRows rows of one image's first-pass output (blocks past its height return) and each thread one
//     (row, column) pair at a time, all three channels in int32 accumulators, into the uint8 intermediate ([h, out_w, 3],
//     or [out_h, w, 3] when the vertical pass runs first).
//   * resize_second_kernel: grid (ceil(out_h * out_w / 256), batch), 256 threads; a thread takes one output pixel, runs the
//     other pass over the intermediate and writes out01[b, c, y, x] = u8 / 255.f (IEEE division) and
//     out_norm[b, c, y, x] = (out01 - mean[c]) / std[c].
// Nothing is staged in shared memory: neighbouring threads read neighbouring taps (n, about 2 scale + 1, per output), so a
// warp's reads of the input, the intermediate and the coefficient rows (the same for every row of an image) fall in a few
// L1 lines.  Per image of h x w pixels (horizontal first): 3 h w bytes read, 3 h out_w bytes written and read back
// (L2-resident), 12 out_h out_w bytes written per output, plus the coefficient tables, 4 (out_w (kx + 2) + out_h (ky + 2))
// bytes.  The tables are computed in double on the host (te_resize_coeffs: Pillow's precompute_coeffs and
// normalize_coeffs_8bpc) and copied into the workspace with the image descriptors in one host-to-device copy.
#include <cmath>
#include <cstring>
#include <vector>

#include "../../include/te_b200.h"
#include "te_kernels.h"

namespace {

constexpr int kThreads = 256;
constexpr int kRows = 8;
constexpr int kPrecisionBits = 22;

struct ImageDesc {
    long long in_off;        // byte offset of the image in the packed buffer
    long long mid_off;       // byte offset of its first-pass output in the intermediate
    long long kx_off;        // int offset of its horizontal table: weights [out_w, kx], then bounds [out_w, 2]
    long long ky_off;        // int offset of its vertical table: weights [out_h, ky], then bounds [out_h, 2]
    int h, w, kx, ky;
    int vfirst;              // 1: the vertical pass runs first (Image.resize of an image taller than 100 x its width)
};

struct Norm {
    float mean[3], std[3];
};

__device__ __forceinline__ unsigned char clip8(int s) {
    if (s >= (255 << kPrecisionBits)) return 255;
    if (s <= 0) return 0;
    return (unsigned char)(s >> kPrecisionBits);
}

// One output pixel of a pass: the three channels of sum_j src[j * step] * k[j] over the n taps, from 2^21
__device__ __forceinline__ void resample_px(const unsigned char* __restrict__ src, long long step, const int* __restrict__ k,
                                            int n, int s[3]) {
    s[0] = s[1] = s[2] = 1 << (kPrecisionBits - 1);
    for (int j = 0; j < n; ++j) {
        const int c = k[j];
        const unsigned char* px = src + j * step;
        s[0] += px[0] * c;
        s[1] += px[1] * c;
        s[2] += px[2] * c;
    }
}

// First pass into the uint8 intermediate: horizontal ([h, w] -> [h, out_w]) or, for vfirst, vertical ([h, w] -> [out_h, w])
__global__ void __launch_bounds__(kThreads) resize_first_kernel(const unsigned char* __restrict__ packed,
                                                                const ImageDesc* __restrict__ desc, const int* __restrict__ coef,
                                                                unsigned char* __restrict__ mid, int oh, int ow) {
    const ImageDesc d = desc[blockIdx.y];
    const int R = d.vfirst ? oh : d.h, C = d.vfirst ? d.w : ow;
    const int r0 = blockIdx.x * kRows;
    if (r0 >= R) return;
    const int rows = min(kRows, R - r0);
    const int ks = d.vfirst ? d.ky : d.kx;
    const int* k = coef + (d.vfirst ? d.ky_off : d.kx_off);
    const int* bounds = k + (long long)(d.vfirst ? oh : ow) * ks;
    const unsigned char* img = packed + d.in_off;
    for (int t = threadIdx.x; t < rows * C; t += kThreads) {
        const int rr = t / C, x = t - rr * C, r = r0 + rr;
        const int i = d.vfirst ? r : x;                            // output index along the resampled axis
        const int lo = bounds[2 * i], n = bounds[2 * i + 1];
        const unsigned char* src = img + (d.vfirst ? (long long)lo * d.w + x : (long long)r * d.w + lo) * 3;
        int s[3];
        resample_px(src, d.vfirst ? 3LL * d.w : 3, k + (long long)i * ks, n, s);
        unsigned char* dst = mid + d.mid_off + ((long long)r * C + x) * 3;
        dst[0] = clip8(s[0]);
        dst[1] = clip8(s[1]);
        dst[2] = clip8(s[2]);
    }
}

// Second pass from the intermediate to fp32: vertical ([h, out_w] -> [out_h, out_w]) or, for vfirst, horizontal
__global__ void __launch_bounds__(kThreads) resize_second_kernel(const unsigned char* __restrict__ mid,
                                                                 const ImageDesc* __restrict__ desc, const int* __restrict__ coef,
                                                                 int oh, int ow, Norm nrm, float* __restrict__ out01,
                                                                 float* __restrict__ out_norm) {
    const int b = blockIdx.y;
    const int p = blockIdx.x * kThreads + threadIdx.x;
    if (p >= oh * ow) return;
    const ImageDesc d = desc[b];
    const int y = p / ow, x = p - y * ow;
    const int ks = d.vfirst ? d.kx : d.ky;
    const int* k = coef + (d.vfirst ? d.kx_off : d.ky_off);
    const int* bounds = k + (long long)(d.vfirst ? ow : oh) * ks;
    const int i = d.vfirst ? x : y;
    const int lo = bounds[2 * i], n = bounds[2 * i + 1];
    const unsigned char* src = mid + d.mid_off + (d.vfirst ? (long long)y * d.w + lo : (long long)lo * ow + x) * 3;
    int s[3];
    resample_px(src, d.vfirst ? 3 : 3LL * ow, k + (long long)i * ks, n, s);
    const long long plane = (long long)oh * ow;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float v = (float)clip8(s[c]) / 255.f;
        const long long o = ((long long)b * 3 + c) * plane + p;
        if (out01) out01[o] = v;
        if (out_norm) out_norm[o] = (v - nrm.mean[c]) / nrm.std[c];
    }
}

long long up256(long long n) { return (n + 255) / 256 * 256; }

// Pillow's ksize: 2 ceil(support) + 1 with support = max(in / out, 1) (bilinear support 1)
int kernel_size(int in, int out) {
    double fs = (double)in / out;
    if (fs < 1.0) fs = 1.0;
    return (int)std::ceil(fs) * 2 + 1;
}

// Pillow 12's Image.resize resizes an image taller than 100 times its width vertically first (two separate resizes)
bool vertical_first(int h, int w, int oh) { return h > 100LL * w && oh < h; }

// bytes of the uint8 intermediate of any image no taller than max_h and no wider than max_w
long long mid_bound(int max_h, int max_w, int oh, int ow) {
    const long long a = (long long)max_h * ow, b = (long long)oh * max_w;
    return 3 * (a > b ? a : b);
}

// ints of one image's two tables
long long table_ints(int h, int w, int oh, int ow) {
    return (long long)ow * (kernel_size(w, ow) + 2) + (long long)oh * (kernel_size(h, oh) + 2);
}

}  // namespace

#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define REQ(c, msg) do { if (!(c)) { te_set_last_error(msg); return TE_ERR_ARG; } } while (0)

extern "C" int te_resize_coeffs(int in_size, int out_size, int* k, int* bounds) {
    REQ(in_size >= 1 && in_size <= TE_PREPARE_MAX_SIDE, "te_resize_coeffs: input size outside 1..TE_PREPARE_MAX_SIDE");
    REQ(out_size >= 1 && out_size <= TE_PREPARE_MAX_OUT, "te_resize_coeffs: output size outside 1..TE_PREPARE_MAX_OUT");
    const int ksize = kernel_size(in_size, out_size);
    if (!k && !bounds) return ksize;
    REQ(k && bounds, "te_resize_coeffs: k and bounds must both be given or both be null");
    // Pillow's precompute_coeffs (bilinear filter, box [0, in_size)), then normalize_coeffs_8bpc
    const double scale = (double)in_size / out_size;
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    const double support = 1.0 * filterscale;
    std::vector<double> w(ksize);
    for (int xx = 0; xx < out_size; ++xx) {
        const double center = (xx + 0.5) * scale;
        const double ss = 1.0 / filterscale;
        int xmin = (int)(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = (int)(center + support + 0.5);
        if (xmax > in_size) xmax = in_size;
        xmax -= xmin;
        double ww = 0.0;
        for (int x = 0; x < xmax; ++x) {
            double t = (x + xmin - center + 0.5) * ss;
            if (t < 0.0) t = -t;
            w[x] = t < 1.0 ? 1.0 - t : 0.0;
            ww += w[x];
        }
        int* kr = k + (long long)xx * ksize;
        for (int x = 0; x < ksize; ++x) {
            double v = x < xmax ? w[x] : 0.0;
            if (x < xmax && ww != 0.0) v /= ww;
            kr[x] = v < 0 ? (int)(-0.5 + v * (1 << kPrecisionBits)) : (int)(0.5 + v * (1 << kPrecisionBits));
        }
        bounds[2 * xx] = xmin;
        bounds[2 * xx + 1] = xmax;
    }
    return ksize;
}

extern "C" long long te_prepare_images_workspace_bytes(int batch, int max_in_h, int max_in_w, int out_h, int out_w) {
    if (batch <= 0 || batch > 65535 || max_in_h < 1 || max_in_h > TE_PREPARE_MAX_SIDE || max_in_w < 1 ||
        max_in_w > TE_PREPARE_MAX_SIDE || out_h < 1 || out_h > TE_PREPARE_MAX_OUT || out_w < 1 || out_w > TE_PREPARE_MAX_OUT)
        return TE_ERR_ARG;
    return up256((long long)sizeof(ImageDesc) * batch) + up256(4LL * batch * table_ints(max_in_h, max_in_w, out_h, out_w)) +
           up256(batch * mid_bound(max_in_h, max_in_w, out_h, out_w));
}

extern "C" int te_prepare_images(const unsigned char* packed, long long packed_bytes, int batch, const int* sizes,
                                 const long long* offsets, int out_h, int out_w, const float* mean, const float* std,
                                 float* out01, float* out_norm, void* workspace, long long workspace_bytes, void* stream) {
    REQ(packed && sizes && offsets, "te_prepare_images: null argument");
    REQ(out01 || out_norm, "te_prepare_images: no output requested");
    REQ(batch > 0 && batch <= 65535, "te_prepare_images: batch must lie in 1..65535");
    REQ(out_h >= 1 && out_h <= TE_PREPARE_MAX_OUT && out_w >= 1 && out_w <= TE_PREPARE_MAX_OUT,
        "te_prepare_images: output sides outside 1..TE_PREPARE_MAX_OUT");
    Norm nrm{};
    if (out_norm) {
        REQ(mean && std, "te_prepare_images: out_norm needs mean and std");
        for (int c = 0; c < 3; ++c) {
            REQ(std::isfinite(mean[c]) && std::isfinite(std[c]) && std[c] != 0.f,
                "te_prepare_images: mean and std must be finite and std non-zero");
            nrm.mean[c] = mean[c];
            nrm.std[c] = std[c];
        }
    }
    int max_h = 0, max_w = 0, max_rows = 0;
    for (int b = 0; b < batch; ++b) {
        const int h = sizes[2 * b], w = sizes[2 * b + 1];
        REQ(h >= 1 && h <= TE_PREPARE_MAX_SIDE && w >= 1 && w <= TE_PREPARE_MAX_SIDE,
            "te_prepare_images: every image side must lie in 1..TE_PREPARE_MAX_SIDE");
        REQ(offsets[b] >= 0 && offsets[b] <= packed_bytes - 3LL * h * w,
            "te_prepare_images: every image [offset, offset + 3 h w) must lie inside the packed buffer");
        max_h = h > max_h ? h : max_h;
        max_w = w > max_w ? w : max_w;
        const int rows = vertical_first(h, w, out_h) ? out_h : h;
        max_rows = rows > max_rows ? rows : max_rows;
    }
    REQ(workspace && (((uintptr_t)workspace) & 255u) == 0, "te_prepare_images: workspace null or not 256-byte aligned");
    if (te_prepare_images_workspace_bytes(batch, max_h, max_w, out_h, out_w) > workspace_bytes) {
        te_set_last_error("te_prepare_images: workspace too small");
        return TE_ERR_WORKSPACE;
    }
    // host image: [descriptors | tables], copied as one block; the intermediate follows the table bound
    const long long desc_bytes = up256((long long)sizeof(ImageDesc) * batch);
    long long ints = 0;
    for (int b = 0; b < batch; ++b) ints += table_ints(sizes[2 * b], sizes[2 * b + 1], out_h, out_w);
    std::vector<char> host(desc_bytes + 4 * ints);
    ImageDesc* desc = reinterpret_cast<ImageDesc*>(host.data());
    int* coef = reinterpret_cast<int*>(host.data() + desc_bytes);
    long long toff = 0, moff = 0;
    for (int b = 0; b < batch; ++b) {
        const int h = sizes[2 * b], w = sizes[2 * b + 1];
        ImageDesc& d = desc[b];
        d.in_off = offsets[b];
        d.mid_off = moff;
        d.h = h;
        d.w = w;
        d.vfirst = vertical_first(h, w, out_h);
        d.kx_off = toff;
        d.kx = te_resize_coeffs(w, out_w, coef + toff, coef + toff + (long long)out_w * kernel_size(w, out_w));
        toff += (long long)out_w * (d.kx + 2);
        d.ky_off = toff;
        d.ky = te_resize_coeffs(h, out_h, coef + toff, coef + toff + (long long)out_h * kernel_size(h, out_h));
        toff += (long long)out_h * (d.ky + 2);
        moff += d.vfirst ? 3LL * out_h * w : 3LL * h * out_w;
    }
    char* p = static_cast<char*>(workspace);
    const ImageDesc* d_desc = reinterpret_cast<const ImageDesc*>(p);
    const int* d_coef = reinterpret_cast<const int*>(p + desc_bytes);
    unsigned char* d_mid =
        reinterpret_cast<unsigned char*>(p + desc_bytes + up256(4LL * batch * table_ints(max_h, max_w, out_h, out_w)));
    cudaStream_t st = ST(stream);
    if (cudaMemcpyAsync(p, host.data(), host.size(), cudaMemcpyHostToDevice, st) != cudaSuccess) {
        te_set_last_error("te_prepare_images: copy of the image descriptors failed");
        return TE_ERR_CUDA;
    }
    resize_first_kernel<<<dim3(te_cdiv(max_rows, kRows), batch), kThreads, 0, st>>>(packed, d_desc, d_coef, d_mid, out_h,
                                                                                     out_w);
    TE_CUDA_CHECK_LAUNCH();
    resize_second_kernel<<<dim3(te_cdiv((long long)out_h * out_w, kThreads), batch), kThreads, 0, st>>>(
        d_mid, d_desc, d_coef, out_h, out_w, nrm, out01, out_norm);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
