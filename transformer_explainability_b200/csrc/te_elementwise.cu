// Row-wise and elementwise kernels of the attribution path: embedding assembly, LayerNorm
// fwd/bwd, softmax fwd/bwd, arg-max / one-hot seed, the elementwise LRP rules (Add, Clone,
// IndexSelect, safe_divide) and the head-mean aggregation.  All HBM-bound: one warp per row with
// float4 accesses, or flat grid-stride float4 streams; per-sample reductions accumulate in fp64.
//
// Reference semantics: modules/layers_ours.py (rules), baselines/ViT/ViT_LRP.py (wiring).
#include "te_kernels.h"

namespace {

constexpr int kThreads = 256;

// ------------------------------------------------------------------------------------------------
// embedding
// ------------------------------------------------------------------------------------------------
__global__ void im2col_kernel(const float* __restrict__ img, float* __restrict__ patches, int B, int C, int H,
                              int W, int P) {
    // one thread per float4 of a patch row: K index = c*P*P + iy*P + ix  (conv weight [D,C,P,P] flattened)
    const int gw = W / P, gh = H / P, pq = P / 4;
    const long long total = (long long)B * gh * gw * C * P * pq;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        long long r = t;
        const int q = (int)(r % pq); r /= pq;
        const int iy = (int)(r % P); r /= P;
        const int c = (int)(r % C); r /= C;
        const int px = (int)(r % gw); r /= gw;
        const int py = (int)(r % gh); r /= gh;
        const int b = (int)r;
        const float4 v = *reinterpret_cast<const float4*>(
            img + (((long long)b * C + c) * H + (py * P + iy)) * W + px * P + q * 4);
        const long long row = ((long long)b * gh + py) * gw + px;
        *reinterpret_cast<float4*>(patches + row * ((long long)C * P * P) + (c * P + iy) * P + q * 4) = v;
    }
}

// the same layout one float at a time, for patches that are not a multiple of 4 wide (14 for the /14 towers: a patch row
// starts at no 16-byte boundary)
__global__ void im2col_scalar_kernel(const float* __restrict__ img, float* __restrict__ patches, int B, int C, int H, int W,
                                     int P) {
    const int gw = W / P, gh = H / P;
    const long long total = (long long)B * gh * gw * C * P * P;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        long long r = t;
        const int ix = (int)(r % P); r /= P;
        const int iy = (int)(r % P); r /= P;
        const int c = (int)(r % C); r /= C;
        const int px = (int)(r % gw); r /= gw;
        const int py = (int)(r % gh); r /= gh;
        const int b = (int)r;
        patches[t] = img[(((long long)b * C + c) * H + (py * P + iy)) * W + px * P + ix];
    }
}

// CLIP's image-text similarity s = ls cos(x, t) of each sample and its gradient ls (t^ - cos x^) / |x| as the backward seed;
// one block per sample
__global__ void similarity_seed_kernel(const float* __restrict__ x, const float* __restrict__ t, float ls, float* __restrict__ sim,
                                       float* __restrict__ seed, int E) {
    const int b = blockIdx.x;
    const float* xb = x + (long long)b * E;
    const float* tb = t + (long long)b * E;
    float xx = 0.f, tt = 0.f, xt = 0.f;
    for (int i = threadIdx.x; i < E; i += blockDim.x) {
        const float a = xb[i], c = tb[i];
        xx = fmaf(a, a, xx); tt = fmaf(c, c, tt); xt = fmaf(a, c, xt);
    }
    __shared__ float red[3][kThreads / 32];
    xx = te_warp_sum(xx); tt = te_warp_sum(tt); xt = te_warp_sum(xt);
    if ((threadIdx.x & 31) == 0) { red[0][threadIdx.x >> 5] = xx; red[1][threadIdx.x >> 5] = tt; red[2][threadIdx.x >> 5] = xt; }
    __syncthreads();
    xx = tt = xt = 0.f;
    for (int w = 0; w < kThreads / 32; ++w) { xx += red[0][w]; tt += red[1][w]; xt += red[2][w]; }
    const float nx = sqrtf(xx), nt = sqrtf(tt), cosv = xt / (nx * nt);
    if (threadIdx.x == 0 && sim) sim[b] = ls * cosv;
    const float g = ls / nx;
    for (int i = threadIdx.x; i < E; i += blockDim.x) seed[(long long)b * E + i] = g * (tb[i] / nt - cosv * (xb[i] / nx));
}

__global__ void assemble_tokens_kernel(const float* __restrict__ patch_out, const float* __restrict__ cls,
                                       const float* __restrict__ dist, const float* __restrict__ pos,
                                       float* __restrict__ x, int B, int N, int D, int n_prefix) {
    // x = cat(cls[,dist], patches) + pos_embed      (ViT_LRP.py:309-311)
    const int d4 = D / 4;
    const long long total = (long long)B * N * d4;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        const int q = (int)(t % d4);
        const long long rt = t / d4;
        const int tok = (int)(rt % N);
        const int b = (int)(rt / N);
        float4 v;
        if (tok < n_prefix) v = *reinterpret_cast<const float4*>((tok == 0 ? cls : dist) + q * 4);
        else v = *reinterpret_cast<const float4*>(patch_out + ((long long)b * (N - n_prefix) + tok - n_prefix) * D + q * 4);
        if (pos != nullptr) {                                   // pos == null: the tokens before ``self.add`` (:311)
            const float4 pe = *reinterpret_cast<const float4*>(pos + (long long)tok * D + q * 4);
            v.x += pe.x; v.y += pe.y; v.z += pe.z; v.w += pe.w;
        }
        *reinterpret_cast<float4*>(x + rt * D + q * 4) = v;
    }
}

// ------------------------------------------------------------------------------------------------
// LayerNorm: one warp per row, three cached passes (mean, variance, write)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void row_stats(const float* __restrict__ xr, int D, int lane, float eps, float& mean,
                                          float& rstd) {
    float s = 0.f;
    for (int i = lane * 4; i < D; i += 128) {
        const float4 v = *reinterpret_cast<const float4*>(xr + i);
        s += (v.x + v.y) + (v.z + v.w);
    }
    mean = te_warp_sum(s) / (float)D;
    float q = 0.f;
    for (int i = lane * 4; i < D; i += 128) {
        const float4 v = *reinterpret_cast<const float4*>(xr + i);
        const float a = v.x - mean, b = v.y - mean, c = v.z - mean, d = v.w - mean;
        q += (a * a + b * b) + (c * c + d * d);
    }
    const float var = te_warp_sum(q) / (float)D;
    rstd = 1.0f / sqrtf(var + eps);
}

// SPLIT: also emit the block-scaled fp16 (hi, lo) split of y (one scale per 128 columns: exactly one warp iteration), the A
// operand of the fp16-split Linear that consumes y (te_tc_wgmma.cu) — saves that GEMM's pre-pass over y.
template <bool SPLIT>
__global__ void layernorm_kernel(const float* __restrict__ x, const float* __restrict__ w,
                                 const float* __restrict__ b, float* __restrict__ y, float* __restrict__ mean_o,
                                 float* __restrict__ rstd_o, long long rows, int D, float eps, __half* __restrict__ hi,
                                 __half* __restrict__ lo, float* __restrict__ scale) {
    const int lane = threadIdx.x & 31;
    const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const float* xr = x + row * D;
    float mean, rstd;
    row_stats(xr, D, lane, eps, mean, rstd);
    float* yr = y + row * D;
    const int nblk = (D + 127) / 128;
    for (int base = 0; base < D; base += 128) {
        const int i = base + lane * 4;
        float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
        if (i < D) {
            const float4 v = *reinterpret_cast<const float4*>(xr + i);
            const float4 ww = *reinterpret_cast<const float4*>(w + i);
            const float4 bb = *reinterpret_cast<const float4*>(b + i);
            o.x = (v.x - mean) * rstd * ww.x + bb.x;
            o.y = (v.y - mean) * rstd * ww.y + bb.y;
            o.z = (v.z - mean) * rstd * ww.z + bb.z;
            o.w = (v.w - mean) * rstd * ww.w + bb.w;
            *reinterpret_cast<float4*>(yr + i) = o;
        }
        if (SPLIT) {
            float s, si;
            te_f16_block_scale(te_warp_max(te_absmax4(o)), s, si);
            if (i < D) {
                uint2 h, l;
                te_f16_split4(o, s, h, l);
                *reinterpret_cast<uint2*>(hi + row * D + i) = h;
                *reinterpret_cast<uint2*>(lo + row * D + i) = l;
            }
            if (lane == 0) scale[row * nblk + base / 128] = si;
        }
    }
    if (lane == 0) {
        if (mean_o) mean_o[row] = mean;
        if (rstd_o) rstd_o[row] = rstd;
    }
}

// dx = dres + rstd * (g - mean(g) - xhat*mean(g*xhat)),  g = dy*w, xhat = (x-mean)*rstd
__device__ __forceinline__ void ln_bwd_row(const float* __restrict__ dyr, const float* __restrict__ xr,
                                           const float* __restrict__ w, const float* __restrict__ dresr,
                                           float* __restrict__ dxr, int D, int lane, float mean, float rstd) {
    float s1 = 0.f, s2 = 0.f;
    for (int i = lane * 4; i < D; i += 128) {
        const float4 dy = *reinterpret_cast<const float4*>(dyr + i);
        const float4 xv = *reinterpret_cast<const float4*>(xr + i);
        const float4 ww = *reinterpret_cast<const float4*>(w + i);
        const float g0 = dy.x * ww.x, g1 = dy.y * ww.y, g2 = dy.z * ww.z, g3 = dy.w * ww.w;
        s1 += (g0 + g1) + (g2 + g3);
        s2 += (g0 * ((xv.x - mean) * rstd) + g1 * ((xv.y - mean) * rstd)) +
              (g2 * ((xv.z - mean) * rstd) + g3 * ((xv.w - mean) * rstd));
    }
    const float c1 = te_warp_sum(s1) / (float)D;
    const float c2 = te_warp_sum(s2) / (float)D;
    for (int i = lane * 4; i < D; i += 128) {
        const float4 dy = *reinterpret_cast<const float4*>(dyr + i);
        const float4 xv = *reinterpret_cast<const float4*>(xr + i);
        const float4 ww = *reinterpret_cast<const float4*>(w + i);
        float4 o;
        o.x = rstd * (dy.x * ww.x - c1 - (xv.x - mean) * rstd * c2);
        o.y = rstd * (dy.y * ww.y - c1 - (xv.y - mean) * rstd * c2);
        o.z = rstd * (dy.z * ww.z - c1 - (xv.z - mean) * rstd * c2);
        o.w = rstd * (dy.w * ww.w - c1 - (xv.w - mean) * rstd * c2);
        if (dresr) {
            const float4 r = *reinterpret_cast<const float4*>(dresr + i);
            o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
        }
        *reinterpret_cast<float4*>(dxr + i) = o;
    }
}

__global__ void layernorm_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                                     const float* __restrict__ w, const float* __restrict__ mean,
                                     const float* __restrict__ rstd, const float* __restrict__ dres,
                                     float* __restrict__ dx, long long rows, int D) {
    const int lane = threadIdx.x & 31;
    const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    ln_bwd_row(dy + row * D, x + row * D, w, dres ? dres + row * D : nullptr, dx + row * D, D, lane, mean[row],
               rstd[row]);
}

__global__ void layernorm_bwd_strided_kernel(const float* __restrict__ dy, long long dy_stride,
                                             const float* __restrict__ x, long long x_stride,
                                             const float* __restrict__ w, float eps, float* __restrict__ dx,
                                             long long dx_stride, int rows, int D) {
    const int lane = threadIdx.x & 31;
    const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const float* xr = x + row * x_stride;
    float mean, rstd;
    row_stats(xr, D, lane, eps, mean, rstd);
    ln_bwd_row(dy + row * dy_stride, xr, w, nullptr, dx + row * dx_stride, D, lane, mean, rstd);
}

// ------------------------------------------------------------------------------------------------
// softmax over the last dim (row length N, row stride ld >= N, pad columns zeroed)
// ------------------------------------------------------------------------------------------------
__global__ void softmax_kernel(float* __restrict__ s, long long rows, int N, int ld,
                               const float* __restrict__ keymask, long long rows_per_batch) {
    const int lane = threadIdx.x & 31;
    const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    float* r = s + row * ld;
    if (keymask) {                                   // scores + extended attention mask  (BERT.py:342)
        const float* mk = keymask + (row / rows_per_batch) * N;
        for (int j = lane; j < N; j += 32) r[j] = r[j] + mk[j];
    }
    float m = -INFINITY;
    for (int j = lane; j < N; j += 32) m = fmaxf(m, r[j]);
    m = te_warp_max(m);
    float sum = 0.f;
    for (int j = lane; j < N; j += 32) {
        const float e = expf(r[j] - m);
        r[j] = e;
        sum += e;
    }
    sum = te_warp_sum(sum);
    for (int j = lane; j < ld; j += 32) r[j] = (j < N) ? r[j] / sum : 0.f;
}

__global__ void softmax_bwd_kernel(const float* __restrict__ p, const float* __restrict__ dp,
                                   float* __restrict__ ds, long long rows, int N, int ld, float scale) {
    const int lane = threadIdx.x & 31;
    const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const float* pr = p + row * ld;
    const float* gr = dp + row * ld;
    float dot = 0.f;
    for (int j = lane; j < N; j += 32) dot = fmaf(pr[j], gr[j], dot);
    dot = te_warp_sum(dot);
    float* o = ds + row * ld;
    for (int j = lane; j < ld; j += 32) o[j] = (j < N) ? pr[j] * (gr[j] - dot) * scale : 0.f;
}

// ------------------------------------------------------------------------------------------------
// arg-max (first maximum, like numpy.argmax — ViT_explanation_generator.py:29) and one-hot seed
// ------------------------------------------------------------------------------------------------
__global__ void argmax_kernel(const float* __restrict__ logits, int* __restrict__ index, int B, int C,
                              int only_negative) {
    const int lane = threadIdx.x & 31;
    const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (b >= B) return;
    const float* r = logits + (long long)b * C;
    float best = -INFINITY;
    int bi = 0x7fffffff;
    for (int j = lane; j < C; j += 32) {
        const float v = r[j];
        if (v > best || (v == best && j < bi)) { best = v; bi = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (lane == 0 && (!only_negative || index[b] < 0)) index[b] = (bi == 0x7fffffff) ? 0 : bi;
}

__global__ void onehot_kernel(const int* __restrict__ index, float* __restrict__ seed, int B, int C, float value) {
    const long long total = (long long)B * C;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(t / C), c = (int)(t % C);
        seed[t] = (index[b] == c) ? value : 0.f;
    }
}

// ------------------------------------------------------------------------------------------------
// LRP elementwise rules
// ------------------------------------------------------------------------------------------------
__global__ void sd_kernel(const float* a, const float* b, float* out,
                          long long n4) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n4;
         t += (long long)gridDim.x * blockDim.x) {
        const float4 va = reinterpret_cast<const float4*>(a)[t];
        const float4 vb = reinterpret_cast<const float4*>(b)[t];
        reinterpret_cast<float4*>(out)[t] =
            make_float4(te_sd(va.x, vb.x), te_sd(va.y, vb.y), te_sd(va.z, vb.z), te_sd(va.w, vb.w));
    }
}

// Clone.relprop (layers_ours.py:151-169): R = X * ((sd(R1,X) + sd(R2,X)) [+ sd(R3,X)])
__global__ void clone_relprop_kernel(const float* __restrict__ x, const float* __restrict__ r1,
                                     const float* __restrict__ r2, const float* __restrict__ r3,
                                     float* __restrict__ out, long long n4) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n4;
         t += (long long)gridDim.x * blockDim.x) {
        const float4 xv = reinterpret_cast<const float4*>(x)[t];
        const float4 a = reinterpret_cast<const float4*>(r1)[t];
        const float4 b = reinterpret_cast<const float4*>(r2)[t];
        float4 c = make_float4(te_sd(a.x, xv.x) + te_sd(b.x, xv.x), te_sd(a.y, xv.y) + te_sd(b.y, xv.y),
                               te_sd(a.z, xv.z) + te_sd(b.z, xv.z), te_sd(a.w, xv.w) + te_sd(b.w, xv.w));
        if (r3) {
            const float4 d = reinterpret_cast<const float4*>(r3)[t];
            c.x += te_sd(d.x, xv.x); c.y += te_sd(d.y, xv.y); c.z += te_sd(d.z, xv.z); c.w += te_sd(d.w, xv.w);
        }
        reinterpret_cast<float4*>(out)[t] = make_float4(xv.x * c.x, xv.y * c.y, xv.z * c.z, xv.w * c.w);
    }
}

// Add.relprop (layers_ours.py:97-120), reductions PER SAMPLE (the reference is B=1), fp64 sums.
// pass 1: partial[b][split] = (sum a, sum b, sum R),  a = x1*sd(R,x1+x2), b = x2*sd(R,x1+x2)
__global__ void add_reduce_kernel(const float* __restrict__ x1, const float* __restrict__ x2,
                                  const float* __restrict__ r, double* __restrict__ partial, long long per4,
                                  long long x2s4) {
    const int b = blockIdx.y, sp = blockIdx.x;
    const long long chunk = (per4 + TE_ADD_SPLIT - 1) / TE_ADD_SPLIT;
    const long long lo = sp * chunk, hi = min(per4, lo + chunk);
    const float4* p1 = reinterpret_cast<const float4*>(x1) + b * per4;
    const float4* p2 = reinterpret_cast<const float4*>(x2) + b * x2s4;
    const float4* pr = reinterpret_cast<const float4*>(r) + b * per4;
    double sa = 0.0, sb = 0.0, sr = 0.0;
    for (long long t = lo + threadIdx.x; t < hi; t += blockDim.x) {
        const float4 a = p1[t], c = p2[t], rr = pr[t];
        const float s0 = te_sd(rr.x, a.x + c.x), s1 = te_sd(rr.y, a.y + c.y);
        const float s2 = te_sd(rr.z, a.z + c.z), s3 = te_sd(rr.w, a.w + c.w);
        sa += ((double)(a.x * s0) + (double)(a.y * s1)) + ((double)(a.z * s2) + (double)(a.w * s3));
        sb += ((double)(c.x * s0) + (double)(c.y * s1)) + ((double)(c.z * s2) + (double)(c.w * s3));
        sr += ((double)rr.x + (double)rr.y) + ((double)rr.z + (double)rr.w);
    }
    __shared__ double red[3][kThreads / 32];
    sa = te_warp_sum(sa); sb = te_warp_sum(sb); sr = te_warp_sum(sr);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (lane == 0) { red[0][wid] = sa; red[1][wid] = sb; red[2][wid] = sr; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double ta = 0, tb = 0, tr = 0;
        for (int i = 0; i < kThreads / 32; ++i) { ta += red[0][i]; tb += red[1][i]; tr += red[2][i]; }
        double* o = partial + ((long long)b * TE_ADD_SPLIT + sp) * 3;
        o[0] = ta; o[1] = tb; o[2] = tr;
    }
}

// pass 2: a *= sd( sd(|A|,|A|+|B|)*rho , A ) ; b likewise
__global__ void add_scale_kernel(const float* __restrict__ x1, const float* __restrict__ x2,
                                 const float* __restrict__ r, float* __restrict__ r1, float* __restrict__ r2,
                                 const double* __restrict__ partial, long long per4, long long x2s4) {
    const int b = blockIdx.y;
    __shared__ float fa_s, fb_s;
    if (threadIdx.x == 0 && partial == nullptr) { fa_s = 1.f; fb_s = 1.f; }     // layers_lrp variant: no ratio normalisation
    if (threadIdx.x == 0 && partial != nullptr) {
        double A = 0, Bs = 0, rho = 0;
        const double* q = partial + (long long)b * TE_ADD_SPLIT * 3;
        for (int i = 0; i < TE_ADD_SPLIT; ++i) { A += q[i * 3]; Bs += q[i * 3 + 1]; rho += q[i * 3 + 2]; }
        const double den = fabs(A) + fabs(Bs);
        const double a_fact = te_sd(fabs(A), den) * rho;
        const double b_fact = te_sd(fabs(Bs), den) * rho;
        fa_s = (float)te_sd(a_fact, A);
        fb_s = (float)te_sd(b_fact, Bs);
    }
    __syncthreads();
    const float fa = fa_s, fb = fb_s;
    const float4* p1 = reinterpret_cast<const float4*>(x1) + b * per4;
    const float4* p2 = reinterpret_cast<const float4*>(x2) + b * x2s4;
    const float4* pr = reinterpret_cast<const float4*>(r) + b * per4;
    float4* o1 = reinterpret_cast<float4*>(r1) + b * per4;
    float4* o2 = r2 ? reinterpret_cast<float4*>(r2) + b * per4 : nullptr;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < per4;
         t += (long long)gridDim.x * blockDim.x) {
        const float4 a = p1[t], c = p2[t], rr = pr[t];
        const float s0 = te_sd(rr.x, a.x + c.x), s1 = te_sd(rr.y, a.y + c.y);
        const float s2 = te_sd(rr.z, a.z + c.z), s3 = te_sd(rr.w, a.w + c.w);
        o1[t] = make_float4(a.x * s0 * fa, a.y * s1 * fa, a.z * s2 * fa, a.w * s3 * fa);
        if (o2) o2[t] = make_float4(c.x * s0 * fb, c.y * s1 * fb, c.z * s2 * fb, c.w * s3 * fb);
    }
}

// IndexSelect.relprop (layers_ours.py:129-147) for the CLS (and distillation) token
__global__ void index_select_relprop_kernel(const float* __restrict__ x, const float* __restrict__ r0,
                                            const float* __restrict__ r1, float* __restrict__ out, int B, int N,
                                            int D) {
    const long long total = (long long)B * N * D;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        const int d = (int)(t % D);
        const long long rt = t / D;
        const int tok = (int)(rt % N);
        const int b = (int)(rt / N);
        float v = 0.f;
        if (tok == 0) v = x[t] * te_sd(r0[(long long)b * D + d], x[t]);
        else if (tok == 1 && r1 != nullptr) v = x[t] * te_sd(r1[(long long)b * D + d], x[t]);
        out[t] = v;
    }
}

// ------------------------------------------------------------------------------------------------
// aggregation: M = mean_h relu(G*cam) (+I) (/rowsum)      ViT_LRP.py:359-365 ; ExplanationGenerator.py:49-55,12-14
// ------------------------------------------------------------------------------------------------
// diag != null ("split" form for the tensor-core chain): the identity is NOT added into M; it still counts in the row
// sum, and its weight after normalisation (1 / rowsum) goes to diag[row].
__global__ void aggregate_kernel(const float* __restrict__ G, const float* __restrict__ cam,
                                 float* __restrict__ M, int B, int H, int N, int ld_in, int ld, int add_eye,
                                 int normalize, float* __restrict__ diag) {
    const int lane = threadIdx.x & 31;
    const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);   // b*N + i
    if (row >= (long long)B * N) return;
    const int b = (int)(row / N), i = (int)(row % N);
    float* out = M + row * ld;
    float rs = 0.f;
    for (int j = lane; j < ld; j += 32) {
        float v = 0.f;
        if (j < N) {
            float s = 0.f;
            for (int h = 0; h < H; ++h) {
                const long long o = (((long long)b * H + h) * N + i) * ld_in + j;
                s += fmaxf(G[o] * cam[o], 0.f);
            }
            v = s / (float)H;
            if (add_eye && j == i) v += 1.0f;
        }
        out[j] = v;
        rs += v;
    }
    if (normalize) {
        rs = te_warp_sum(rs);
        if (diag != nullptr) rs += 1.0f;
        __syncwarp();
        for (int j = lane; j < N; j += 32) out[j] = out[j] / rs;
        if (diag != nullptr && lane == 0) diag[row] = 1.0f / rs;
    }
}

// same, 128-bit streaming loads (ld_in % 4 == 0, ld % 4 == 0): every lane keeps H independent float4 pairs in flight
__global__ void aggregate_vec_kernel(const float* __restrict__ G, const float* __restrict__ cam, float* __restrict__ M,
                                     int B, int H, int N, int ld_in, int ld, int add_eye, int normalize,
                                     float* __restrict__ diag) {
    const int lane = threadIdx.x & 31;
    const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);   // b*N + i
    if (row >= (long long)B * N) return;
    const int b = (int)(row / N), i = (int)(row % N);
    float* out = M + row * ld;
    float rs = 0.f;
    for (int j4 = lane; j4 * 4 < ld; j4 += 32) {
        const int j = j4 * 4;
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        if (j < N && j < ld_in) {
#pragma unroll 4
            for (int h = 0; h < H; ++h) {
                const long long o = (((long long)b * H + h) * N + i) * ld_in + j;
                const float4 g = __ldcs(reinterpret_cast<const float4*>(G + o));
                const float4 c = __ldcs(reinterpret_cast<const float4*>(cam + o));
                s.x += fmaxf(g.x * c.x, 0.f); s.y += fmaxf(g.y * c.y, 0.f);
                s.z += fmaxf(g.z * c.z, 0.f); s.w += fmaxf(g.w * c.w, 0.f);
            }
        }
        float v[4] = {s.x / (float)H, s.y / (float)H, s.z / (float)H, s.w / (float)H};
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            if (j + u >= N) v[u] = 0.f;                         // the row padding of G / cam is never trusted
            else if (add_eye && j + u == i) v[u] += 1.0f;
            rs += v[u];
        }
        *reinterpret_cast<float4*>(out + j) = make_float4(v[0], v[1], v[2], v[3]);
    }
    if (normalize) {
        rs = te_warp_sum(rs);
        if (diag != nullptr) rs += 1.0f;
        __syncwarp();
        for (int j = lane; j < N; j += 32) out[j] = out[j] / rs;
        if (diag != nullptr && lane == 0) diag[row] = 1.0f / rs;
    }
}

// All layers of the dense rollout in ONE launch (blockIdx.y = layer - first_layer): the per-layer launches of the composed
// path left the aggregation latency-bound (one short row per warp, a few thousand warps per launch: 0.39-0.47 of the HBM
// peak for the whole dense call); with every layer in flight at once and all H head rows of a lane's float4 column issued
// back to back the stream is deep enough to approach the copy bandwidth.  Layer `first_layer` keeps its identity inside M
// (it is the chain's start, ViT_LRP.py:46); the others are written WITHOUT it (residual form of te_tc_bmm_nk_resid) and, when
// normalising, export the identity's weight 1 / rowsum to diag.
__global__ void aggregate_layers_vec_kernel(const float* __restrict__ G0, const float* __restrict__ cam0, long long in_layer_stride,
                                            float* __restrict__ M0, long long m_layer_stride, int B, int H, int N, int ld_in,
                                            int ld, int first_layer, int normalize, float* __restrict__ diag0) {
    const int lane = threadIdx.x & 31;
    const int layer = first_layer + blockIdx.y;
    const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);   // b*N + i
    if (row >= (long long)B * N) return;
    const int b = (int)(row / N), i = (int)(row % N);
    const float* __restrict__ G = G0 + (long long)layer * in_layer_stride;
    const float* __restrict__ cam = cam0 + (long long)layer * in_layer_stride;
    float* out = M0 + (long long)layer * m_layer_stride + row * ld;
    const bool eye = blockIdx.y == 0;
    float* diag = (!eye && diag0) ? diag0 + (long long)layer * B * N : nullptr;
    float rs = 0.f;
    const float inv_h = 1.0f / (float)H;
    for (int j4 = lane; j4 * 4 < ld; j4 += 32) {
        const int j = j4 * 4;
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
        if (j < N && j < ld_in) {
            const long long o0 = (((long long)b * H) * N + i) * ld_in + j;
            const long long hs = (long long)N * ld_in;
#pragma unroll 6
            for (int h = 0; h < H; ++h) {
                const float4 g = __ldcs(reinterpret_cast<const float4*>(G + o0 + h * hs));
                const float4 c = __ldcs(reinterpret_cast<const float4*>(cam + o0 + h * hs));
                s.x += fmaxf(g.x * c.x, 0.f); s.y += fmaxf(g.y * c.y, 0.f);
                s.z += fmaxf(g.z * c.z, 0.f); s.w += fmaxf(g.w * c.w, 0.f);
            }
        }
        float v[4] = {s.x / (float)H, s.y / (float)H, s.z / (float)H, s.w / (float)H};
        (void)inv_h;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            if (j + u >= N) v[u] = 0.f;                         // the row padding of G / cam is never trusted
            else if (eye && j + u == i) v[u] += 1.0f;
            rs += v[u];
        }
        *reinterpret_cast<float4*>(out + j) = make_float4(v[0], v[1], v[2], v[3]);
    }
    if (normalize) {
        rs = te_warp_sum(rs);
        if (diag != nullptr) rs += 1.0f;
        __syncwarp();
        for (int j = lane; j < N; j += 32) out[j] = out[j] / rs;
        if (diag != nullptr && lane == 0) diag[row] = 1.0f / rs;
    }
}

// generate_visualization (example.ipynb:57-60): [g,g] relevance -> bilinear x scale (align_corners=False, the arithmetic of
// torch.nn.functional.interpolate(mode='bilinear', scale_factor=scale)) -> per-sample min-max.  One block per sample.
// fminf / fmaxf skip NaN, so a NaN flag rides along the reduction: like torch's t.min() / t.max(), a NaN anywhere in the
// up-sampled map makes the minimum, hence every normalised pixel, NaN.
__global__ void relevance_heatmap_kernel(const float* __restrict__ maps, float* __restrict__ out, int g, int scale) {
    const int G = g * scale, total = G * G;
    const float* m = maps + (long long)blockIdx.x * g * g;
    float* o = out + (long long)blockIdx.x * total;
    const float rs = 1.0f / (float)scale;
    float mn = INFINITY, mx = -INFINITY;
    int nan = 0;
    for (int p = threadIdx.x; p < total; p += blockDim.x) {
        const int y = p / G, x = p % G;
        const float sy = fmaxf(rs * ((float)y + 0.5f) - 0.5f, 0.f), sx = fmaxf(rs * ((float)x + 0.5f) - 0.5f, 0.f);
        const int y0 = (int)sy, x0 = (int)sx;
        const int y1 = y0 + (y0 < g - 1 ? 1 : 0), x1 = x0 + (x0 < g - 1 ? 1 : 0);
        const float ly1 = sy - (float)y0, ly0 = 1.f - ly1, lx1 = sx - (float)x0, lx0 = 1.f - lx1;
        const float v = ly0 * (lx0 * m[y0 * g + x0] + lx1 * m[y0 * g + x1]) + ly1 * (lx0 * m[y1 * g + x0] + lx1 * m[y1 * g + x1]);
        o[p] = v;
        mn = fminf(mn, v); mx = fmaxf(mx, v);
        nan |= v != v;
    }
    __shared__ float smn[kThreads / 32], smx[kThreads / 32], bmn, bmx;
    __shared__ int snan[kThreads / 32];
    for (int s = 16; s > 0; s >>= 1) {
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, s));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, s));
        nan |= __shfl_xor_sync(0xffffffffu, nan, s);
    }
    if ((threadIdx.x & 31) == 0) { smn[threadIdx.x >> 5] = mn; smx[threadIdx.x >> 5] = mx; snan[threadIdx.x >> 5] = nan; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < kThreads / 32; ++i) { mn = fminf(mn, smn[i]); mx = fmaxf(mx, smx[i]); nan |= snan[i]; }
        bmn = nan ? NAN : mn; bmx = mx;
    }
    __syncthreads();
    const float lo = bmn, range = bmx - bmn;
    for (int p = threadIdx.x; p < total; p += blockDim.x) o[p] = (o[p] - lo) / range;      // each thread re-reads its own writes
}

// head reductions for the secondary methods: one warp per output row
__global__ void head_reduce_kernel(const float* __restrict__ A, const float* __restrict__ G,
                                   const float* __restrict__ hw, float* __restrict__ out, int B, int H, int N, int ld,
                                   int mode) {
    const int lane = threadIdx.x & 31;
    const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);   // b*N + i
    if (row >= (long long)B * N) return;
    const int b = (int)(row / N), i = (int)(row % N);
    for (int j = lane; j < N; j += 32) {
        float s = 0.f;
        for (int h = 0; h < H; ++h) {
            const long long o = (((long long)b * H + h) * N + i) * ld + j;
            float v = A[o];
            if (G != nullptr) v *= G[o];
            if (hw != nullptr) v *= hw[b * H + h];
            s += (mode == 1) ? fmaxf(v, 0.f) : v;
        }
        s /= (float)H;
        out[row * N + j] = (mode == 2) ? fmaxf(s, 0.f) : s;
    }
}
// out[b,h] = mean of G[b,h,r0:r1,c0:c1]; one block per (b,h)
__global__ void head_region_mean_kernel(const float* __restrict__ G, float* __restrict__ out, int N, int ld, int r0, int r1,
                                        int c0, int c1) {
    const float* g = G + (long long)blockIdx.x * N * ld;
    const int w = c1 - c0, total = (r1 - r0) * w;
    double s = 0.0;
    for (int t = threadIdx.x; t < total; t += blockDim.x) s += (double)g[(long long)(r0 + t / w) * ld + c0 + t % w];
    __shared__ double red[kThreads / 32];
    s = te_warp_sum(s);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0;
        for (int i = 0; i < kThreads / 32; ++i) t += red[i];
        out[blockIdx.x] = (float)(t / (double)total);
    }
}

// all_layer_matrices[i] + eye (/ rowsum)     (ViT_LRP.py:41-44 ; ExplanationGenerator.py:11-14)
__global__ void prep_mats_kernel(const float* __restrict__ in, float* __restrict__ out, long long rows, int N,
                                 int ld_in, int ld_out, int normalize) {
    const int lane = threadIdx.x & 31;
    const long long row = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int i = (int)(row % N);
    const float* r = in + row * ld_in;
    float* o = out + row * ld_out;
    float rs = 0.f;
    for (int j = lane; j < ld_out; j += 32) {
        float v = 0.f;
        if (j < N) v = r[j] + ((j == i) ? 1.0f : 0.0f);
        o[j] = v;
        rs += v;
    }
    if (normalize) {
        rs = te_warp_sum(rs);
        __syncwarp();
        for (int j = lane; j < N; j += 32) o[j] = o[j] / rs;
    }
}

__global__ void extract_row_kernel(const float* __restrict__ joint, float* __restrict__ out, int B, int N, int ld,
                                   int first, int bert_fix) {
    const int lane = threadIdx.x & 31;
    const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (b >= B) return;
    const float* r = joint + (long long)b * N * ld;
    float mn = INFINITY;
    if (bert_fix) {
        for (int j = lane; j < N; j += 32) mn = fminf(mn, r[j]);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    }
    float* o = out + (long long)b * (N - first);
    for (int j = first + lane; j < N; j += 32) o[j - first] = (bert_fix && j == 0) ? mn : r[j];
}

__global__ void average2_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out,
                                long long n) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n;
         t += (long long)gridDim.x * blockDim.x) out[t] = (a[t] + b[t]) / 2.0f;
}

// ------------------------------------------------------------------------------------------------
// BERT extras: embeddings, additive mask, tanh, elementwise add, Add rule with a key-broadcast operand
// ------------------------------------------------------------------------------------------------
// (token_type + position) + word   (BertEmbeddings.forward, BERT.py:80-81; position_ids = arange).  tt == NULL: every
// token is segment 0 (row 0 of the token-type table).
__global__ void bert_embed_kernel(const long long* __restrict__ ids, const long long* __restrict__ tt,
                                  const float* __restrict__ word, const float* __restrict__ pos,
                                  const float* __restrict__ type, float* __restrict__ out, int B, int S, int D, int vocab,
                                  int type_vocab) {
    const int d4 = D / 4;
    const long long total = (long long)B * S * d4;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total;
         t += (long long)gridDim.x * blockDim.x) {
        const int q = (int)(t % d4);
        const long long rt = t / d4;
        const int s = (int)(rt % S);
        const long long id = ids[rt];
        const long long ty_id = tt ? tt[rt] : 0;
        // never index a table out of bounds: the row becomes NaN (loud, memory-safe)
        if (id < 0 || id >= vocab || ty_id < 0 || ty_id >= type_vocab) {
            const float qn = __int_as_float(0x7fc00000);
            *reinterpret_cast<float4*>(out + rt * D + q * 4) = make_float4(qn, qn, qn, qn);
            continue;
        }
        const float4 w = *reinterpret_cast<const float4*>(word + id * D + q * 4);
        const float4 p = *reinterpret_cast<const float4*>(pos + (long long)s * D + q * 4);
        const float4 ty = *reinterpret_cast<const float4*>(type + ty_id * D + q * 4);
        *reinterpret_cast<float4*>(out + rt * D + q * 4) =
            make_float4((ty.x + p.x) + w.x, (ty.y + p.y) + w.y, (ty.z + p.z) + w.z, (ty.w + p.w) + w.w);
    }
}
// RoBERTa / DistilBERT embeddings (transformers RobertaEmbeddings / distilbert Embeddings .forward).  Block (tile, b)
// writes tokens [32 tile, 32 tile + 32) of row b.  pad >= 0 (RoBERTa, create_position_ids_from_input_ids): a token's
// position is pad + (number of ids != pad up to and including it), or pad for a pad token; the count before the tile
// is one block-wide count of the row's earlier ids, the count inside it one warp ballot.  pad < 0: position = token
// index.  type != NULL: (word + type) + position (RoBERTa); type == NULL: word + position (DistilBERT).
constexpr int kEmbedTile = 32;
__global__ void __launch_bounds__(256) hf_embed_kernel(const long long* __restrict__ ids, const long long* __restrict__ tt,
                                                       const float* __restrict__ word, const float* __restrict__ pos,
                                                       const float* __restrict__ type, float* __restrict__ out, int S, int D,
                                                       int vocab, int max_position, int type_vocab, int pad) {
    __shared__ int spos[kEmbedTile];
    const int b = blockIdx.y, s0 = blockIdx.x * kEmbedTile;
    const long long* row = ids + (long long)b * S;
    int before = 0;
    if (pad >= 0)
        for (int base = 0; base < s0; base += blockDim.x) {        // block-uniform trip count
            const int s = base + (int)threadIdx.x;
            before += __syncthreads_count(s < s0 && row[s] != pad);
        }
    if (threadIdx.x < kEmbedTile) {
        const int lane = threadIdx.x, s = s0 + lane;
        if (pad >= 0) {
            const bool counted = s < S && row[s] != pad;
            const unsigned upto = __ballot_sync(0xffffffffu, counted) & (0xffffffffu >> (31 - lane));
            spos[lane] = counted ? pad + before + __popc(upto) : pad;
        } else {
            spos[lane] = s;
        }
    }
    __syncthreads();
    const int d4 = D / 4, n = min(kEmbedTile, S - s0);
    for (int t = threadIdx.x; t < n * d4; t += blockDim.x) {
        const int j = t / d4, q = t - j * d4;
        const long long rt = (long long)b * S + s0 + j;
        const long long id = ids[rt];
        const long long ty_id = tt ? tt[rt] : 0;
        const int p = spos[j];
        float4* o = reinterpret_cast<float4*>(out + rt * D) + q;
        // never index a table out of bounds: the row becomes NaN (loud, memory-safe)
        if (id < 0 || id >= vocab || p < 0 || p >= max_position || (type && (ty_id < 0 || ty_id >= type_vocab))) {
            const float qn = __int_as_float(0x7fc00000);
            *o = make_float4(qn, qn, qn, qn);
            continue;
        }
        const float4 w = reinterpret_cast<const float4*>(word + id * D)[q];
        const float4 ps = reinterpret_cast<const float4*>(pos + (long long)p * D)[q];
        if (type) {
            const float4 ty = reinterpret_cast<const float4*>(type + ty_id * D)[q];
            *o = make_float4((w.x + ty.x) + ps.x, (w.y + ty.y) + ps.y, (w.z + ty.z) + ps.z, (w.w + ty.w) + ps.w);
        } else {
            *o = make_float4(w.x + ps.x, w.y + ps.y, w.z + ps.z, w.w + ps.w);
        }
    }
}
// transformers 3.5.1 get_extended_attention_mask: (1 - mask) * -10000   (call site BERT.py:598)
__global__ void bert_mask_kernel(const long long* __restrict__ mask, float* __restrict__ out, long long n) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x)
        out[t] = (1.0f - (float)mask[t]) * -10000.0f;
}
__global__ void tanh_kernel(const float* __restrict__ x, float* __restrict__ y, long long n) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x)
        y[t] = tanhf(x[t]);
}
__global__ void tanh_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ dx,
                                long long n) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x)
        dx[t] = dy[t] * (1.0f - y[t] * y[t]);
}
__global__ void relu_kernel(const float* __restrict__ x, float* __restrict__ y, long long n) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x) {
        const float v = x[t];
        y[t] = (v > 0.f || v != v) ? v : 0.f;             // torch.relu: NaN stays NaN
    }
}
__global__ void relu_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ y, float* __restrict__ dx,
                                long long n) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n; t += (long long)gridDim.x * blockDim.x)
        dx[t] = y[t] > 0.f ? dy[t] : 0.f;
}
__global__ void add2_kernel(const float* a, const float* b, float* out, long long n4) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n4;
         t += (long long)gridDim.x * blockDim.x) {
        const float4 u = reinterpret_cast<const float4*>(a)[t], v = reinterpret_cast<const float4*>(b)[t];
        reinterpret_cast<float4*>(out)[t] = make_float4(u.x + v.x, u.y + v.y, u.z + v.z, u.w + v.w);
    }
}

// Add.relprop for add([scores, extended_mask]) (BERT.py:386-388): x1 [B,H,N,ld], x2[b,j] broadcast over (h,i).
// pass 1: per-sample sums (a = x1*S, b = x2*S, rho = R) ; the mask's own relevance is discarded by the caller,
// but its sum enters the renormalisation factors.
__global__ void add_keymask_reduce_kernel(const float* __restrict__ x1, const float* __restrict__ mk,
                                          const float* __restrict__ r, double* __restrict__ partial, int HN, int N,
                                          int ld) {
    const int b = blockIdx.y, sp = blockIdx.x;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const float* m = mk + (long long)b * N;
    double sa = 0.0, sb = 0.0, sr = 0.0;
    for (int row = sp * nw + wid; row < HN; row += TE_ADD_SPLIT * nw) {
        const float* xr = x1 + ((long long)b * HN + row) * ld;
        const float* rr = r + ((long long)b * HN + row) * ld;
        for (int j = lane; j < N; j += 32) {
            const float a = xr[j], c = m[j], rv = rr[j];
            const float s = te_sd(rv, a + c);
            sa += (double)(a * s); sb += (double)(c * s); sr += (double)rv;
        }
    }
    __shared__ double red[3][kThreads / 32];
    sa = te_warp_sum(sa); sb = te_warp_sum(sb); sr = te_warp_sum(sr);
    if (lane == 0) { red[0][wid] = sa; red[1][wid] = sb; red[2][wid] = sr; }
    __syncthreads();
    if (threadIdx.x == 0) {
        double ta = 0, tb = 0, tr = 0;
        for (int i = 0; i < nw; ++i) { ta += red[0][i]; tb += red[1][i]; tr += red[2][i]; }
        double* o = partial + ((long long)b * TE_ADD_SPLIT + sp) * 3;
        o[0] = ta; o[1] = tb; o[2] = tr;
    }
}
__global__ void add_keymask_scale_kernel(const float* __restrict__ x1, const float* __restrict__ mk,
                                         const float* __restrict__ r, float* __restrict__ r1,
                                         const double* __restrict__ partial, int HN, int N, int ld) {
    const int b = blockIdx.y;
    __shared__ float fa_s;
    if (threadIdx.x == 0 && partial == nullptr) fa_s = 1.f;      // layers_lrp variant: no ratio normalisation
    else if (threadIdx.x == 0) {
        double A = 0, Bs = 0, rho = 0;
        const double* q = partial + (long long)b * TE_ADD_SPLIT * 3;
        for (int i = 0; i < TE_ADD_SPLIT; ++i) { A += q[i * 3]; Bs += q[i * 3 + 1]; rho += q[i * 3 + 2]; }
        const double den = fabs(A) + fabs(Bs);
        fa_s = (float)te_sd(te_sd(fabs(A), den) * rho, A);
    }
    __syncthreads();
    const float fa = fa_s;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const float* m = mk + (long long)b * N;
    for (int row = blockIdx.x * nw + wid; row < HN; row += gridDim.x * nw) {
        const float* xr = x1 + ((long long)b * HN + row) * ld;
        const float* rr = r + ((long long)b * HN + row) * ld;
        float* o = r1 + ((long long)b * HN + row) * ld;
        for (int j = lane; j < ld; j += 32) {
            float v = 0.f;
            if (j < N) { const float a = xr[j]; v = a * te_sd(rr[j], a + m[j]) * fa; }
            o[j] = v;
        }
    }
}

__global__ void fill_kernel(float* __restrict__ p, float v, long long n) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < n;
         t += (long long)gridDim.x * blockDim.x) p[t] = v;
}

inline int flat_grid(long long work) {
    long long g = (work + kThreads - 1) / kThreads;
    const long long cap = 132LL * 16;
    return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}
inline int warp_rows_grid(long long rows) { return (int)((rows + (kThreads / 32) - 1) / (kThreads / 32)); }

}  // namespace

#define TE_REQ(c, msg) do { if (!(c)) { te_set_last_error(msg); return TE_ERR_ARG; } } while (0)

int te_launch_im2col(const float* img, float* patches, int B, int C, int H, int W, int P, cudaStream_t st) {
    TE_REQ(P > 0 && W % P == 0 && H % P == 0, "im2col: patch must divide the image");
    if (P % 4 == 0 && W % 4 == 0) {
        const long long total = (long long)B * (H / P) * (W / P) * C * P * (P / 4);
        im2col_kernel<<<flat_grid(total), kThreads, 0, st>>>(img, patches, B, C, H, W, P);
    } else {
        im2col_scalar_kernel<<<flat_grid((long long)B * C * H * W), kThreads, 0, st>>>(img, patches, B, C, H, W, P);
    }
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_similarity_seed(const float* x, const float* t, float logit_scale, float* sim, float* seed, int B, int E,
                              cudaStream_t st) {
    TE_REQ(B > 0 && B <= 65535 && E > 0, "similarity_seed: bad shape");
    similarity_seed_kernel<<<B, kThreads, 0, st>>>(x, t, logit_scale, sim, seed, E);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_assemble_tokens(const float* patch_out, const float* cls, const float* dist, const float* pos,
                              float* x, int B, int N, int D, int n_prefix, cudaStream_t st) {
    TE_REQ(D % 4 == 0, "assemble: D % 4 != 0");
    assemble_tokens_kernel<<<flat_grid((long long)B * N * (D / 4)), kThreads, 0, st>>>(patch_out, cls, dist, pos, x,
                                                                                     B, N, D, n_prefix);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_layernorm(const float* x, const float* w, const float* b, float* y, float* mean, float* rstd,
                        long long rows, int D, float eps, cudaStream_t st) {
    TE_REQ(D % 4 == 0, "layernorm: D % 4 != 0");
    if (rows <= 0) return TE_OK;
    layernorm_kernel<false><<<warp_rows_grid(rows), kThreads, 0, st>>>(x, w, b, y, mean, rstd, rows, D, eps, nullptr, nullptr,
                                                                       nullptr);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
// LayerNorm that also emits the block-scaled fp16 split of y: split = [hi | lo] fp16 [rows, D] (rows*D floats), scale [rows, ceil(D/128)]
int te_launch_layernorm_split(const float* x, const float* w, const float* b, float* y, float* mean, float* rstd,
                              long long rows, int D, float eps, float* split, float* scale, cudaStream_t st) {
    TE_REQ(D % 4 == 0, "layernorm: D % 4 != 0");
    TE_REQ(split && scale, "layernorm_split: null split buffers");
    if (rows <= 0) return TE_OK;
    __half* hi = reinterpret_cast<__half*>(split);
    layernorm_kernel<true><<<warp_rows_grid(rows), kThreads, 0, st>>>(x, w, b, y, mean, rstd, rows, D, eps, hi, hi + rows * D, scale);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_layernorm_bwd(const float* dy, const float* x, const float* w, const float* mean, const float* rstd,
                            const float* dres, float* dx, long long rows, int D, cudaStream_t st) {
    TE_REQ(D % 4 == 0, "layernorm_bwd: D % 4 != 0");
    if (rows <= 0) return TE_OK;
    layernorm_bwd_kernel<<<warp_rows_grid(rows), kThreads, 0, st>>>(dy, x, w, mean, rstd, dres, dx, rows, D);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_layernorm_bwd_strided(const float* dy, long long dy_stride, const float* x, long long x_stride,
                                    const float* w, float eps, float* dx, long long dx_stride, int rows, int D,
                                    cudaStream_t st) {
    TE_REQ(D % 4 == 0 && dy_stride % 4 == 0 && x_stride % 4 == 0 && dx_stride % 4 == 0, "layernorm_bwd_strided: align");
    if (rows <= 0) return TE_OK;
    layernorm_bwd_strided_kernel<<<warp_rows_grid(rows), kThreads, 0, st>>>(dy, dy_stride, x, x_stride, w, eps, dx,
                                                                          dx_stride, rows, D);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_softmax(float* s, long long rows, int N, int ld, cudaStream_t st) {
    return te_launch_softmax_masked(s, rows, N, ld, nullptr, 1, st);
}
int te_launch_softmax_masked(float* s, long long rows, int N, int ld, const float* keymask, long long rows_per_batch,
                             cudaStream_t st) {
    if (rows <= 0) return TE_OK;
    softmax_kernel<<<warp_rows_grid(rows), kThreads, 0, st>>>(s, rows, N, ld, keymask, rows_per_batch);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_softmax_bwd(const float* p, const float* dp, float* ds, long long rows, int N, int ld, float scale,
                          cudaStream_t st) {
    if (rows <= 0) return TE_OK;
    softmax_bwd_kernel<<<warp_rows_grid(rows), kThreads, 0, st>>>(p, dp, ds, rows, N, ld, scale);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_argmax(const float* logits, int* index, int B, int C, int only_negative, cudaStream_t st) {
    argmax_kernel<<<warp_rows_grid(B), kThreads, 0, st>>>(logits, index, B, C, only_negative);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_onehot(const int* index, float* seed, int B, int C, float value, cudaStream_t st) {
    onehot_kernel<<<flat_grid((long long)B * C), kThreads, 0, st>>>(index, seed, B, C, value);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_sd(const float* a, const float* b, float* out, long long n, cudaStream_t st) {
    TE_REQ(n % 4 == 0, "sd: n % 4 != 0");
    sd_kernel<<<flat_grid(n / 4), kThreads, 0, st>>>(a, b, out, n / 4);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_clone_relprop(const float* x, const float* r1, const float* r2, const float* r3, float* out,
                            long long n, cudaStream_t st) {
    TE_REQ(n % 4 == 0, "clone_relprop: n % 4 != 0");
    clone_relprop_kernel<<<flat_grid(n / 4), kThreads, 0, st>>>(x, r1, r2, r3, out, n / 4);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_add_relprop_strided(const float* x1, const float* x2, long long x2_sample_stride, const float* r, float* r1,
                                  float* r2, double* partial, int B, long long per_sample, cudaStream_t st) {
    TE_REQ(per_sample % 4 == 0 && x2_sample_stride % 4 == 0, "add_relprop: per-sample size % 4 != 0");
    TE_REQ(B <= 65535, "add_relprop: batch too large for one launch");
    const long long per4 = per_sample / 4, x2s4 = x2_sample_stride / 4;
    if (partial) {                            // null: Add of modules/layers_lrp.py (RelPropSimple) — a = x1*S, b = x2*S only
        add_reduce_kernel<<<dim3(TE_ADD_SPLIT, B), kThreads, 0, st>>>(x1, x2, r, partial, per4, x2s4);
        TE_CUDA_CHECK_LAUNCH();
    }
    int gx = (int)((per4 + kThreads - 1) / kThreads);
    gx = gx > 64 ? 64 : (gx < 1 ? 1 : gx);
    add_scale_kernel<<<dim3(gx, B), kThreads, 0, st>>>(x1, x2, r, r1, r2, partial, per4, x2s4);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_add_relprop(const float* x1, const float* x2, const float* r, float* r1, float* r2, double* partial,
                          int B, long long per_sample, cudaStream_t st) {
    return te_launch_add_relprop_strided(x1, x2, per_sample, r, r1, r2, partial, B, per_sample, st);
}
int te_launch_index_select_relprop(const float* x, const float* r_tok0, const float* r_tok1, float* out, int B,
                                   int N, int D, cudaStream_t st) {
    index_select_relprop_kernel<<<flat_grid((long long)B * N * D), kThreads, 0, st>>>(x, r_tok0, r_tok1, out, B, N, D);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_aggregate(const float* G, const float* cam, float* M, int B, int H, int N, int ld_in, int ld_out,
                        int add_eye, int normalize, cudaStream_t st, float* diag) {
    const bool vec = ld_in % 4 == 0 && ld_out % 4 == 0 && ld_in >= ((N + 3) & ~3) &&
                     ((reinterpret_cast<uintptr_t>(G) | reinterpret_cast<uintptr_t>(cam) | reinterpret_cast<uintptr_t>(M)) & 15u) == 0;
    if (vec)
        aggregate_vec_kernel<<<warp_rows_grid((long long)B * N), kThreads, 0, st>>>(G, cam, M, B, H, N, ld_in, ld_out,
                                                                                  add_eye, normalize, diag);
    else
        aggregate_kernel<<<warp_rows_grid((long long)B * N), kThreads, 0, st>>>(G, cam, M, B, H, N, ld_in, ld_out, add_eye,
                                                                              normalize, diag);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_aggregate_layers(const float* G0, const float* cam0, long long in_layer_stride, float* M0, long long m_layer_stride,
                               int B, int H, int N, int ld_in, int ld_out, int first_layer, int num_layers, int normalize,
                               cudaStream_t st, float* diag0) {
    const bool vec = ld_in % 4 == 0 && ld_out % 4 == 0 && ld_in >= ((N + 3) & ~3) && in_layer_stride % 4 == 0 &&
                     m_layer_stride % 4 == 0 &&
                     ((reinterpret_cast<uintptr_t>(G0) | reinterpret_cast<uintptr_t>(cam0) | reinterpret_cast<uintptr_t>(M0)) & 15u) == 0;
    TE_REQ(vec && num_layers >= 1 && num_layers <= 65535, "aggregate_layers: unsupported layout");
    dim3 grid(warp_rows_grid((long long)B * N), num_layers);
    aggregate_layers_vec_kernel<<<grid, kThreads, 0, st>>>(G0, cam0, in_layer_stride, M0, m_layer_stride, B, H, N, ld_in, ld_out,
                                                          first_layer, normalize, diag0);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_relevance_heatmap(const float* maps, float* out, int B, int g, int scale, cudaStream_t st) {
    TE_REQ(B > 0 && g > 0 && scale > 0, "relevance_heatmap: bad shape");
    relevance_heatmap_kernel<<<B, kThreads, 0, st>>>(maps, out, g, scale);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_head_reduce(const float* a, const float* g, const float* hw, float* out, int B, int H, int N, int ld,
                          int mode, cudaStream_t st) {
    head_reduce_kernel<<<warp_rows_grid((long long)B * N), kThreads, 0, st>>>(a, g, hw, out, B, H, N, ld, mode);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_head_region_mean(const float* g, float* out, int BH, int N, int ld, int r0, int r1, int c0, int c1,
                               cudaStream_t st) {
    TE_REQ(BH > 0 && r0 >= 0 && r1 > r0 && r1 <= N && c0 >= 0 && c1 > c0 && c1 <= N, "head_region_mean: bad region");
    head_region_mean_kernel<<<BH, kThreads, 0, st>>>(g, out, N, ld, r0, r1, c0, c1);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_prep_mats(const float* in, float* out, long long rows, int N, int ld_in, int ld_out, int normalize,
                        cudaStream_t st) {
    if (rows <= 0) return TE_OK;
    prep_mats_kernel<<<warp_rows_grid(rows), kThreads, 0, st>>>(in, out, rows, N, ld_in, ld_out, normalize);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_extract_row(const float* joint, float* out, int B, int N, int ld, int first, int bert_fix,
                          cudaStream_t st) {
    extract_row_kernel<<<warp_rows_grid(B), kThreads, 0, st>>>(joint, out, B, N, ld, first, bert_fix);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_average2(const float* a, const float* b, float* out, long long n, cudaStream_t st) {
    average2_kernel<<<flat_grid(n), kThreads, 0, st>>>(a, b, out, n);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_bert_embed(const long long* ids, const long long* token_type_ids, const float* word, const float* pos,
                         const float* type, float* out, int B, int S, int D, int vocab, int type_vocab, cudaStream_t st) {
    TE_REQ(D % 4 == 0, "bert_embed: D % 4 != 0");
    bert_embed_kernel<<<flat_grid((long long)B * S * (D / 4)), kThreads, 0, st>>>(ids, token_type_ids, word, pos, type, out,
                                                                                 B, S, D, vocab, type_vocab);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_hf_embed(const long long* ids, const long long* token_type_ids, const float* word, const float* pos,
                       const float* type, float* out, int B, int S, int D, int vocab, int max_position, int type_vocab,
                       int pad, cudaStream_t st) {
    TE_REQ(D % 4 == 0, "hf_embed: D % 4 != 0");
    TE_REQ(B >= 1 && B <= 65535 && S >= 1, "hf_embed: batch outside 1..65535 or empty sequence");
    hf_embed_kernel<<<dim3((S + kEmbedTile - 1) / kEmbedTile, B), 256, 0, st>>>(ids, token_type_ids, word, pos, type, out, S,
                                                                               D, vocab, max_position, type_vocab, pad);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_bert_mask(const long long* mask, float* out, long long n, cudaStream_t st) {
    bert_mask_kernel<<<flat_grid(n), kThreads, 0, st>>>(mask, out, n);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_tanh(const float* x, float* y, long long n, cudaStream_t st) {
    tanh_kernel<<<flat_grid(n), kThreads, 0, st>>>(x, y, n);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_tanh_bwd(const float* dy, const float* y, float* dx, long long n, cudaStream_t st) {
    tanh_bwd_kernel<<<flat_grid(n), kThreads, 0, st>>>(dy, y, dx, n);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_relu(const float* x, float* y, long long n, cudaStream_t st) {
    relu_kernel<<<flat_grid(n), kThreads, 0, st>>>(x, y, n);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_relu_bwd(const float* dy, const float* y, float* dx, long long n, cudaStream_t st) {
    relu_bwd_kernel<<<flat_grid(n), kThreads, 0, st>>>(dy, y, dx, n);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_add2(const float* a, const float* b, float* out, long long n, cudaStream_t st) {
    TE_REQ(n % 4 == 0, "add2: n % 4 != 0");
    add2_kernel<<<flat_grid(n / 4), kThreads, 0, st>>>(a, b, out, n / 4);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_add_relprop_keymask(const float* x1, const float* keymask, const float* r, float* r1, double* partial,
                                  int B, int H, int N, int ld, cudaStream_t st) {
    TE_REQ(B <= 65535, "add_relprop_keymask: batch too large for one launch");
    if (partial) {                            // null: Add of modules/layers_lrp.py (RelPropSimple) — x1 * S only
        add_keymask_reduce_kernel<<<dim3(TE_ADD_SPLIT, B), kThreads, 0, st>>>(x1, keymask, r, partial, H * N, N, ld);
        TE_CUDA_CHECK_LAUNCH();
    }
    int gx = (H * N + 7) / 8;
    gx = gx > 64 ? 64 : gx;
    add_keymask_scale_kernel<<<dim3(gx, B), kThreads, 0, st>>>(x1, keymask, r, r1, partial, H * N, N, ld);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
int te_launch_fill(float* p, float v, long long n, cudaStream_t st) {
    if (n <= 0) return TE_OK;
    fill_kernel<<<flat_grid(n), kThreads, 0, st>>>(p, v, n);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
