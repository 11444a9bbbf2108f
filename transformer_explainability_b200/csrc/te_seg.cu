// ImageNet-segmentation evaluation (baselines/ViT/imagenet_seg_eval.py:212-277, 312-314; utils/metrices.py):
//   * seg_prepare_kernel: one block per sample.  The map is up-sampled on the fly (the bilinear arithmetic of
//     relevance_heatmap_kernel, te_elementwise.cu), min-max normalised and thresholded at its mean; it counts TP / FP / FN /
//     TN and emits the sort keys of the two AP score channels (1 - Res, Res) and, optionally, of the PR-curve scores.
//   * te_sort_keys_u32: stable LSD radix sort of uint32 keys (4 passes of 8-bit digits), one segment or `segments` equal
//     segments sorted independently; per pass a tile histogram, a scan of the [segment, digit, tile] counts and a stable
//     scatter (per-warp ranks through __match_any_sync, then per-digit warp offsets).
//   * seg_ap_kernel: one block per sample over its sorted keys: sklearn's average_precision_score (step integral of the
//     precision-recall curve, tie groups of bit-equal scores) in fp64, in a fixed order.
//   * te_pr_curve: sklearn's _binary_clf_curve over globally sorted keys (device-wide scan + compaction).
// A key is bits(score) << 1 | is_positive for a score >= 0 (-0 mapped to +0), so ascending key order is ascending score
// order and equal scores form one contiguous run.
#include "../../include/te_b200.h"
#include "te_kernels.h"

namespace {

constexpr int kPrepThreads = 1024;
constexpr int kApThreads = 1024;
constexpr int kSortThreads = 256;
constexpr int kSortWarps = kSortThreads / 32;
constexpr int kSortItems = 16;
constexpr int kSortTile = kSortThreads * kSortItems;      // 4096 keys: each warp owns 512 consecutive keys
constexpr int kScanThreads = 1024;
constexpr int kPrThreads = 256;
constexpr int kPrItems = 16;
constexpr int kPrTile = kPrThreads * kPrItems;
constexpr int kMaxSegShared = 45056;                       // dynamic shared bytes of seg_prepare_kernel: map + row counts

__device__ __forceinline__ uint32_t score_key(float s, bool positive) {
    if (s == 0.f) s = 0.f;                                 // -0 == +0
    return (__float_as_uint(s) << 1) | (positive ? 1u : 0u);
}

// ---- block reductions in a fixed order (deterministic for a fixed thread -> element assignment) ------------------------
template <typename T> __device__ __forceinline__ T warp_sum_t(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
template <typename T, int THREADS> __device__ T block_sum(T v, T* red) {
    v = warp_sum_t(v);
    __syncthreads();                                       // red may still be read by a previous call
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x < 32) {
        T w = threadIdx.x < THREADS / 32 ? red[threadIdx.x] : T(0);
        w = warp_sum_t(w);
        if (threadIdx.x == 0) red[0] = w;
    }
    __syncthreads();
    return red[0];
}

// relevance_heatmap_kernel's bilinear value at pixel p of the G x G output (G = g * scale); scale 1: the map itself
__device__ __forceinline__ float seg_value(const float* m, int g, int scale, int G, float rs, int p) {
    if (scale == 1) return m[p];
    const int y = p / G, x = p % G;
    const float sy = fmaxf(rs * ((float)y + 0.5f) - 0.5f, 0.f), sx = fmaxf(rs * ((float)x + 0.5f) - 0.5f, 0.f);
    const int y0 = (int)sy, x0 = (int)sx;
    const int y1 = y0 + (y0 < g - 1 ? 1 : 0), x1 = x0 + (x0 < g - 1 ? 1 : 0);
    const float ly1 = sy - (float)y0, ly0 = 1.f - ly1, lx1 = sx - (float)x0, lx0 = 1.f - lx1;
    return ly0 * (lx0 * m[y0 * g + x0] + lx1 * m[y0 * g + x1]) + ly1 * (lx0 * m[y1 * g + x0] + lx1 * m[y1 * g + x1]);
}

// One block per sample.  Pass 1: min / max of the up-sampled map; pass 2: mean of Res = (v - min) / (max - min) (fp64
// accumulation, one rounding to fp32); pass 3: threshold Res > mean, counts, AP keys [2P] (channel 0: 1 - Res positive on
// label 0, channel 1: Res positive on label 1) and the PR keys [P] of clamp(Res, thr) / max(Res), positive on label 1.
// A degenerate map (max == min, or NaN in the map) normalises to NaN everywhere: every pixel is background and every score
// is 0, as in the reference after its NaN -> 0 replacement.
__global__ void __launch_bounds__(kPrepThreads) seg_prepare_kernel(
        const float* __restrict__ maps, const int* __restrict__ labels, int g, int scale, float thr, float* __restrict__ mean_out,
        long long* __restrict__ counts, int* __restrict__ row_counts, int* __restrict__ degenerate, long long* __restrict__ invalid,
        uint32_t* __restrict__ ap_keys, uint32_t* __restrict__ pr_keys) {
    extern __shared__ float sgrid[];                       // [scale > 1 ? g*g : 0] map, then [G][3] row counts
    __shared__ double dred[32];
    __shared__ long long lred[32];
    __shared__ float fmn[32], fmx[32];
    __shared__ int snan[32];
    const int b = blockIdx.x;
    const int G = g * scale, P = G * G;
    const float rs = 1.0f / (float)scale;
    const float* src = maps + (long long)b * g * g;
    const float* m = src;
    int* srow = reinterpret_cast<int*>(sgrid + (scale > 1 ? g * g : 0));
    for (int i = threadIdx.x; i < 3 * G; i += blockDim.x) srow[i] = 0;
    if (scale > 1) {
        for (int i = threadIdx.x; i < g * g; i += blockDim.x) sgrid[i] = src[i];
        m = sgrid;
    }
    __syncthreads();
    // pass 1
    float mn = INFINITY, mx = -INFINITY;
    int nan = 0;
    for (int p = threadIdx.x; p < P; p += blockDim.x) {
        const float v = seg_value(m, g, scale, G, rs, p);
        mn = fminf(mn, v); mx = fmaxf(mx, v);
        nan |= v != v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        nan |= __shfl_xor_sync(0xffffffffu, nan, o);
    }
    if ((threadIdx.x & 31) == 0) { fmn[threadIdx.x >> 5] = mn; fmx[threadIdx.x >> 5] = mx; snan[threadIdx.x >> 5] = nan; }
    __syncthreads();
    mn = fmn[0]; mx = fmx[0]; nan = snan[0];
    for (int w = 1; w < kPrepThreads / 32; ++w) { mn = fminf(mn, fmn[w]); mx = fmaxf(mx, fmx[w]); nan |= snan[w]; }
    const float range = __fsub_rn(mx, mn);
    const bool degen = nan || !(mx > mn);
    // pass 2
    double s = 0.0;
    if (!degen)
        for (int p = threadIdx.x; p < P; p += blockDim.x)
            s += (double)__fdiv_rn(__fsub_rn(seg_value(m, g, scale, G, rs, p), mn), range);
    s = block_sum<double, kPrepThreads>(s, dred);
    const float mean = degen ? NAN : (float)(s / (double)P);
    const float vmax = __fdiv_rn(range, range);            // max(Res): 1 for a finite non-degenerate map
    // pass 3
    long long tp = 0, fp = 0, fn = 0, tn = 0, bad = 0;
    uint32_t* ak = ap_keys + (long long)b * 2 * P;
    uint32_t* pk = pr_keys ? pr_keys + (long long)b * P : nullptr;
    for (int p = threadIdx.x; p < P; p += blockDim.x) {
        const int l = labels[(long long)b * P + p];
        bad += (l != 0 && l != 1);
        const bool pos = l == 1;
        float r = 0.f, r0 = 0.f, pred = 0.f;
        bool fg = false;
        if (!degen) {
            r = __fdiv_rn(__fsub_rn(seg_value(m, g, scale, G, rs, p), mn), range);
            r0 = __fsub_rn(1.f, r);
            fg = r > mean;
            pred = __fdiv_rn(fmaxf(r, thr), vmax);
        }
        tp += fg && pos; fp += fg && !pos; fn += !fg && pos; tn += !fg && !pos;
        if (fg || pos) atomicAdd(&srow[3 * (p / G) + (fg && pos ? 0 : fg ? 1 : 2)], 1);
        ak[p] = score_key(r0, !pos);
        ak[P + p] = score_key(r, pos);
        if (pk) pk[p] = score_key(pred, pos);
    }
    tp = block_sum<long long, kPrepThreads>(tp, lred);
    fp = block_sum<long long, kPrepThreads>(fp, lred);
    fn = block_sum<long long, kPrepThreads>(fn, lred);
    tn = block_sum<long long, kPrepThreads>(tn, lred);
    bad = block_sum<long long, kPrepThreads>(bad, lred);
    if (threadIdx.x == 0) {
        mean_out[b] = mean;
        counts[4 * b + 0] = tp; counts[4 * b + 1] = fp; counts[4 * b + 2] = fn; counts[4 * b + 3] = tn;
        degenerate[b] = degen ? 1 : 0;
        invalid[b] = bad;
    }
    for (int i = threadIdx.x; i < 3 * G; i += blockDim.x) row_counts[(long long)b * 3 * G + i] = srow[i];
}

// ---- LSD radix sort ------------------------------------------------------------------------------------------------------
// counts[(seg * 256 + digit) * tiles + tile]: keys of the tile with that digit.  grid (tiles, segments)
__global__ void __launch_bounds__(kSortThreads) sort_hist_kernel(const uint32_t* __restrict__ in, long long L, int tiles, int shift,
                                                                 uint32_t* __restrict__ counts) {
    __shared__ uint32_t h[256];
    const int tile = blockIdx.x, seg = blockIdx.y;
    const int lane = threadIdx.x & 31;
    for (int i = threadIdx.x; i < 256; i += blockDim.x) h[i] = 0;
    __syncthreads();
    const long long t0 = (long long)tile * kSortTile;
    const uint32_t* src = in + (long long)seg * L;
    for (int i = 0; i < kSortItems; ++i) {
        const long long idx = t0 + (long long)i * kSortThreads + threadIdx.x;
        const bool valid = idx < L;
        const uint32_t d = valid ? (src[idx] >> shift) & 255u : 256u + lane;
        const uint32_t peers = __match_any_sync(0xffffffffu, d);
        if (valid && lane == __ffs(peers) - 1) atomicAdd(&h[d], (uint32_t)__popc(peers));
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 256; i += blockDim.x) counts[((long long)seg * 256 + i) * tiles + tile] = h[i];
}

// totals[seg * 256 + digit] = sum over tiles.  grid (256, segments)
__global__ void __launch_bounds__(kScanThreads) sort_total_kernel(const uint32_t* __restrict__ counts, int tiles,
                                                                  uint32_t* __restrict__ totals) {
    __shared__ long long red[32];
    const uint32_t* c = counts + ((long long)blockIdx.y * 256 + blockIdx.x) * tiles;
    long long s = 0;
    for (int t = threadIdx.x; t < tiles; t += blockDim.x) s += c[t];
    s = block_sum<long long, kScanThreads>(s, red);
    if (threadIdx.x == 0) totals[blockIdx.y * 256 + blockIdx.x] = (uint32_t)s;
}

// counts -> exclusive offsets within the segment: base(digit) + scan over the tiles.  grid (256, segments)
__global__ void __launch_bounds__(kScanThreads) sort_offsets_kernel(uint32_t* __restrict__ counts, int tiles,
                                                                    const uint32_t* __restrict__ totals) {
    __shared__ uint32_t wsum[32];
    __shared__ uint32_t carry;
    const int d = blockIdx.x, seg = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) {
        uint32_t base = 0;
        for (int e = 0; e < d; ++e) base += totals[seg * 256 + e];
        carry = base;
    }
    __syncthreads();
    uint32_t* c = counts + ((long long)seg * 256 + d) * tiles;
    for (int t0 = 0; t0 < tiles; t0 += blockDim.x) {
        const int t = t0 + threadIdx.x;
        const uint32_t v = t < tiles ? c[t] : 0u;
        uint32_t incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t u = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += u;
        }
        if (lane == 31) wsum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            uint32_t w = wsum[lane], wi = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t u = __shfl_up_sync(0xffffffffu, wi, o);
                if (lane >= o) wi += u;
            }
            wsum[lane] = wi - w;                            // exclusive prefix of the warps
        }
        __syncthreads();
        const uint32_t base = carry;
        if (t < tiles) c[t] = base + wsum[warp] + incl - v;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry = base + wsum[warp] + incl;
        __syncthreads();
    }
}

// stable scatter of one tile: warp w owns keys [w*512, (w+1)*512) of the tile in 16 rounds of 32 consecutive keys.  grid (tiles, segments)
__global__ void __launch_bounds__(kSortThreads) sort_scatter_kernel(const uint32_t* __restrict__ in, uint32_t* __restrict__ out,
                                                                    long long L, int tiles, int shift,
                                                                    const uint32_t* __restrict__ offsets) {
    __shared__ uint32_t wcnt[kSortWarps][256];
    __shared__ uint32_t tbase[256];
    const int tile = blockIdx.x, seg = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < kSortWarps * 256; i += blockDim.x) (&wcnt[0][0])[i] = 0;
    for (int i = threadIdx.x; i < 256; i += blockDim.x) tbase[i] = offsets[((long long)seg * 256 + i) * tiles + tile];
    __syncthreads();
    const long long t0 = (long long)tile * kSortTile + warp * (kSortItems * 32);
    const uint32_t* src = in + (long long)seg * L;
    uint32_t key[kSortItems], loc[kSortItems];
#pragma unroll
    for (int r = 0; r < kSortItems; ++r) {
        const long long idx = t0 + r * 32 + lane;
        const bool valid = idx < L;
        key[r] = valid ? src[idx] : 0u;
        const uint32_t d = valid ? (key[r] >> shift) & 255u : 256u + lane;
        const uint32_t peers = __match_any_sync(0xffffffffu, d);
        const uint32_t before = valid ? wcnt[warp][d] : 0u;
        __syncwarp();
        if (valid && lane == __ffs(peers) - 1) wcnt[warp][d] = before + __popc(peers);
        __syncwarp();
        loc[r] = before + __popc(peers & ((1u << lane) - 1u));
    }
    __syncthreads();
    {
        const int d = threadIdx.x;                          // kSortThreads == 256: one digit per thread
        uint32_t run = 0;
        for (int w = 0; w < kSortWarps; ++w) { const uint32_t c = wcnt[w][d]; wcnt[w][d] = run; run += c; }
    }
    __syncthreads();
    uint32_t* dst = out + (long long)seg * L;
#pragma unroll
    for (int r = 0; r < kSortItems; ++r) {
        const long long idx = t0 + r * 32 + lane;
        if (idx < L) {
            const uint32_t d = (key[r] >> shift) & 255u;
            dst[tbase[d] + wcnt[warp][d] + loc[r]] = key[r];
        }
    }
}

struct SortLayout {
    long long L;
    int tiles;
    long long keys_bytes, counts_bytes, totals_bytes;
};
SortLayout sort_layout(long long n, int segments) {
    SortLayout s;
    s.L = n / segments;
    s.tiles = (int)((s.L + kSortTile - 1) / kSortTile);
    s.keys_bytes = (n * 4 + 255) / 256 * 256;
    s.counts_bytes = ((long long)segments * 256 * s.tiles * 4 + 255) / 256 * 256;
    s.totals_bytes = ((long long)segments * 256 * 4 + 255) / 256 * 256;
    return s;
}

int sort_keys(const uint32_t* in, uint32_t* out, long long n, int segments, char* ws, cudaStream_t st) {
    if (n == 0) return TE_OK;
    const SortLayout s = sort_layout(n, segments);
    uint32_t* tmp = reinterpret_cast<uint32_t*>(ws);
    uint32_t* counts = reinterpret_cast<uint32_t*>(ws + s.keys_bytes);
    uint32_t* totals = reinterpret_cast<uint32_t*>(ws + s.keys_bytes + s.counts_bytes);
    // in -> tmp -> out -> tmp -> out (in == out is fine: in is consumed by the first pass)
    const uint32_t* src = in;
    for (int pass = 0; pass < 4; ++pass) {
        uint32_t* dst = (pass & 1) ? out : tmp;
        const int shift = 8 * pass;
        const dim3 grid(s.tiles, segments);
        sort_hist_kernel<<<grid, kSortThreads, 0, st>>>(src, s.L, s.tiles, shift, counts);
        TE_CUDA_CHECK_LAUNCH();
        sort_total_kernel<<<dim3(256, segments), kScanThreads, 0, st>>>(counts, s.tiles, totals);
        TE_CUDA_CHECK_LAUNCH();
        sort_offsets_kernel<<<dim3(256, segments), kScanThreads, 0, st>>>(counts, s.tiles, totals);
        TE_CUDA_CHECK_LAUNCH();
        sort_scatter_kernel<<<grid, kSortThreads, 0, st>>>(src, dst, s.L, s.tiles, shift, counts);
        TE_CUDA_CHECK_LAUNCH();
        src = dst;
    }
    return TE_OK;
}

// ---- block scans over per-thread aggregates (warp 0 scans the shared array, lane l owns THREADS/32 consecutive entries) ---
// tie-group aggregate: tp = positives; f = a group starts in the range; c = positives since the last group start in the
// range (or since its beginning).  (a then b) = (a.tp + b.tp, a.f | b.f, b.f ? b.c : a.c + b.c)
struct GroupAgg {
    long long tp;
    int f;
    long long c;
};
__device__ __forceinline__ GroupAgg combine(const GroupAgg& a, const GroupAgg& b) {
    return GroupAgg{a.tp + b.tp, a.f | b.f, b.f ? b.c : a.c + b.c};
}
// in: agg[threadIdx.x] (inclusive aggregate of the thread's range); out: agg[threadIdx.x] = exclusive prefix
template <int THREADS> __device__ void block_exclusive_scan(GroupAgg* agg) {
    __syncthreads();
    if (threadIdx.x < 32) {
        constexpr int per = THREADS / 32;
        const int lane = threadIdx.x;
        GroupAgg run{0, 0, 0};
        for (int i = 0; i < per; ++i) run = combine(run, agg[lane * per + i]);
        GroupAgg incl = run;                                // inclusive scan of the lane totals (Hillis-Steele)
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            GroupAgg u;
            u.tp = __shfl_up_sync(0xffffffffu, incl.tp, o);
            u.f = __shfl_up_sync(0xffffffffu, incl.f, o);
            u.c = __shfl_up_sync(0xffffffffu, incl.c, o);
            if (lane >= o) incl = combine(u, incl);
        }
        GroupAgg ex;
        ex.tp = __shfl_up_sync(0xffffffffu, incl.tp, 1);
        ex.f = __shfl_up_sync(0xffffffffu, incl.f, 1);
        ex.c = __shfl_up_sync(0xffffffffu, incl.c, 1);
        if (lane == 0) ex = GroupAgg{0, 0, 0};
        for (int i = 0; i < per; ++i) {
            const GroupAgg v = agg[lane * per + i];
            agg[lane * per + i] = ex;
            ex = combine(ex, v);
        }
    }
    __syncthreads();
}

// AP of one sample over its 2P ascending keys, visited in descending order (position d <-> index n - 1 - d):
// AP = sum over tie groups of (positives in the group) * tp(end) / (end + 1), divided by the number of positives.
// Thread t owns descending positions [t*C, (t+1)*C).
__global__ void __launch_bounds__(kApThreads) seg_ap_kernel(const uint32_t* __restrict__ keys, long long n, double* __restrict__ ap) {
    __shared__ GroupAgg agg[kApThreads];
    __shared__ double dred[32];
    __shared__ long long lred[32];
    const uint32_t* k = keys + (long long)blockIdx.x * n;
    const long long C = (n + kApThreads - 1) / kApThreads;
    const long long d0 = threadIdx.x * C, d1 = min(n, d0 + C);
    auto at = [&](long long d) { return k[n - 1 - d]; };
    GroupAgg a{0, 0, 0};
    for (long long d = d0; d < d1; ++d) {
        const uint32_t v = at(d);
        const bool start = d == 0 || (at(d - 1) >> 1) != (v >> 1);
        if (start) { a.f = 1; a.c = 0; }
        const long long pos = v & 1u;
        a.tp += pos; a.c += pos;
    }
    agg[threadIdx.x] = a;
    block_exclusive_scan<kApThreads>(agg);
    GroupAgg e = agg[threadIdx.x];
    long long tp = e.tp, c = e.c;
    double sum = 0.0;
    for (long long d = d0; d < d1; ++d) {
        const uint32_t v = at(d);
        if (d == 0 || (at(d - 1) >> 1) != (v >> 1)) c = 0;
        const long long pos = v & 1u;
        tp += pos; c += pos;
        if (d == n - 1 || (at(d + 1) >> 1) != (v >> 1)) sum += (double)c * ((double)tp / (double)(d + 1));
    }
    sum = block_sum<double, kApThreads>(sum, dred);
    const long long P = block_sum<long long, kApThreads>(d1 > d0 ? a.tp : 0, lred);
    if (threadIdx.x == 0) ap[blockIdx.x] = P > 0 ? fmax(0.0, sum / (double)P) : 0.0;   // no positive: sklearn's NaN -> 0
}

// ---- PR curve ------------------------------------------------------------------------------------------------------------
// per tile of kPrTile descending positions: (positives, group ends).  grid tiles
__global__ void __launch_bounds__(kPrThreads) pr_count_kernel(const uint32_t* __restrict__ k, long long n, long long* __restrict__ tile_tp,
                                                              long long* __restrict__ tile_ends) {
    __shared__ long long red[32];
    const long long d0 = (long long)blockIdx.x * kPrTile;
    long long tp = 0, ends = 0;
    for (int i = threadIdx.x; i < kPrTile; i += blockDim.x) {
        const long long d = d0 + i;
        if (d < n) {
            const uint32_t v = k[n - 1 - d];
            tp += v & 1u;
            ends += d == n - 1 || (k[n - 2 - d] >> 1) != (v >> 1);
        }
    }
    tp = block_sum<long long, kPrThreads>(tp, red);
    ends = block_sum<long long, kPrThreads>(ends, red);
    if (threadIdx.x == 0) { tile_tp[blockIdx.x] = tp; tile_ends[blockIdx.x] = ends; }
}

// exclusive scan of the tile totals in place, one block; *count = the number of groups
__global__ void __launch_bounds__(kScanThreads) pr_scan_kernel(long long* __restrict__ tile_tp, long long* __restrict__ tile_ends,
                                                               int tiles, long long* __restrict__ count) {
    __shared__ long long wtp[32], wen[32];
    __shared__ long long ctp, cen;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) { ctp = 0; cen = 0; }
    __syncthreads();
    for (int t0 = 0; t0 < tiles; t0 += blockDim.x) {
        const int t = t0 + threadIdx.x;
        const long long a = t < tiles ? tile_tp[t] : 0, b = t < tiles ? tile_ends[t] : 0;
        long long ia = a, ib = b;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const long long ua = __shfl_up_sync(0xffffffffu, ia, o), ub = __shfl_up_sync(0xffffffffu, ib, o);
            if (lane >= o) { ia += ua; ib += ub; }
        }
        if (lane == 31) { wtp[warp] = ia; wen[warp] = ib; }
        __syncthreads();
        if (warp == 0) {
            const long long xa = wtp[lane], xb = wen[lane];
            long long sa = xa, sb = xb;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const long long ua = __shfl_up_sync(0xffffffffu, sa, o), ub = __shfl_up_sync(0xffffffffu, sb, o);
                if (lane >= o) { sa += ua; sb += ub; }
            }
            wtp[lane] = sa - xa; wen[lane] = sb - xb;
        }
        __syncthreads();
        const long long btp = ctp, ben = cen;
        if (t < tiles) { tile_tp[t] = btp + wtp[warp] + ia - a; tile_ends[t] = ben + wen[warp] + ib - b; }
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) { ctp = btp + wtp[warp] + ia; cen = ben + wen[warp] + ib; }
        __syncthreads();
    }
    if (threadIdx.x == 0) *count = cen;
}

// each group end at descending position d: thresholds[j] = score, tps[j] = positives in [0, d], fps[j] = d + 1 - tps[j],
// j = the number of group ends before d.  Thread t of a tile owns kPrItems consecutive positions.
__global__ void __launch_bounds__(kPrThreads) pr_write_kernel(const uint32_t* __restrict__ k, long long n,
                                                              const long long* __restrict__ tile_tp,
                                                              const long long* __restrict__ tile_ends, float* __restrict__ thr,
                                                              long long* __restrict__ tps, long long* __restrict__ fps) {
    __shared__ GroupAgg agg[kPrThreads];                   // tp = positives, c = group ends (f unused: plain sums)
    const long long d0 = (long long)blockIdx.x * kPrTile + (long long)threadIdx.x * kPrItems;
    GroupAgg a{0, 0, 0};
    for (int i = 0; i < kPrItems; ++i) {
        const long long d = d0 + i;
        if (d < n) {
            const uint32_t v = k[n - 1 - d];
            a.tp += v & 1u;
            a.c += d == n - 1 || (k[n - 2 - d] >> 1) != (v >> 1);
        }
    }
    agg[threadIdx.x] = a;
    block_exclusive_scan<kPrThreads>(agg);
    long long tp = tile_tp[blockIdx.x] + agg[threadIdx.x].tp, j = tile_ends[blockIdx.x] + agg[threadIdx.x].c;
    for (int i = 0; i < kPrItems; ++i) {
        const long long d = d0 + i;
        if (d >= n) break;
        const uint32_t v = k[n - 1 - d];
        tp += v & 1u;
        if (d == n - 1 || (k[n - 2 - d] >> 1) != (v >> 1)) {
            thr[j] = __uint_as_float(v >> 1);
            tps[j] = tp;
            fps[j] = d + 1 - tp;
            ++j;
        }
    }
}

}  // namespace

#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define REQ(c, msg) do { if (!(c)) { te_set_last_error(msg); return TE_ERR_ARG; } } while (0)

extern "C" long long te_sort_workspace_bytes(long long n, int segments) {
    if (n < 0 || segments <= 0 || n % segments != 0 || n / segments > 0x7fffffffLL) return TE_ERR_ARG;
    const SortLayout s = sort_layout(n, segments);
    return s.keys_bytes + s.counts_bytes + s.totals_bytes;
}

extern "C" int te_sort_keys_u32(const unsigned* keys_in, unsigned* keys_out, long long n, int segments, void* workspace,
                                long long workspace_bytes, void* stream) {
    REQ(n >= 0 && segments > 0 && n % segments == 0, "te_sort_keys_u32: n must be a non-negative multiple of segments");
    REQ(n / segments <= 0x7fffffffLL, "te_sort_keys_u32: a segment holds at most 2^31 - 1 keys");
    if (n == 0) return TE_OK;
    REQ(keys_in && keys_out, "te_sort_keys_u32: null argument");
    REQ(workspace && (((uintptr_t)workspace) & 255u) == 0, "te_sort_keys_u32: workspace null or not 256-byte aligned");
    if (te_sort_workspace_bytes(n, segments) > workspace_bytes) {
        te_set_last_error("te_sort_keys_u32: workspace too small");
        return TE_ERR_WORKSPACE;
    }
    return sort_keys(keys_in, keys_out, n, segments, static_cast<char*>(workspace), ST(stream));
}

extern "C" long long te_seg_workspace_bytes(int batch, int grid, int scale) {
    if (batch <= 0 || grid <= 0 || scale <= 0 || (long long)grid * scale > 46340) return TE_ERR_ARG;
    const long long P = (long long)grid * scale * grid * scale;
    const long long n = 2 * P * batch;
    const long long sort = te_sort_workspace_bytes(n, batch);
    if (sort < 0) return sort;
    return (n * 4 + 255) / 256 * 256 + sort;
}

extern "C" int te_seg_metrics(const float* maps, const int* labels, int batch, int grid, int scale, float thr, float* mean,
                              long long* counts, int* row_counts, double* ap, int* degenerate, long long* invalid, unsigned* pr_keys,
                              void* workspace, long long workspace_bytes, void* stream) {
    REQ(maps && labels && mean && counts && row_counts && ap && degenerate && invalid, "te_seg_metrics: null argument");
    REQ(batch > 0 && grid > 0 && scale > 0 && (long long)grid * scale <= 46340, "te_seg_metrics: bad batch / grid / scale");
    const size_t smem = ((scale > 1 ? (size_t)grid * grid : 0) + 3 * (size_t)grid * scale) * 4;
    REQ(smem <= (size_t)kMaxSegShared, "te_seg_metrics: 4 * grid^2 (scale > 1) + 12 * grid * scale must be at most 45056 bytes");
    REQ(!(thr != thr), "te_seg_metrics: thr is NaN");
    REQ(workspace && (((uintptr_t)workspace) & 255u) == 0, "te_seg_metrics: workspace null or not 256-byte aligned");
    const long long ws = te_seg_workspace_bytes(batch, grid, scale);
    REQ(ws >= 0, "te_seg_metrics: the keys of one sample exceed 2^31 - 1");
    if (ws > workspace_bytes) {
        te_set_last_error("te_seg_metrics: workspace too small");
        return TE_ERR_WORKSPACE;
    }
    const long long P = (long long)grid * scale * grid * scale;
    const long long n = 2 * P * batch;
    uint32_t* ak = static_cast<uint32_t*>(workspace);
    char* sort_ws = static_cast<char*>(workspace) + (n * 4 + 255) / 256 * 256;
    seg_prepare_kernel<<<batch, kPrepThreads, smem, ST(stream)>>>(maps, labels, grid, scale, thr, mean, counts, row_counts, degenerate, invalid,
                                                                  ak, pr_keys);
    TE_CUDA_CHECK_LAUNCH();
    const int rc = sort_keys(ak, ak, n, batch, sort_ws, ST(stream));
    if (rc != TE_OK) return rc;
    seg_ap_kernel<<<batch, kApThreads, 0, ST(stream)>>>(ak, 2 * P, ap);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}

extern "C" long long te_pr_curve_workspace_bytes(long long n) {
    if (n <= 0) return TE_ERR_ARG;
    const long long tiles = (n + kPrTile - 1) / kPrTile;
    if (tiles > 0x7fffffffLL) return TE_ERR_ARG;
    return (tiles * 16 + 255) / 256 * 256;
}

extern "C" int te_pr_curve(const unsigned* keys, long long n, float* thresholds, long long* tps, long long* fps, long long* count,
                           void* workspace, long long workspace_bytes, void* stream) {
    REQ(keys && thresholds && tps && fps && count, "te_pr_curve: null argument");
    REQ(n > 0, "te_pr_curve: n must be positive");
    REQ(workspace && (((uintptr_t)workspace) & 255u) == 0, "te_pr_curve: workspace null or not 256-byte aligned");
    if (te_pr_curve_workspace_bytes(n) > workspace_bytes) {
        te_set_last_error("te_pr_curve: workspace too small");
        return TE_ERR_WORKSPACE;
    }
    const long long tiles = (n + kPrTile - 1) / kPrTile;
    long long* tile_tp = static_cast<long long*>(workspace);
    long long* tile_ends = tile_tp + tiles;
    pr_count_kernel<<<(unsigned)tiles, kPrThreads, 0, ST(stream)>>>(keys, n, tile_tp, tile_ends);
    TE_CUDA_CHECK_LAUNCH();
    pr_scan_kernel<<<1, kScanThreads, 0, ST(stream)>>>(tile_tp, tile_ends, (int)tiles, count);
    TE_CUDA_CHECK_LAUNCH();
    pr_write_kernel<<<(unsigned)tiles, kPrThreads, 0, ST(stream)>>>(keys, n, tile_tp, tile_ends, thresholds, tps, fps);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
