// ERASER rationale evaluation (BERT_rationale_benchmark/models/pipeline/bert_pipeline.py:96-138,547-582; metrics.py:111-215):
//   * eraser_kernel: one block per document.  Word scores are the max over each word's word-piece range of the clamped map
//     (NaN propagates); the words are ranked NaN first, then by descending score, then by ascending word index (the order
//     key of te_perturb_images); the first kmax ranks are written out, and per k the counts of the predicted words that
//     metrics.py's hard-rationale scores need come from prefix sums along that order.
//   * reduce_kernel: one block per document, the ranking of eraser_kernel; each piece is marked with the smallest rank of
//     the words holding it, and per selection size n the pieces of the first n ranks (sufficiency) and the other inner
//     pieces (comprehensiveness) are compacted, between the document's [CLS] and [SEP], by one block scan.
//   * soft_kernel: one block per document, the ranking of eraser_kernel over given word scores; the tie groups' cumulative
//     (tps, fps) come from one warp scan, and metrics.py's soft-token areas (:217-253) are reduced in fp64.
//   * latex_kernel: one block per row, the colour weights of bert_pipeline.py's generate() (:49-56): the row's NaN-aware
//     min / max by a block reduction, then the reference's fp32 operations in its order with explicit IEEE roundings.
// The ragged host arrays (word piece ranges, truth spans, their offsets) are validated on the host and copied into the
// workspace, so no index the caller passes is read from the map before it has been checked.
#include "../../include/te_b200.h"
#include "te_kernels.h"

namespace {

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr int kIndicators = 2 + TE_ERASER_MAX_THRESHOLDS;     // tok_hits, span_hits, iou_hits[t]

struct EraserParams {
    int nk, nthr, kmax;
    int k[TE_ERASER_MAX_KS];
    double thr[TE_ERASER_MAX_THRESHOLDS];
};

// te_perturb_images' order key: larger = ranked earlier; -0 == +0; NaN on top
__device__ __forceinline__ uint32_t order_key(float v) {
    if (v != v) return 0xffffffffu;
    if (v == 0.f) v = 0.f;
    const uint32_t b = __float_as_uint(v);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// Rank the W words of one document by the scores score(w): skey[w] = (~order_key << 32) | w, sword[r] = the word at rank r
// (NaN first, then descending score, then ascending word index).  Ends with a block barrier.
template <class Score>
__device__ __forceinline__ void rank_scores(Score score, int W, unsigned long long* skey, int* sword) {
    for (int w = threadIdx.x; w < W; w += blockDim.x)
        skey[w] = ((unsigned long long)(~order_key(score(w))) << 32) | (unsigned)w;   // ascending = ranking order
    __syncthreads();
    // rank = number of smaller keys (all keys are distinct)
    for (int w = threadIdx.x; w < W; w += blockDim.x) {
        const unsigned long long k = skey[w];
        int rank = 0;
        for (int u = 0; u < W; ++u) rank += skey[u] < k;
        sword[rank] = w;
    }
    __syncthreads();
}

// Score and rank the W words of one document (map row m, inclusive piece ranges): word_scores[w] (may be null) = the max
// of the clamped map over the word's pieces (NaN propagates), ranked by rank_scores.  Ends with a block barrier.
__device__ __forceinline__ void rank_words(const float* __restrict__ m, const int2* __restrict__ ranges, int W,
                                           float* __restrict__ word_scores, unsigned long long* skey, int* sword) {
    rank_scores([&](int w) {
        const int2 r = ranges[w];
        float s = 0.f;
        bool nan = false, first = true;
        for (int p = r.x; p <= r.y; ++p) {
            float v = m[p];
            if (v != v) { nan = true; continue; }
            v = v < 0.f ? 0.f : v;                                 // clamp(min=0)
            s = first ? v : fmaxf(s, v);
            first = false;
        }
        if (nan) s = __int_as_float(0x7fc00000);
        if (word_scores) word_scores[w] = s;
        return s;
    }, W, skey, sword);
}

__global__ void __launch_bounds__(kThreads) eraser_kernel(
        const float* __restrict__ maps, int seq, const int* __restrict__ word_off, const int2* __restrict__ ranges,
        const int* __restrict__ span_off, const int2* __restrict__ spans, EraserParams prm, float* __restrict__ word_scores,
        int* __restrict__ order, int* __restrict__ counts) {
    __shared__ unsigned long long skey[TE_ERASER_MAX_WORDS];       // (~key << 32) | word: ascending = ranking order
    __shared__ int sword[TE_ERASER_MAX_WORDS];                     // word at each rank
    __shared__ unsigned short sind[kIndicators][TE_ERASER_MAX_WORDS];   // indicators along the ranking, then their prefix sums
    const int b = blockIdx.x;
    const int w0 = word_off[b], W = word_off[b + 1] - w0;
    const int s0 = span_off[b], S = span_off[b + 1] - s0;
    const float* m = maps + (long long)b * seq;
    const int nind = 2 + prm.nthr;

    rank_words(m, ranges + w0, W, word_scores + w0, skey, sword);
    int* ord = order + (long long)b * prm.kmax;
    for (int r = threadIdx.x; r < prm.kmax; r += kThreads) ord[r] = r < W ? sword[r] : -1;

    // indicators of the word at each rank against the document's truth spans [start, end)
    for (int r = threadIdx.x; r < W; r += kThreads) {
        const int w = sword[r];
        bool tok = false, single = false;
        int minlen = 0x7fffffff;
        for (int j = 0; j < S; ++j) {
            const int2 t = spans[s0 + j];
            if (t.x <= w && w < t.y) {
                tok = true;
                minlen = min(minlen, t.y - t.x);
                single |= t.y - t.x == 1;
            }
        }
        // best IoU of the one-word span [w, w + 1): 1 / len of the shortest truth span holding w, else 0 (fp64, as Python)
        const double iou = tok ? 1.0 / (double)minlen : 0.0;
        sind[0][r] = tok;
        sind[1][r] = single;
        for (int t = 0; t < prm.nthr; ++t) sind[2 + t][r] = iou >= prm.thr[t];
    }
    __syncthreads();
    // inclusive prefix sums along the ranking: warp c scans indicator c, lane l owns ranks [l*C, (l+1)*C)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int C = (W + 31) / 32;
    for (int c = warp; c < nind; c += kWarps) {
        unsigned short* a = sind[c];
        const int r0 = lane * C, r1 = min(W, r0 + C);
        int sum = 0;
        for (int r = r0; r < r1; ++r) sum += a[r];
        int incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += u;
        }
        int run = incl - sum;
        for (int r = r0; r < r1; ++r) { run += a[r]; a[r] = (unsigned short)run; }
    }
    __syncthreads();
    // counts[b, i, :] = (n_pred, tok_hits, span_hits, iou_hits[0..nthr)) over the first min(k_i, W) ranks
    const int ncol = 1 + nind;
    for (int e = threadIdx.x; e < prm.nk * ncol; e += kThreads) {
        const int i = e / ncol, c = e - i * ncol;
        const int n = min(prm.k[i], W);
        counts[((long long)b * prm.nk + i) * ncol + c] = c == 0 ? n : (n > 0 ? (int)sind[c - 1][n - 1] : 0);
    }
}

// Reduced rows of document b for each selection size n = n_select[b, j]: every inner piece p in [1, len - 2] whose
// smallest holding rank is < n goes to the sufficiency row, every other inner piece to the comprehensiveness row, both in
// position order between the document's first ([CLS]) and last ([SEP]) token; zeros past each row's length.
__global__ void __launch_bounds__(kThreads) reduce_kernel(
        const float* __restrict__ maps, const long long* __restrict__ ids, int seq, const int* __restrict__ lens,
        const int* __restrict__ word_off, const int2* __restrict__ ranges, const int* __restrict__ n_select, int J,
        long long* __restrict__ out_ids, int* __restrict__ out_len) {
    __shared__ unsigned long long skey[TE_ERASER_MAX_WORDS];
    __shared__ int sword[TE_ERASER_MAX_WORDS];
    __shared__ int swarp[kWarps];
    extern __shared__ int pmin[];                                  // [seq]: smallest rank of the words holding each piece
    const int b = blockIdx.x;
    const int w0 = word_off[b], W = word_off[b + 1] - w0;
    const int len = lens[b];
    const long long* row = ids + (long long)b * seq;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

    for (int p = threadIdx.x; p < len; p += kThreads) pmin[p] = 0x7fffffff;
    rank_words(maps + (long long)b * seq, ranges + w0, W, nullptr, skey, sword);
    for (int r = threadIdx.x; r < W; r += kThreads) {
        const int2 rg = ranges[w0 + sword[r]];
        for (int p = rg.x; p <= rg.y; ++p) atomicMin(&pmin[p], r);
    }
    __syncthreads();
    const long long cls = row[0], sep = row[len - 1];
    for (int j = 0; j < J; ++j) {
        const int n = n_select[b * J + j];
        long long* comp = out_ids + (((long long)b * J + j) * 2) * seq;
        long long* suff = comp + seq;
        int carry = 0;                                             // rationale pieces before the current tile
        for (int t0 = 1; t0 <= len - 2; t0 += kThreads) {
            const int p = t0 + threadIdx.x;
            const bool in = p <= len - 2;
            const bool sel = in && pmin[p] < n;
            const unsigned ball = __ballot_sync(0xffffffffu, sel);
            if (lane == 0) swarp[warp] = __popc(ball);
            __syncthreads();
            int before = carry, total = carry;
            for (int u = 0; u < kWarps; ++u) {
                before += u < warp ? swarp[u] : 0;
                total += swarp[u];
            }
            before += __popc(ball & ((1u << lane) - 1u));
            if (in) {
                if (sel) suff[1 + before] = row[p];
                else comp[p - before] = row[p];                    // 1 + (p - 1 - before)
            }
            carry = total;
            __syncthreads();                                       // swarp is rewritten by the next tile
        }
        const int R = carry;
        const int lc = len - R, ls = 2 + R;
        for (int p = threadIdx.x; p < seq; p += kThreads) {
            if (p >= lc) comp[p] = 0;
            if (p >= ls) suff[p] = 0;
        }
        if (threadIdx.x == 0) {
            comp[0] = cls;
            comp[lc - 1] = sep;
            suff[0] = cls;
            suff[ls - 1] = sep;
            out_len[(b * J + j) * 2] = lc;
            out_len[(b * J + j) * 2 + 1] = ls;
        }
    }
}

// score_soft_tokens' three areas of document b (metrics.py:217-253) from its W word scores and its tail (tail[b] = the
// positive and negative words past truncation, which score 0): the words are ranked by rank_scores, so bit-equal scores
// (-0 == +0) are contiguous; a warp scan of (positive, tie-group end) along the ranks gives each group's cumulative
// (tps, fps), _binary_clf_curve's points; the tail joins the last group when it scores 0, else follows it as its own
// group (the scores are >= 0); the areas are summed per group in fp64 and reduced over the block.
__global__ void __launch_bounds__(kThreads) soft_kernel(
        const float* __restrict__ word_scores, const int* __restrict__ word_off, const int* __restrict__ span_off,
        const int2* __restrict__ spans, const int2* __restrict__ tail, double* __restrict__ scores, int* __restrict__ flags) {
    __shared__ unsigned long long skey[TE_ERASER_MAX_WORDS];
    __shared__ int sword[TE_ERASER_MAX_WORDS];
    __shared__ int sscan[TE_ERASER_MAX_WORDS];                     // positive | group end << 16, then inclusive prefix sums
    __shared__ long long gtp[TE_ERASER_MAX_WORDS + 1], gfp[TE_ERASER_MAX_WORDS + 1];   // cumulative counts per tie group
    __shared__ double sred[2][kWarps];
    __shared__ long long sroc[kWarps];
    __shared__ int sG, sbad;
    const int b = blockIdx.x;
    const int w0 = word_off[b], W = word_off[b + 1] - w0;
    const int s0 = span_off[b], S = span_off[b + 1] - s0;
    const float* s = word_scores + w0;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) sbad = 0;
    __syncthreads();
    rank_scores([&](int w) {
        const float v = s[w];
        if (!(v >= 0.f)) sbad = 1;                                 // NaN or negative: no soft scores
        return v;
    }, W, skey, sword);
    const auto group_end = [&](int r) {
        return r == W - 1 || (unsigned)(skey[sword[r]] >> 32) != (unsigned)(skey[sword[r + 1]] >> 32);
    };
    for (int r = threadIdx.x; r < W; r += kThreads) {
        const int w = sword[r];
        int pos = 0;
        for (int j = 0; j < S; ++j) {
            const int2 t = spans[s0 + j];
            pos |= t.x <= w && w < t.y;
        }
        sscan[r] = pos | (int)group_end(r) << 16;
    }
    __syncthreads();
    if (warp == 0) {                                               // lane l owns ranks [l*C, (l+1)*C)
        const int C = (W + 31) / 32;
        const int r0 = lane * C, r1 = min(W, r0 + C);
        int sum = 0;
        for (int r = r0; r < r1; ++r) sum += sscan[r];
        int incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += u;
        }
        int run = incl - sum;
        for (int r = r0; r < r1; ++r) { run += sscan[r]; sscan[r] = run; }
    }
    __syncthreads();
    for (int r = threadIdx.x; r < W; r += kThreads) {
        if (!group_end(r)) continue;
        const int g = (sscan[r] >> 16) - 1, tp = sscan[r] & 0xffff;
        gtp[g] = tp;
        gfp[g] = r + 1 - tp;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int G = W ? sscan[W - 1] >> 16 : 0;
        const long long tp = G ? gtp[G - 1] : 0, fp = G ? gfp[G - 1] : 0;
        if (tail[b].x + tail[b].y > 0) {
            if (!(G && (unsigned)(skey[sword[W - 1]] >> 32) == ~order_key(0.f))) ++G;
            gtp[G - 1] = tp + tail[b].x;
            gfp[G - 1] = fp + tail[b].y;
        }
        sG = G;
    }
    __syncthreads();
    const int G = sG;                                              // >= 1: W + tail >= 1 is checked on the host
    const long long P = gtp[G - 1], N = gfp[G - 1];
    // precision_recall_curve's points (recall tp / P, 1 without positives; precision tp / (tp + fp)) after the point
    // (0, 1): auc(recall, precision) is their trapezoid area, average_precision_score the step area; roc_curve's points
    // (fp / N, tp / P) after (0, 0): roc_auc_score's trapezoid area, summed in integers
    double pr = 0.0, ap = 0.0;
    long long roc = 0;
    for (int g = threadIdx.x; g < G; g += kThreads) {
        const long long tp = gtp[g], fp = gfp[g];
        const long long tq = g ? gtp[g - 1] : 0, fq = g ? gfp[g - 1] : 0;
        const double p = (double)tp / (double)(tp + fp), q = g ? (double)tq / (double)(tq + fq) : 1.0;
        const double r = P ? (double)tp / (double)P : 1.0, rq = g ? (P ? (double)tq / (double)P : 1.0) : 0.0;
        pr += (r - rq) * (p + q) / 2.0;
        ap += (r - rq) * p;
        roc += (fp - fq) * (tp + tq);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        pr += __shfl_down_sync(0xffffffffu, pr, o);
        ap += __shfl_down_sync(0xffffffffu, ap, o);
        roc += __shfl_down_sync(0xffffffffu, roc, o);
    }
    if (lane == 0) {
        sred[0][warp] = pr;
        sred[1][warp] = ap;
        sroc[warp] = roc;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        pr = ap = 0.0;
        roc = 0;
        for (int u = 0; u < kWarps; ++u) {
            pr += sred[0][u];
            ap += sred[1][u];
            roc += sroc[u];
        }
        const bool single = P == 0 || N == 0;
        const double nan = __longlong_as_double(0x7ff8000000000000LL);
        scores[3 * b] = sbad ? nan : pr;
        scores[3 * b + 1] = sbad ? nan : ap;
        scores[3 * b + 2] = sbad || single ? nan : (double)roc / (2.0 * (double)P * (double)N);
        flags[2 * b] = single;
        flags[2 * b + 1] = sbad;
    }
}

constexpr int kLatexThreads = 256;

// generate()'s weights of row b: a = the first L entries (clamped at 0 when clamp; NaN stays); mn / mx = min / max of a,
// NaN when any entry is NaN, as torch.min / torch.max; w = 0 for a constant row (mx == mn, false for NaN), else
// (100 * (a - mn)) / (mx - mn) with one fp32 rounding per operation; w < 1 -> 0; zeros past L.
__global__ void __launch_bounds__(kLatexThreads) latex_kernel(const float* __restrict__ maps, int seq,
                                                              const int* __restrict__ lengths, int clamp,
                                                              float* __restrict__ out) {
    __shared__ float smn[kLatexThreads / 32], smx[kLatexThreads / 32];
    __shared__ int snan[kLatexThreads / 32];
    const int b = blockIdx.x;
    const int L = min(max(lengths[b], 0), seq);
    const float* row = maps + (long long)b * seq;
    float* o = out + (long long)b * seq;
    const float inf = __int_as_float(0x7f800000);
    float mn = inf, mx = -inf;
    int nan = 0;
    for (int p = threadIdx.x; p < L; p += kLatexThreads) {
        float v = row[p];
        if (clamp && v < 0.f) v = 0.f;
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
    for (int u = 1; u < kLatexThreads / 32; ++u) {
        mn = fminf(mn, smn[u]);
        mx = fmaxf(mx, smx[u]);
        nan |= snan[u];
    }
    if (nan) mn = mx = __int_as_float(0x7fc00000);
    const float range = __fsub_rn(mx, mn);
    for (int p = threadIdx.x; p < seq; p += kLatexThreads) {
        float w = 0.f;
        if (p < L && !(mx == mn)) {
            float v = row[p];
            if (clamp && v < 0.f) v = 0.f;
            w = __fdiv_rn(__fmul_rn(100.f, __fsub_rn(v, mn)), range);
            if (w < 1.f) w = 0.f;
        }
        o[p] = w;
    }
}

}  // namespace

#define ST(s) reinterpret_cast<cudaStream_t>(s)
#define REQ(c, msg) do { if (!(c)) { te_set_last_error(msg); return TE_ERR_ARG; } } while (0)

namespace {
long long up256(long long n) { return (n + 255) / 256 * 256; }
}

extern "C" long long te_eraser_workspace_bytes(int batch, long long words, long long spans) {
    if (batch <= 0 || words < 0 || spans < 0 || words > 0x7fffffffLL || spans > 0x7fffffffLL) return TE_ERR_ARG;
    return 2 * up256(4LL * (batch + 1)) + up256(8 * words) + up256(8 * spans);
}

extern "C" int te_eraser_rationales(const float* maps, int batch, int seq, const int* word_offsets, const int* piece_ranges,
                                    const int* span_offsets, const int* spans, const int* ks, int nk, const double* thresholds,
                                    int nthr, float* word_scores, int* order, int* counts, void* workspace,
                                    long long workspace_bytes, void* stream) {
    REQ(maps && word_offsets && span_offsets && ks && counts, "te_eraser_rationales: null argument");
    REQ(batch > 0 && batch <= 65535 && seq > 0, "te_eraser_rationales: batch must lie in 1..65535 and seq be positive");
    REQ(nk > 0 && nk <= TE_ERASER_MAX_KS, "te_eraser_rationales: nk outside 1..TE_ERASER_MAX_KS");
    REQ(nthr >= 0 && nthr <= TE_ERASER_MAX_THRESHOLDS, "te_eraser_rationales: nthr outside 0..TE_ERASER_MAX_THRESHOLDS");
    REQ(nthr == 0 || thresholds, "te_eraser_rationales: null thresholds");
    EraserParams prm;
    prm.nk = nk;
    prm.nthr = nthr;
    for (int i = 0; i < nk; ++i) {
        REQ(ks[i] >= 0 && ks[i] <= (1 << 20), "te_eraser_rationales: every k must lie in [0, 2^20]");
        REQ(i == 0 || ks[i] >= ks[i - 1], "te_eraser_rationales: ks must be non-decreasing");
        prm.k[i] = ks[i];
    }
    prm.kmax = ks[nk - 1];
    REQ(prm.kmax == 0 || order, "te_eraser_rationales: null order");
    for (int t = 0; t < nthr; ++t) {
        REQ(!(thresholds[t] != thresholds[t]), "te_eraser_rationales: a threshold is NaN");
        prm.thr[t] = thresholds[t];
    }
    REQ(word_offsets[0] == 0 && span_offsets[0] == 0, "te_eraser_rationales: offsets must start at 0");
    for (int b = 0; b < batch; ++b) {
        const long long nw = (long long)word_offsets[b + 1] - word_offsets[b];
        REQ(nw >= 0 && nw <= TE_ERASER_MAX_WORDS, "te_eraser_rationales: a document holds 0..TE_ERASER_MAX_WORDS words");
        REQ(span_offsets[b + 1] >= span_offsets[b], "te_eraser_rationales: span offsets must be non-decreasing");
    }
    const long long words = word_offsets[batch], nspans = span_offsets[batch];
    REQ(words == 0 || (piece_ranges && word_scores), "te_eraser_rationales: null piece ranges or word scores");
    REQ(nspans == 0 || spans, "te_eraser_rationales: null spans");
    for (long long w = 0; w < words; ++w)
        REQ(piece_ranges[2 * w] >= 0 && piece_ranges[2 * w] <= piece_ranges[2 * w + 1] && piece_ranges[2 * w + 1] < seq,
            "te_eraser_rationales: every piece range [first, last] must satisfy 0 <= first <= last < seq");
    for (long long j = 0; j < nspans; ++j)
        REQ(spans[2 * j] >= 0 && spans[2 * j] <= spans[2 * j + 1],
            "te_eraser_rationales: every truth span (start, end) must satisfy 0 <= start <= end");
    REQ(workspace && (((uintptr_t)workspace) & 255u) == 0, "te_eraser_rationales: workspace null or not 256-byte aligned");
    const long long ws = te_eraser_workspace_bytes(batch, words, nspans);
    if (ws > workspace_bytes) {
        te_set_last_error("te_eraser_rationales: workspace too small");
        return TE_ERR_WORKSPACE;
    }
    char* p = static_cast<char*>(workspace);
    int* d_woff = reinterpret_cast<int*>(p);
    int* d_soff = reinterpret_cast<int*>(p + up256(4LL * (batch + 1)));
    int2* d_ranges = reinterpret_cast<int2*>(p + 2 * up256(4LL * (batch + 1)));
    int2* d_spans = reinterpret_cast<int2*>(p + 2 * up256(4LL * (batch + 1)) + up256(8 * words));
    cudaStream_t st = ST(stream);
    if (cudaMemcpyAsync(d_woff, word_offsets, 4 * (size_t)(batch + 1), cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(d_soff, span_offsets, 4 * (size_t)(batch + 1), cudaMemcpyHostToDevice, st) != cudaSuccess ||
        (words && cudaMemcpyAsync(d_ranges, piece_ranges, 8 * (size_t)words, cudaMemcpyHostToDevice, st) != cudaSuccess) ||
        (nspans && cudaMemcpyAsync(d_spans, spans, 8 * (size_t)nspans, cudaMemcpyHostToDevice, st) != cudaSuccess)) {
        te_set_last_error("te_eraser_rationales: copy of the host arrays failed");
        return TE_ERR_CUDA;
    }
    eraser_kernel<<<batch, kThreads, 0, st>>>(maps, seq, d_woff, d_ranges, d_soff, d_spans, prm, word_scores, order, counts);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}

extern "C" long long te_eraser_reduce_workspace_bytes(int batch, long long words, int selections) {
    if (batch <= 0 || words < 0 || words > 0x7fffffffLL || selections <= 0) return TE_ERR_ARG;
    return up256(4LL * (batch + 1)) + up256(8 * words) + up256(4LL * batch) + up256(4LL * batch * selections);
}

extern "C" int te_eraser_reduce_inputs(const float* maps, const long long* input_ids, int batch, int seq, const int* lengths,
                                       const int* word_offsets, const int* piece_ranges, const int* n_select, int selections,
                                       long long* out_ids, int* out_len, void* workspace, long long workspace_bytes,
                                       void* stream) {
    REQ(maps && input_ids && lengths && word_offsets && n_select && out_ids && out_len,
        "te_eraser_reduce_inputs: null argument");
    REQ(batch > 0 && batch <= 65535, "te_eraser_reduce_inputs: batch must lie in 1..65535");
    REQ(seq >= 2 && seq <= TE_ERASER_MAX_SEQ, "te_eraser_reduce_inputs: seq outside 2..TE_ERASER_MAX_SEQ");
    REQ(selections > 0 && selections <= TE_ERASER_MAX_SELECTIONS,
        "te_eraser_reduce_inputs: selections outside 1..TE_ERASER_MAX_SELECTIONS");
    REQ(word_offsets[0] == 0, "te_eraser_reduce_inputs: word offsets must start at 0");
    for (int b = 0; b < batch; ++b) {
        const long long nw = (long long)word_offsets[b + 1] - word_offsets[b];
        REQ(nw >= 0 && nw <= TE_ERASER_MAX_WORDS, "te_eraser_reduce_inputs: a document holds 0..TE_ERASER_MAX_WORDS words");
        REQ(lengths[b] >= 2 && lengths[b] <= seq, "te_eraser_reduce_inputs: every length must lie in 2..seq");
        for (long long w = word_offsets[b]; w < word_offsets[b + 1]; ++w)
            REQ(piece_ranges[2 * w] >= 1 && piece_ranges[2 * w] <= piece_ranges[2 * w + 1] &&
                piece_ranges[2 * w + 1] <= lengths[b] - 2,
                "te_eraser_reduce_inputs: every piece range [first, last] must satisfy 1 <= first <= last <= length - 2");
        for (int j = 0; j < selections; ++j)
            REQ(n_select[(long long)b * selections + j] >= 0 && n_select[(long long)b * selections + j] <= nw,
                "te_eraser_reduce_inputs: every selection size must lie in 0..W of its document");
    }
    const long long words = word_offsets[batch];
    REQ(words == 0 || piece_ranges, "te_eraser_reduce_inputs: null piece ranges");
    REQ(workspace && (((uintptr_t)workspace) & 255u) == 0, "te_eraser_reduce_inputs: workspace null or not 256-byte aligned");
    if (te_eraser_reduce_workspace_bytes(batch, words, selections) > workspace_bytes) {
        te_set_last_error("te_eraser_reduce_inputs: workspace too small");
        return TE_ERR_WORKSPACE;
    }
    char* p = static_cast<char*>(workspace);
    int* d_woff = reinterpret_cast<int*>(p);
    p += up256(4LL * (batch + 1));
    int2* d_ranges = reinterpret_cast<int2*>(p);
    p += up256(8 * words);
    int* d_lens = reinterpret_cast<int*>(p);
    p += up256(4LL * batch);
    int* d_nsel = reinterpret_cast<int*>(p);
    cudaStream_t st = ST(stream);
    if (cudaMemcpyAsync(d_woff, word_offsets, 4 * (size_t)(batch + 1), cudaMemcpyHostToDevice, st) != cudaSuccess ||
        (words && cudaMemcpyAsync(d_ranges, piece_ranges, 8 * (size_t)words, cudaMemcpyHostToDevice, st) != cudaSuccess) ||
        cudaMemcpyAsync(d_lens, lengths, 4 * (size_t)batch, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(d_nsel, n_select, 4 * (size_t)batch * selections, cudaMemcpyHostToDevice, st) != cudaSuccess) {
        te_set_last_error("te_eraser_reduce_inputs: copy of the host arrays failed");
        return TE_ERR_CUDA;
    }
    reduce_kernel<<<batch, kThreads, 4 * (size_t)seq, st>>>(maps, input_ids, seq, d_lens, d_woff, d_ranges, d_nsel,
                                                             selections, out_ids, out_len);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}

extern "C" long long te_eraser_soft_workspace_bytes(int batch, long long spans) {
    if (batch <= 0 || spans < 0 || spans > 0x7fffffffLL) return TE_ERR_ARG;
    return 2 * up256(4LL * (batch + 1)) + up256(8 * spans) + up256(8LL * batch);
}

extern "C" int te_eraser_soft_scores(const float* word_scores, int batch, const int* word_offsets, const int* span_offsets,
                                     const int* spans, const int* tail_counts, double* scores, int* flags, void* workspace,
                                     long long workspace_bytes, void* stream) {
    REQ(word_offsets && span_offsets && tail_counts && scores && flags, "te_eraser_soft_scores: null argument");
    REQ(batch > 0 && batch <= 65535, "te_eraser_soft_scores: batch must lie in 1..65535");
    REQ(word_offsets[0] == 0 && span_offsets[0] == 0, "te_eraser_soft_scores: offsets must start at 0");
    for (int b = 0; b < batch; ++b) {
        const long long nw = (long long)word_offsets[b + 1] - word_offsets[b];
        REQ(nw >= 0 && nw <= TE_ERASER_MAX_WORDS, "te_eraser_soft_scores: a document holds 0..TE_ERASER_MAX_WORDS words");
        REQ(span_offsets[b + 1] >= span_offsets[b], "te_eraser_soft_scores: span offsets must be non-decreasing");
        const long long tp = tail_counts[2 * b], tn = tail_counts[2 * b + 1];
        REQ(tp >= 0 && tn >= 0 && tp + tn <= (1 << 30), "te_eraser_soft_scores: tail counts must lie in 0..2^30");
        REQ(nw + tp + tn >= 1, "te_eraser_soft_scores: a document needs a word or a tail word");
    }
    const long long words = word_offsets[batch], nspans = span_offsets[batch];
    REQ(words == 0 || word_scores, "te_eraser_soft_scores: null word scores");
    REQ(nspans == 0 || spans, "te_eraser_soft_scores: null spans");
    for (long long j = 0; j < nspans; ++j)
        REQ(spans[2 * j] >= 0 && spans[2 * j] <= spans[2 * j + 1],
            "te_eraser_soft_scores: every truth span (start, end) must satisfy 0 <= start <= end");
    REQ(workspace && (((uintptr_t)workspace) & 255u) == 0, "te_eraser_soft_scores: workspace null or not 256-byte aligned");
    if (te_eraser_soft_workspace_bytes(batch, nspans) > workspace_bytes) {
        te_set_last_error("te_eraser_soft_scores: workspace too small");
        return TE_ERR_WORKSPACE;
    }
    char* p = static_cast<char*>(workspace);
    int* d_woff = reinterpret_cast<int*>(p);
    p += up256(4LL * (batch + 1));
    int* d_soff = reinterpret_cast<int*>(p);
    p += up256(4LL * (batch + 1));
    int2* d_spans = reinterpret_cast<int2*>(p);
    p += up256(8 * nspans);
    int2* d_tail = reinterpret_cast<int2*>(p);
    cudaStream_t st = ST(stream);
    if (cudaMemcpyAsync(d_woff, word_offsets, 4 * (size_t)(batch + 1), cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(d_soff, span_offsets, 4 * (size_t)(batch + 1), cudaMemcpyHostToDevice, st) != cudaSuccess ||
        (nspans && cudaMemcpyAsync(d_spans, spans, 8 * (size_t)nspans, cudaMemcpyHostToDevice, st) != cudaSuccess) ||
        cudaMemcpyAsync(d_tail, tail_counts, 8 * (size_t)batch, cudaMemcpyHostToDevice, st) != cudaSuccess) {
        te_set_last_error("te_eraser_soft_scores: copy of the host arrays failed");
        return TE_ERR_CUDA;
    }
    soft_kernel<<<batch, kThreads, 0, st>>>(word_scores, d_woff, d_soff, d_spans, d_tail, scores, flags);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}

extern "C" int te_eraser_latex_weights(const float* maps, int batch, int seq, const int* lengths, int clamp, float* out,
                                       void* stream) {
    REQ(maps && lengths && out, "te_eraser_latex_weights: null argument");
    REQ(batch > 0 && batch <= 65535 && seq > 0, "te_eraser_latex_weights: batch must lie in 1..65535 and seq be positive");
    REQ(clamp == 0 || clamp == 1, "te_eraser_latex_weights: clamp must be 0 or 1");
    latex_kernel<<<batch, kLatexThreads, 0, ST(stream)>>>(maps, seq, lengths, clamp, out);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
