// ERASER rationale evaluation (BERT_rationale_benchmark/models/pipeline/bert_pipeline.py:96-138,547-582; metrics.py:111-215):
//   * eraser_kernel: one block per document.  Word scores are the max over each word's word-piece range of the clamped map
//     (NaN propagates); the words are ranked NaN first, then by descending score, then by ascending word index (the order
//     key of te_perturb_images); the first kmax ranks are written out, and per k the counts of the predicted words that
//     metrics.py's hard-rationale scores need come from prefix sums along that order.
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

    // word scores and ranking keys
    for (int w = threadIdx.x; w < W; w += kThreads) {
        const int2 r = ranges[w0 + w];
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
        word_scores[w0 + w] = s;
        skey[w] = ((unsigned long long)(~order_key(s)) << 32) | (unsigned)w;
    }
    __syncthreads();
    // rank = number of smaller keys (all keys are distinct)
    for (int w = threadIdx.x; w < W; w += kThreads) {
        const unsigned long long k = skey[w];
        int rank = 0;
        for (int u = 0; u < W; ++u) rank += skey[u] < k;
        sword[rank] = w;
    }
    __syncthreads();
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
