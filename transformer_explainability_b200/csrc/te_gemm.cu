// FP32 SIMT strided-batched GEMM (see te_gemm.cuh).  256 threads, (16*TM)x(16*TM)x16 tiles,
// TM x TM register micro-tile per thread, register-prefetched double-buffered shared memory.
#include "te_gemm.cuh"

namespace {

constexpr int BK = 16;

template <int TM, int LAY>
__device__ __forceinline__ float4 load_tile4(const float* __restrict__ base, int ld, int R, int K,
                                             int mn0, int k0, int f, int vec) {
    constexpr int BM = 16 * TM;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (LAY == TE_L_K) {
        const int row = f >> 2, kq = f & 3;
        const int r = mn0 + row, k = k0 + kq * 4;
        if (r < R && k < K) {
            const float* ptr = base + (long long)r * ld + k;
            if (vec && k + 3 < K) {
                v = __ldg(reinterpret_cast<const float4*>(ptr));
            } else {
                v.x = __ldg(ptr);
                if (k + 1 < K) v.y = __ldg(ptr + 1);
                if (k + 2 < K) v.z = __ldg(ptr + 2);
                if (k + 3 < K) v.w = __ldg(ptr + 3);
            }
        }
    } else {
        const int kk = f / (BM / 4), c4 = f % (BM / 4);
        const int k = k0 + kk, r = mn0 + c4 * 4;
        if (k < K && r < R) {
            const float* ptr = base + (long long)k * ld + r;
            if (vec && r + 3 < R) {
                v = __ldg(reinterpret_cast<const float4*>(ptr));
            } else {
                v.x = __ldg(ptr);
                if (r + 1 < R) v.y = __ldg(ptr + 1);
                if (r + 2 < R) v.z = __ldg(ptr + 2);
                if (r + 3 < R) v.w = __ldg(ptr + 3);
            }
        }
    }
    return v;
}

template <int TM, int LAY>
__device__ __forceinline__ void store_tile4(float (*S)[16 * TM + 4], int f, float4 v) {
    constexpr int BM = 16 * TM;
    if (LAY == TE_L_K) {
        const int row = f >> 2, kq = f & 3;
        S[kq * 4 + 0][row] = v.x;
        S[kq * 4 + 1][row] = v.y;
        S[kq * 4 + 2][row] = v.z;
        S[kq * 4 + 3][row] = v.w;
    } else {
        const int kk = f / (BM / 4), c4 = f % (BM / 4);
        *reinterpret_cast<float4*>(&S[kk][c4 * 4]) = v;
    }
}

__device__ __forceinline__ float4 clamp4(float4 v, int mode) {   // 1: max(.,0)  2: min(.,0)
    if (mode == 1) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
    else if (mode == 2) { v.x = fminf(v.x, 0.f); v.y = fminf(v.y, 0.f); v.z = fminf(v.z, 0.f); v.w = fminf(v.w, 0.f); }
    return v;
}

template <int EPI>
__device__ __forceinline__ void epilogue4(const TeGemm& p, float* __restrict__ C, float* __restrict__ C2,
                                          const float* __restrict__ E0, int row, int col, const float* acc) {
    if (row >= p.M || col >= p.N) return;
    const int nv = min(4, p.N - col);
    float e[4] = {0.f, 0.f, 0.f, 0.f}, c[4] = {0.f, 0.f, 0.f, 0.f}, o[4], o2[4] = {0.f, 0.f, 0.f, 0.f};
    constexpr bool needE = (EPI == TE_EPI_BIAS_ADD || EPI == TE_EPI_GELU_BWD || EPI == TE_EPI_SD || EPI == TE_EPI_SD_SCALED ||
                            EPI == TE_EPI_MUL || EPI == TE_EPI_MULPOS || EPI == TE_EPI_MULNEG_ACC || EPI == TE_EPI_MULPOS_ACC ||
                            EPI == TE_EPI_QUICK_GELU_BWD);
    constexpr bool needC = (EPI == TE_EPI_MULNEG_ACC || EPI == TE_EPI_MULPOS_ACC || EPI == TE_EPI_ACCUM);
    constexpr bool hasC2 = (EPI == TE_EPI_BIAS_GELU || EPI == TE_EPI_BIAS_ADD || EPI == TE_EPI_BIAS_QUICK_GELU);
    const long long co = (long long)row * p.ldc + col;
    if (needE) {
        const float* ep = E0 + (long long)row * p.lde0 + col;
        if (nv == 4 && p.vecE) { float4 t = *reinterpret_cast<const float4*>(ep); e[0] = t.x; e[1] = t.y; e[2] = t.z; e[3] = t.w; }
        else {
#pragma unroll
            for (int j = 0; j < 4; ++j) if (j < nv) e[j] = ep[j];
        }
    }
    if (needC) {
        if (nv == 4 && p.vecC) { float4 t = *reinterpret_cast<const float4*>(C + co); c[0] = t.x; c[1] = t.y; c[2] = t.z; c[3] = t.w; }
        else {
#pragma unroll
            for (int j = 0; j < 4; ++j) if (j < nv) c[j] = C[co + j];
        }
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const float a = acc[j];
        float bj = 0.f;
        if (EPI == TE_EPI_BIAS || EPI == TE_EPI_BIAS_GELU || EPI == TE_EPI_BIAS_ADD || EPI == TE_EPI_BIAS_QUICK_GELU)
            bj = (p.bias != nullptr && j < nv) ? __ldg(p.bias + col + j) : 0.f;
        if (EPI == TE_EPI_STORE) o[j] = p.alpha * a;
        else if (EPI == TE_EPI_BIAS) o[j] = a + bj;
        else if (EPI == TE_EPI_BIAS_GELU) { o[j] = a + bj; o2[j] = te_gelu(o[j]); }
        else if (EPI == TE_EPI_BIAS_ADD) { o[j] = a + bj; o2[j] = e[j] + o[j]; }
        else if (EPI == TE_EPI_GELU_BWD) o[j] = a * te_gelu_grad(e[j]);
        else if (EPI == TE_EPI_BIAS_QUICK_GELU) { o[j] = a + bj; o2[j] = te_quick_gelu(o[j]); }
        else if (EPI == TE_EPI_QUICK_GELU_BWD) o[j] = a * te_quick_gelu_grad(e[j]);
        else if (EPI == TE_EPI_SD) o[j] = te_sd(e[j], p.alpha * a);
        else if (EPI == TE_EPI_SD_SCALED) o[j] = p.scale * te_sd(e[j], p.alpha * a);
        else if (EPI == TE_EPI_MUL) o[j] = p.alpha * a * e[j];
        else if (EPI == TE_EPI_MULPOS) o[j] = fmaxf(e[j], 0.f) * a;
        else if (EPI == TE_EPI_MULNEG_ACC) o[j] = c[j] + fminf(e[j], 0.f) * a;
        else if (EPI == TE_EPI_MULPOS_ACC) o[j] = c[j] + fmaxf(e[j], 0.f) * a;
        else o[j] = c[j] + p.alpha * a;   // ACCUM
    }
    if (nv == 4 && p.vecC) *reinterpret_cast<float4*>(C + co) = make_float4(o[0], o[1], o[2], o[3]);
    else {
#pragma unroll
        for (int j = 0; j < 4; ++j) if (j < nv) C[co + j] = o[j];
    }
    if (hasC2) {
        const long long c2o = (long long)row * p.ldc2 + col;
        if (nv == 4 && p.vecC2) *reinterpret_cast<float4*>(C2 + c2o) = make_float4(o2[0], o2[1], o2[2], o2[3]);
        else {
#pragma unroll
            for (int j = 0; j < 4; ++j) if (j < nv) C2[c2o + j] = o2[j];
        }
    }
}

template <int TM, int ALAY, int BLAY, int XF, int EPI>
__global__ void __launch_bounds__(256, (TM == 8) ? 2 : 3) te_gemm_kernel(const TeGemm p) {
    constexpr int BM = 16 * TM, BN = 16 * TM;
    constexpr int NLD = TM / 4;             // float4 loads per thread per operand per k-tile
    __shared__ __align__(16) float As[2][BK][BM + 4];
    __shared__ __align__(16) float Bs[2][BK][BN + 4];

    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    const int z = blockIdx.z;
    const int b1 = z / p.nb2, b2 = z % p.nb2;
    const float* __restrict__ A = p.A + b1 * p.sA1 + b2 * p.sA2;
    const float* __restrict__ B = p.B + b1 * p.sB1 + b2 * p.sB2;
    float* __restrict__ C = p.C + b1 * p.sC1 + b2 * p.sC2;
    float* __restrict__ C2 = p.C2 ? p.C2 + b1 * p.sD1 + b2 * p.sD2 : nullptr;
    const float* __restrict__ E0 = p.E0 ? p.E0 + b1 * p.sE1 + b2 * p.sE2 : nullptr;

    const int T = (p.K + BK - 1) / BK;
    constexpr bool KCAT = (XF == TE_XF_AB_POSNEG || XF == TE_XF_AB_NEGPOS);   // K-concatenated: two phases over K
    const int ntiles = KCAT ? 2 * T : T;

    float acc[TM][TM];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TM; ++j) acc[i][j] = 0.f;

    float4 ra[NLD], rb[NLD];

    auto gload = [&](int t) {
        int k0 = t * BK, amode = 0, bmode = 0;
        if (KCAT) {
            const int ph = (t >= T) ? 1 : 0;
            k0 = (t - ph * T) * BK;
            amode = ph + 1;
            bmode = (XF == TE_XF_AB_POSNEG) ? ph + 1 : 2 - ph;    // NEGPOS: x+ with W-, then x- with W+
        } else if (XF == TE_XF_B_POS) bmode = 1;
        else if (XF == TE_XF_B_NEG) bmode = 2;
        else if (XF == TE_XF_AB_POS) amode = bmode = 1;         // x+ W+^T  (layers_lrp Linear rule: separate denominators)
        else if (XF == TE_XF_AB_NEG) amode = bmode = 2;         // x- W-^T
        else if (XF == TE_XF_A_POS_B_NEG) { amode = 1; bmode = 2; }   // x+ W-^T  (layers_lrp inhibitor half)
        else if (XF == TE_XF_A_NEG_B_POS) { amode = 2; bmode = 1; }   // x- W+^T
#pragma unroll
        for (int i = 0; i < NLD; ++i) {
            ra[i] = clamp4(load_tile4<TM, ALAY>(A, p.lda, p.M, p.K, m0, k0, tid + i * 256, p.vecA), amode);
            rb[i] = clamp4(load_tile4<TM, BLAY>(B, p.ldb, p.N, p.K, n0, k0, tid + i * 256, p.vecB), bmode);
        }
    };
    auto sstore = [&](int buf) {
#pragma unroll
        for (int i = 0; i < NLD; ++i) {
            store_tile4<TM, ALAY>(As[buf], tid + i * 256, ra[i]);
            store_tile4<TM, BLAY>(Bs[buf], tid + i * 256, rb[i]);
        }
    };

    gload(0);
    sstore(0);
    __syncthreads();

    for (int t = 0; t < ntiles; ++t) {
        const int cur = t & 1;
        if (t + 1 < ntiles) gload(t + 1);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float a[TM], b[TM];
#pragma unroll
            for (int g = 0; g < TM / 4; ++g) {
                const float4 va = *reinterpret_cast<const float4*>(&As[cur][k][g * 64 + ty * 4]);
                const float4 vb = *reinterpret_cast<const float4*>(&Bs[cur][k][g * 64 + tx * 4]);
                a[g * 4 + 0] = va.x; a[g * 4 + 1] = va.y; a[g * 4 + 2] = va.z; a[g * 4 + 3] = va.w;
                b[g * 4 + 0] = vb.x; b[g * 4 + 1] = vb.y; b[g * 4 + 2] = vb.z; b[g * 4 + 3] = vb.w;
            }
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TM; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (t + 1 < ntiles) {
            sstore(cur ^ 1);
            __syncthreads();
        }
    }

#pragma unroll
    for (int gr = 0; gr < TM / 4; ++gr)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int row = m0 + gr * 64 + ty * 4 + i;
#pragma unroll
            for (int gc = 0; gc < TM / 4; ++gc) {
                const int col = n0 + gc * 64 + tx * 4;
                epilogue4<EPI>(p, C, C2, E0, row, col, &acc[gr * 4 + i][gc * 4]);
            }
        }
}

inline int aligned16(const void* ptr) { return ((uintptr_t)ptr & 15u) == 0; }

template <int TM, int ALAY, int BLAY, int XF, int EPI>
int launch_one(const TeGemm& p, cudaStream_t st) {
    constexpr int BM = 16 * TM;
    dim3 grid(te_cdiv(p.N, BM), te_cdiv(p.M, BM), p.nb1 * p.nb2);
    if (grid.y > 65535 || grid.z > 65535) { te_set_last_error("te_gemm: grid too large"); return TE_ERR_ARG; }
    te_gemm_kernel<TM, ALAY, BLAY, XF, EPI><<<grid, 256, 0, st>>>(p);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}

template <int ALAY, int BLAY, int XF, int EPI>
int launch_tm(const TeGemm& p, cudaStream_t st) {
    // small tiles when the problem would leave most of a 128x128 tile empty or the grid tiny
    const long long ctas128 = (long long)te_cdiv(p.M, 128) * te_cdiv(p.N, 128) * p.nb1 * p.nb2;
    const bool small = (p.M <= 64 || p.N <= 64 || ctas128 < 132 ||
                        (p.M < 256 && (p.M % 128) != 0 && (p.M % 128) <= 80) );
    if (small) return launch_one<4, ALAY, BLAY, XF, EPI>(p, st);
    return launch_one<8, ALAY, BLAY, XF, EPI>(p, st);
}

}  // namespace

#define TE_CASE(AL, BL, X, E) \
    if (alay == AL && blay == BL && xf == X && epi == E) return launch_tm<AL, BL, X, E>(p, st);
// small tiles only: at 128 x 128 these variants spill under the two-CTA register cap
#define TE_CASE4(AL, BL, X, E) \
    if (alay == AL && blay == BL && xf == X && epi == E) return launch_one<4, AL, BL, X, E>(p, st);

int te_gemm_launch(TeGemm p, int alay, int blay, int xf, int epi, cudaStream_t st) {
    if (p.M <= 0 || p.N <= 0 || p.K <= 0 || p.nb1 <= 0 || p.nb2 <= 0) return TE_OK;
    auto vec = [](const void* ptr, int ld, long long s1, long long s2) {
        return (ptr == nullptr || (aligned16(ptr) && (ld % 4) == 0 && (s1 % 4) == 0 && (s2 % 4) == 0)) ? 1 : 0;
    };
    p.vecA = vec(p.A, p.lda, p.sA1, p.sA2);
    p.vecB = vec(p.B, p.ldb, p.sB1, p.sB2);
    p.vecC = vec(p.C, p.ldc, p.sC1, p.sC2);
    p.vecC2 = vec(p.C2, p.ldc2, p.sD1, p.sD2);
    p.vecE = vec(p.E0, p.lde0, p.sE1, p.sE2);
    // forward
    TE_CASE(TE_L_K, TE_L_K, TE_XF_NONE, TE_EPI_BIAS)
    TE_CASE(TE_L_K, TE_L_K, TE_XF_NONE, TE_EPI_BIAS_ADD)
    TE_CASE(TE_L_K, TE_L_K, TE_XF_NONE, TE_EPI_BIAS_GELU)
    TE_CASE(TE_L_K, TE_L_K, TE_XF_NONE, TE_EPI_STORE)
    TE_CASE(TE_L_K, TE_L_MN, TE_XF_NONE, TE_EPI_STORE)
    // backward
    TE_CASE(TE_L_K, TE_L_MN, TE_XF_NONE, TE_EPI_GELU_BWD)
    TE_CASE(TE_L_MN, TE_L_MN, TE_XF_NONE, TE_EPI_STORE)
    // QuickGELU (CLIP) forward / backward epilogues: small tiles only, spill-free (the fp32 checker of the tensor-core families)
    TE_CASE4(TE_L_K, TE_L_K, TE_XF_NONE, TE_EPI_BIAS_QUICK_GELU)
    TE_CASE4(TE_L_K, TE_L_MN, TE_XF_NONE, TE_EPI_QUICK_GELU_BWD)
    // relprop
    TE_CASE(TE_L_K, TE_L_K, TE_XF_AB_POSNEG, TE_EPI_SD)
    TE_CASE(TE_L_K, TE_L_K, TE_XF_AB_POS, TE_EPI_SD)
    TE_CASE(TE_L_K, TE_L_K, TE_XF_AB_NEG, TE_EPI_SD)
    TE_CASE(TE_L_K, TE_L_MN, TE_XF_B_POS, TE_EPI_MULPOS)
    TE_CASE(TE_L_K, TE_L_MN, TE_XF_B_NEG, TE_EPI_MULNEG_ACC)
    // relprop, alpha-beta rule (alpha != 1): S scaled by alpha / -beta, the inhibitor half with the weight signs swapped
    TE_CASE4(TE_L_K, TE_L_K, TE_XF_AB_POSNEG, TE_EPI_SD_SCALED)
    TE_CASE4(TE_L_K, TE_L_K, TE_XF_AB_NEGPOS, TE_EPI_SD_SCALED)
    TE_CASE4(TE_L_K, TE_L_K, TE_XF_AB_POS, TE_EPI_SD_SCALED)
    TE_CASE4(TE_L_K, TE_L_K, TE_XF_AB_NEG, TE_EPI_SD_SCALED)
    TE_CASE4(TE_L_K, TE_L_K, TE_XF_A_POS_B_NEG, TE_EPI_SD_SCALED)
    TE_CASE4(TE_L_K, TE_L_K, TE_XF_A_NEG_B_POS, TE_EPI_SD_SCALED)
    TE_CASE4(TE_L_K, TE_L_MN, TE_XF_B_NEG, TE_EPI_MULPOS_ACC)
    TE_CASE4(TE_L_K, TE_L_MN, TE_XF_B_POS, TE_EPI_MULNEG_ACC)
    TE_CASE(TE_L_K, TE_L_K, TE_XF_NONE, TE_EPI_SD)
    TE_CASE(TE_L_K, TE_L_K, TE_XF_NONE, TE_EPI_MUL)
    TE_CASE(TE_L_MN, TE_L_MN, TE_XF_NONE, TE_EPI_MUL)
    TE_CASE(TE_L_K, TE_L_MN, TE_XF_NONE, TE_EPI_MUL)
    TE_CASE(TE_L_K, TE_L_MN, TE_XF_NONE, TE_EPI_ACCUM)
    // first-layer z^B rule: S W+, S W-
    TE_CASE(TE_L_K, TE_L_MN, TE_XF_B_POS, TE_EPI_STORE)
    TE_CASE(TE_L_K, TE_L_MN, TE_XF_B_NEG, TE_EPI_STORE)
    te_set_last_error("te_gemm: unsupported (layout, transform, epilogue) combination");
    return TE_ERR_UNSUPPORTED;
}
