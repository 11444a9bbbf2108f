// Tensor-core GEMMs of the engines on Hopper (sm_90a): every contraction of te_gemm_tc.h runs on ONE kernel template,
// wg_kernel<P>, built on wgmma.mma_async with fp32 accumulators in registers.
//
//   Two consumer warpgroups (threads 0..255), tile BM = 128 rows (64 per warpgroup) x P::BN columns.
//   Operand tiles are K-major, one 128-byte row per tile row (32 tf32 / 64 fp16 / bf16 elements), in the 128-byte
//   swizzled layout wgmma reads (16-byte chunk c of row r at r * 128 + ((c ^ (r % 8)) << 4)).  Two mainloops:
//   P::TMA: persistent CTAs with a third, producer warpgroup whose one thread feeds a ring of up to 8 shared-memory stages
//   by TMA behind full / empty mbarriers, and the consumers apply the problem's operand transform (TF32 rounding, |x|,
//   hi / lo split, transposition of MN-major sources) in shared memory (tma_tiles).  Otherwise every thread of a
//   256-thread CTA loads its share of the next k-block from global memory into registers, applies the transform (x+ / x-,
//   hi / lo split) and stores it into the other of two shared-memory stages while the wgmmas of the current k-block run
//   (reg_tile).  Both issue the same wgmmas in the same order per tile.
//   P::CHUNK > 0: the reduction is cut into chunks of CHUNK k-blocks; each chunk accumulates in its own registers and is
//   added into fp32 sums with round-to-nearest adds (optionally times a per-row power-of-two block scale), so a long
//   reduction does not ride on the tensor core's accumulator rounding and block-scaled fp16 operands get their scale.
//   A problem declares its operand format (P::FMT), its tile width (P::BN) and its products in issue order (P::PRODS);
//   the stage layout and the wgmma sequence of every k-block follow from those (Stage, issue below).
//
// Problems (structs below): the z+ rule's two contractions (two-pass S, single-pass S1, R; TF32, bf16 and block-scaled fp16
// operand forms), the two halves of the layers_lrp Linear rule (single-pass TF32), the Linear GEMMs (3xTF32, single-pass TF32, fp16 split, single-pass fp16), the attention-shaped N x N and
// token-reduced N x d contractions and the dense rollout product.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <string.h>
#include <algorithm>
#include <string>
#include <type_traits>
#include <utility>

#include "te_gemm_tc.h"
#include "te_wgmma.cuh"

namespace {

constexpr int BM = 128, NTHREADS = 256;

// ---- PTX helpers --------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void wg_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }

// mbarriers (CTA scope), TMA tile loads, warpgroup register hand-over
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
// returns once the phase of parity `parity` has completed (a fresh barrier counts its phase of parity 1 as completed)
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
                     : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    } while (!done);
}
// the box of map at (k, row) into shared memory at dst; completes its bytes on bar
__device__ __forceinline__ void tma_load(uint32_t dst, const CUtensorMap* map, int k, int row, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(dst), "l"((uint64_t)map), "r"(k), "r"(row), "r"(bar) : "memory");
}
// the same for a 3-D map at (x, y, z)
__device__ __forceinline__ void tma_load3(uint32_t dst, const CUtensorMap* map, int x, int y, int z, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 ::"r"(dst), "l"((uint64_t)map), "r"(x), "r"(y), "r"(z), "r"(bar) : "memory");
}
__device__ __forceinline__ void bar_named(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

__device__ __forceinline__ float to_tf32(float x) {
    uint32_t u;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(x));
    return __uint_as_float(u);
}
__device__ __forceinline__ float4 tf32x4(float4 v) { return make_float4(to_tf32(v.x), to_tf32(v.y), to_tf32(v.z), to_tf32(v.w)); }
__device__ __forceinline__ float4 absx4(float4 v) { return make_float4(fabsf(v.x), fabsf(v.y), fabsf(v.z), fabsf(v.w)); }
__device__ __forceinline__ float4 posx4(float4 v) { return make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f)); }
__device__ __forceinline__ float4 negx4(float4 v) { return make_float4(fminf(v.x, 0.f), fminf(v.y, 0.f), fminf(v.z, 0.f), fminf(v.w, 0.f)); }
__device__ __forceinline__ float4 subx4(float4 a, float4 b) { return make_float4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }

// 2^x for x <= 0 in one MUFU instruction (ex2.approx.ftz: 2^-22 relative)
__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// byte offset of 16-byte chunk c of row r in a swizzled K-major tile
__device__ __forceinline__ uint32_t swz(int r, int c) { return (uint32_t)r * 128u + ((uint32_t)(c ^ (r & 7)) << 4); }

// wgmma shared-memory descriptor of a K-major, 128-byte-swizzled tile (1024-byte aligned): start >> 4, LBO = 1 (unused for
// swizzled K-major), SBO = 1024 B (8 rows x 128 B), layout type 1 = SWIZZLE_128B.  Advancing K by 32 bytes inside the
// 128-byte row adds 2 to the start field.
__device__ __forceinline__ uint64_t sdesc(uint32_t saddr) {
    uint64_t d = (uint64_t)((saddr & 0x3FFFFu) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

constexpr int TILE128 = 128 * 128;                         // bytes of a 128-row operand tile

// ---- products and stage layout ----------------------------------------------------------------------------------------
// One product of a k-step: accumulator ACC += A tile A times B tile B.  Prods lists a problem's products in issue order; the
// order of products into one accumulator fixes its rounding, so it is part of the problem's arithmetic.
template <int ACC, int A, int B>
struct Pr {
    static constexpr int acc = ACC, a = A, b = B;
};
template <class... T>
struct Prods {
    static constexpr int N = sizeof...(T), NACC = 1 + std::max({T::acc...});
    static constexpr int NTA = 1 + std::max({T::a...}), NTB = 1 + std::max({T::b...});
    // the first product into its accumulator: the one that takes scale_d (0 starts a sum) on k-step 0
    __host__ __device__ static constexpr bool first(int i) {
        constexpr int acc[] = {T::acc...};
        for (int j = 0; j < i; ++j)
            if (acc[j] == acc[i]) return false;
        return true;
    }
};
using One = Prods<Pr<0, 0, 0>>;
// A = [hi | lo], B = [hi | lo]: hi*hi + lo*hi + hi*lo, the small terms first (3xTF32 and the three-term fp16 split)
using Split3 = Prods<Pr<0, 1, 0>, Pr<0, 0, 1>, Pr<0, 0, 0>>;

// A stage: the problem's A tiles (BM rows each), then its B tiles (BN rows each), then LAND bytes where TMA lands MN-major
// sources before the consumers transpose them into the tiles; a(i) / b(j) / land() are byte offsets in it.
template <class PRODS, int BN, int LAND = 0>
struct Stage {
    static constexpr int NTA = PRODS::NTA, NTB = PRODS::NTB;
    static constexpr int BYTES = NTA * TILE128 + NTB * BN * 128 + LAND;
    __host__ __device__ static constexpr uint32_t a(int i) { return (uint32_t)i * TILE128; }
    __host__ __device__ static constexpr uint32_t b(int j) { return (uint32_t)(NTA * TILE128 + j * BN * 128); }
    __host__ __device__ static constexpr uint32_t land() { return (uint32_t)(NTA * TILE128 + NTB * BN * 128); }
};

enum { OP_TF32 = 0, OP_BF16 = 1, OP_F16 = 2 };
template <int FMT, int NR>
__device__ __forceinline__ void wgmma_fmt(float (&d)[NR], uint64_t a, uint64_t b, uint32_t scale_d) {
    if constexpr (FMT == OP_TF32) wgmma_tf32(d, a, b, scale_d);
    else if constexpr (FMT == OP_BF16) wgmma_bf16(d, a, b, scale_d);
    else wgmma_f16(d, a, b, scale_d);
}
template <int FMT, class... T, size_t... I, int NA, int NR, int TA, int TB>
__device__ __forceinline__ void issue_kstep(Prods<T...>, std::index_sequence<I...>, float (&acc)[NA][NR], const uint64_t (&a)[TA],
                                            const uint64_t (&b)[TB], uint64_t q, uint32_t sd) {
    (wgmma_fmt<FMT>(acc[T::acc], a[T::a] + q, b[T::b] + q, Prods<T...>::first(I) ? sd : 1u), ...);
}
// The wgmmas of one k-block (the four 32-byte k-steps of a 128-byte row) on stage st; sd = 0 starts the sums.
// Warpgroup wg takes rows 64 wg .. 64 wg + 63 of every A tile.
template <class P, int NA, int NR>
__device__ __forceinline__ void issue(uint32_t st, int wg, float (&acc)[NA][NR], uint32_t sd) {
    using L = typename P::L;
    uint64_t a[L::NTA], b[L::NTB];
#pragma unroll
    for (int i = 0; i < L::NTA; ++i) a[i] = sdesc(st + L::a(i) + (uint32_t)wg * 64u * 128u);
#pragma unroll
    for (int j = 0; j < L::NTB; ++j) b[j] = sdesc(st + L::b(j));
#pragma unroll
    for (int k = 0; k < 4; ++k)
        issue_kstep<P::FMT>(typename P::PRODS{}, std::make_index_sequence<P::PRODS::N>{}, acc, a, b, (uint64_t)(2 * k),
                            (k == 0) ? sd : 1u);
}

// ---- operand loaders: each thread handles 16-byte chunks idx = tid, tid + 256, ... of a rows x 128-byte tile ----------
// fp32 source, K-major: tile row r = source row row0 + r (valid below nrows), chunk c = elements k0 + 4c .. +3 (valid below K).
// f(r, c, v) stores the (transformed) chunk.
template <class F>
__device__ __forceinline__ void for_k32(int rows, const float* __restrict__ base, long long ld, long long row0, long long nrows,
                                        int k0, int K, int tid, F f) {
    for (int idx = tid; idx < rows * 8; idx += NTHREADS) {
        const int r = idx >> 3, c = idx & 7;
        const long long gr = row0 + r;
        const int k = k0 + 4 * c;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (gr < nrows) {
            const float* src = base + gr * ld + k;
            if (k + 3 < K) v = *reinterpret_cast<const float4*>(src);
            else {
                if (k < K) v.x = src[0];
                if (k + 1 < K) v.y = src[1];
                if (k + 2 < K) v.z = src[2];
            }
        }
        f(r, c, v);
    }
}
__device__ __forceinline__ void st4(uint8_t* tile, int r, int c, float4 v) { *reinterpret_cast<float4*>(tile + swz(r, c)) = v; }
// hi / lo split of a chunk into two tiles: hi = tf32(v), lo = tf32(v - hi)
__device__ __forceinline__ void st_split(uint8_t* hi, uint8_t* lo, int r, int c, float4 v) {
    const float4 h = tf32x4(v);
    st4(hi, r, c, h);
    st4(lo, r, c, tf32x4(subx4(v, h)));
}

// ---- operand transforms in shared memory (TMA mainloop), rows r0 .. r0 + n - 1 of a tile by thread t of nt ------------
// The swizzle permutes the chunks within a row, so an element-wise transform walks the rows' 16-byte chunks in order.
// In place: v = f(v).
template <class F>
__device__ __forceinline__ void map_rows(uint8_t* tile, int r0, int n, int t, int nt, F f) {
    float4* a = reinterpret_cast<float4*>(tile + r0 * 128);
    for (int i = t; i < n * 8; i += nt) a[i] = f(a[i]);
}
// hi / lo split in place: the raw value landed in hi; the same arithmetic as st_split
__device__ __forceinline__ void split_rows(uint8_t* hi, uint8_t* lo, int r0, int n, int t, int nt) {
    float4* h = reinterpret_cast<float4*>(hi + r0 * 128);
    float4* l = reinterpret_cast<float4*>(lo + r0 * 128);
    for (int i = t; i < n * 8; i += nt) {
        const float4 v = h[i], vh = tf32x4(v);
        h[i] = vh;
        l[i] = tf32x4(subx4(v, vh));
    }
}
// Transposition of an MN-major source.  It lands as boxes of 32 source rows (k) x 32 fp32 (tile rows), 128-byte swizzled
// like a tile (element (k, m) of a box at k * 128 + ((m / 4) ^ (k % 8)) * 16 + (m % 4) * 4), box j holding tile rows
// 32 j .. 32 j + 31.  Chunk c of tile row r is (k = 4c .. 4c + 3, m = r): f(r, c, v) stores it.  Consecutive threads take
// consecutive rows, so a warp's four loads of one k each hit 32 different banks and each quarter-warp's float4 stores
// (rows r .. r + 7, one chunk) hit 8 different 16-byte bank groups.
template <class F>
__device__ __forceinline__ void transpose_rows(const uint8_t* land, int r0, int n, int t, int nt, F f) {
    for (int i = t; i < n * 8; i += nt) {
        const int r = r0 + i % n, c = i / n, m = r & 31;
        const uint8_t* box = land + (r >> 5) * 4096 + (m & 3) * 4;
        float e[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int k = 4 * c + u;
            e[u] = *reinterpret_cast<const float*>(box + k * 128 + (((m >> 2) ^ (k & 7)) << 4));
        }
        f(r, c, make_float4(e[0], e[1], e[2], e[3]));
    }
}
// The stores of a transposed chunk into a single-pass (TF32-rounded) or split (hi / lo) tile pair
template <bool SP>
__device__ __forceinline__ auto put_tf32(uint8_t* hi, uint8_t* lo) {
    return [=](int r, int c, float4 v) {
        if (SP) st4(hi, r, c, tf32x4(v));
        else st_split(hi, lo, r, c, v);
    };
}
// An operand that landed K-major: TF32-rounded (SP) or split into hi / lo in place
template <bool SP>
__device__ __forceinline__ void fix_tf32(uint8_t* hi, uint8_t* lo, int r0, int n, int t, int nt) {
    if (SP) map_rows(hi, r0, n, t, nt, [](float4 v) { return tf32x4(v); });
    else split_rows(hi, lo, r0, n, t, nt);
}

// ---- accumulator fragments: element j of a warpgroup's m64nN accumulator sits at
//      row = 16 * warp + lane / 4 + 8 * ((j / 2) % 2), column = 8 * (j / 4) + 2 * (lane % 4) + j % 2 --------------------
__device__ __forceinline__ int frag_row(int tid, int j) { return 64 * (tid >> 7) + 16 * ((tid >> 5) & 3) + ((tid & 31) >> 2) + 8 * ((j >> 1) & 1); }
__device__ __forceinline__ int frag_col(int tid, int j) { return 8 * (j >> 2) + 2 * (tid & 3) + (j & 1); }

// ---- the kernel -----------------------------------------------------------------------------------------------------
// The TMA problems' tensor maps, one per source (A tiles, then B tiles), and their tile grid: nz batches (the attention
// problems' sample x head) of mtiles x ntiles tiles.
// After the P::NMAPS stage maps come the P::EPI_MAPS maps of the epilogue operands.
constexpr int TMA_MAPS = 5;
struct TmaArgs {
    CUtensorMap map[TMA_MAPS];
    int mtiles, ntiles, nz;
};
// what the consumers of a TMA problem transform in shared memory before the wgmmas read a stage (P::FIX, P::fix)
enum { FIX_NONE = 0, FIX_A = 1, FIX_AB = 2 };
constexpr int NTHREADS_TMA = 384, SMEM_MAX = 227 * 1024;
// stages of a TMA problem: as many as fit next to its epilogue buffer (epi bytes), the 1024-byte alignment slack and the
// barriers, at most 8
__host__ __device__ constexpr int tma_stages(int bytes, int epi) {
    return (SMEM_MAX - 1024 - 256 - epi) / bytes < 8 ? (SMEM_MAX - 1024 - 256 - epi) / bytes : 8;
}

// ---- epilogue operands (TMA mainloop) ---------------------------------------------------------------------------------
// A problem's P::EPI_MAPS fp32 operands of the output's shape ([rows, cols] at a row stride, e.g. R and y of the z+ S
// kernel) are loaded per tile by the producer into an epilogue buffer behind the stages: each operand's BM x BN tile at
// (m0, n0) as BN / 32 boxes of 32 columns x BM rows, 128-byte swizzled like an operand tile, so that a warp's float2 reads
// of a fragment (8 rows x 32 bytes) hit every bank group at most twice.
template <class P>
__host__ __device__ constexpr int epi_bytes() { return P::EPI_MAPS * BM * P::BN * 4; }
// the float2 at columns c, c + 1 (c even) of tile-local row r of the epilogue operand tile at t
__device__ __forceinline__ float2 epi_f2(const uint8_t* t, int r, int c) {
    return *reinterpret_cast<const float2*>(t + (c >> 5) * (BM * 128) + swz(r, (c & 31) >> 2) + (c & 3) * 4);
}

// chunk fold: tot += acc times the per-row block scale of chunk ch
template <class P, int NA, int NR, int NT, int NTR>
__device__ __forceinline__ void fold(const P& p, float (&acc)[NA][NR], float (&tot)[NT][NTR], int m0, int ch, int z, int tid) {
    const float s0 = p.chunk_scale(m0 + frag_row(tid, 0), ch, z), s1 = p.chunk_scale(m0 + frag_row(tid, 2), ch, z);
#pragma unroll
    for (int a = 0; a < NA; ++a)
#pragma unroll
        for (int j = 0; j < NR; ++j) tot[a][j] = fmaf(acc[a][j], ((j >> 1) & 1) ? s1 : s0, tot[a][j]);
}
template <int NA, int NR>
__device__ __forceinline__ void zero(float (&v)[NA][NR]) {
#pragma unroll
    for (int a = 0; a < NA; ++a)
#pragma unroll
        for (int j = 0; j < NR; ++j) v[a][j] = 0.f;
}

// Register mainloop: all 256 threads load the next k-block (with the problem's element transform) into the other of two
// stages while the current k-block's wgmmas run; one tile per CTA.
template <class P>
__device__ __forceinline__ void reg_tile(const P& p, uint8_t* smem, int col_fast) {
    constexpr int NR = P::BN / 2;
    constexpr int NA = P::PRODS::NACC;
    constexpr int STAGE = P::L::BYTES;
    constexpr int NT = P::CHUNK ? NA : 1, NTR = P::CHUNK ? NR : 1;
    const int tid = threadIdx.x, wg = tid >> 7;
    const int m0 = (col_fast ? blockIdx.y : blockIdx.x) * BM, n0 = (col_fast ? blockIdx.x : blockIdx.y) * P::BN;
    const int z = blockIdx.z;
    float acc[NA][NR];
    float tot[NT][NTR];
    zero(acc);
    zero(tot);

    const int kb = p.kblocks();
    p.load(smem, 0, m0, n0, z, tid);
    fence_proxy_async();
    __syncthreads();
    for (int it = 0; it < kb; ++it) {
        const bool fresh = P::CHUNK ? (it % P::CHUNK == 0) : (it == 0);
        wg_fence();
        issue<P>(smem_u32(smem + (it & 1) * STAGE), wg, acc, fresh ? 0u : 1u);
        wg_commit();
        if (it + 1 < kb) p.load(smem + ((it + 1) & 1) * STAGE, it + 1, m0, n0, z, tid);
        wg_wait0();
        if constexpr (P::CHUNK > 0)
            if ((it + 1) % P::CHUNK == 0 || it + 1 == kb) fold(p, acc, tot, m0, it / P::CHUNK, z, tid);
        fence_proxy_async();
        __syncthreads();
    }
    if constexpr (P::CHUNK > 0) p.epilogue(tot, m0, n0, z, tid, nullptr);
    else p.epilogue(acc, m0, n0, z, tid, nullptr);
}

// TMA mainloop on persistent CTAs.  Warpgroups 0 and 1 (threads 0..255, the same rows and fragments as the register
// mainloop) consume; warpgroup 2 produces: one thread issues the TMA boxes of every stage tile into a ring of S stages,
// each with a full barrier (the producer's expect_tx in P::produce, completed by the TMA bytes) and an empty barrier (one
// arrive per consumer warp once the stage's wgmmas have retired).  Tile t = blockIdx.x, blockIdx.x + gridDim.x, ... is
// decoded batch-major, then column-fastest (the tiles of one batch are adjacent, so its operand panels are reused from L2),
// and the producer runs into the next tile's k-blocks while the consumers run the epilogue.
// Consumers keep one k-block's wgmmas in flight (wait_group 1) and wait for all only before a chunk fold and the epilogue;
// wgmmas into one accumulator execute in issue order, so every tile's sums are those of the register mainloop.
// P::FIX: the stage lands raw and the consumers run P::fix on it (TF32 rounding, hi / lo split, transposition of MN-major
// sources): FIX_A, each consumer warpgroup its own 64 rows of A behind its own named barrier; FIX_AB, in addition the B tiles
// shared by both warpgroups, their rows split over all 256 consumer threads, behind one 256-thread named barrier.
// P::EPI_MAPS > 0: the producer also loads the tile's epilogue operands into the epilogue buffer behind the stages, with its
// own full barrier (expect_tx) and empty barrier (one arrive per consumer warp after the epilogue).  It issues them once the
// first min(S, kb) k-blocks of the tile are issued, where it would next wait for a stage the consumers free only after the
// previous tile's epilogue, so the one buffer costs the stage ring no prefetch; the operands land during the mainloop.
template <class P>
__device__ __forceinline__ void tma_tiles(const P& p, const TmaArgs& ta, uint8_t* smem) {
    using L = typename P::L;
    constexpr int NR = P::BN / 2;
    constexpr int NA = P::PRODS::NACC;
    constexpr int STAGE = L::BYTES, EPI = epi_bytes<P>(), S = tma_stages(STAGE, EPI);
    constexpr int NT = P::CHUNK ? NA : 1, NTR = P::CHUNK ? NR : 1;
    static_assert(S >= 2, "a TMA problem needs two stages");
    __shared__ __align__(8) uint64_t bars[2 * S + 2];        // full[S], empty[S], then the epilogue buffer's full, empty
    const int tid = threadIdx.x, wg = tid >> 7;
    const uint32_t full0 = smem_u32(bars), empty0 = full0 + 8u * S, st0 = smem_u32(smem);
    const uint32_t efull = full0 + 16u * S, eempty = efull + 8u, ebuf = st0 + (uint32_t)S * STAGE;
    if (tid == 0) {
        for (int s = 0; s < S; ++s) {
            mbar_init(full0 + 8u * s, 1);
            mbar_init(empty0 + 8u * s, 8);
        }
        mbar_init(efull, 1);
        mbar_init(eempty, 8);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    const int kb = p.kblocks(), per_z = ta.mtiles * ta.ntiles, ntiles = ta.nz * per_z;
    int stage = 0;
    uint32_t phase = 0;
    auto decode = [&](int t, int& m0, int& n0, int& z) {
        z = t / per_z;
        const int r = t - z * per_z;
        m0 = (r / ta.ntiles) * BM;
        n0 = (r % ta.ntiles) * P::BN;
    };

    if (wg == 2) {
        setmaxnreg_dec<40>();
        if (tid != 2 * 128) return;
        uint32_t ephase = 0;
        for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
            int m0, n0, z;
            decode(t, m0, n0, z);
            for (int it = 0; it < kb; ++it) {
                mbar_wait(empty0 + 8u * stage, phase ^ 1u);
                p.produce(ta, st0 + (uint32_t)stage * STAGE, full0 + 8u * stage, it, m0, n0, z);
                if (++stage == S) { stage = 0; phase ^= 1u; }
                if constexpr (EPI > 0) {
                    if (it == min(S, kb) - 1) {
                        mbar_wait(eempty, ephase ^ 1u);
                        mbar_expect_tx(efull, EPI);
#pragma unroll
                        for (int i = 0; i < P::EPI_MAPS; ++i)
#pragma unroll
                            for (int b = 0; b < P::BN / 32; ++b)
                                tma_load(ebuf + (uint32_t)(i * BM * P::BN * 4 + b * BM * 128), &ta.map[P::NMAPS + i], n0 + 32 * b,
                                         m0, efull);
                        ephase ^= 1u;
                    }
                }
            }
        }
        return;
    }

    setmaxnreg_inc<232>();
    float acc[NA][NR];
    float tot[NT][NTR];
    auto release = [&](int s) {
        if ((tid & 31) == 0) mbar_arrive(empty0 + 8u * s);
    };
    // the wgmmas of the next k-block (sd = 0 starts the sums) on the next stage, committed as one group
    auto consume = [&](uint32_t sd) {
        mbar_wait(full0 + 8u * stage, phase);
        if constexpr (P::FIX != FIX_NONE) {
            p.fix(smem + (uint32_t)stage * STAGE, wg, tid);
            fence_proxy_async();
            if constexpr (P::FIX == FIX_A) bar_named(1 + wg, 128);
            else bar_named(3, 256);
        }
        wg_fence();
        issue<P>(st0 + (uint32_t)stage * STAGE, wg, acc, sd);
        wg_commit();
    };
    auto next = [&] {
        if (++stage == S) { stage = 0; phase ^= 1u; }
    };
    constexpr int CH = P::CHUNK;
    uint32_t ephase = 0;
    for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
        int m0, n0, z;
        decode(t, m0, n0, z);
        zero(acc);
        zero(tot);
        // One chunk (the whole reduction when CHUNK = 0) per pass: its first k-block starts the sums, the steady state
        // waits for all but the newest group and releases the previous stage, and only the chunk's end waits for all.
        // No branch inside the k-loop selects between the two waits, so ptxas keeps the one group in flight.
        for (int k0 = 0; k0 < kb; k0 += CH ? CH : kb) {
            const int k1 = CH ? min(k0 + CH, kb) : kb;
            consume(0u);
            for (int it = k0 + 1; it < k1; ++it) {
                const int prev = stage;
                next();
                consume(1u);
                wg_wait1();
                release(prev);
            }
            wg_wait0();
            release(stage);
            next();
            if constexpr (CH > 0) fold(p, acc, tot, m0, k0 / CH, z, tid);
        }
        if constexpr (EPI > 0) mbar_wait(efull, ephase);
        if constexpr (P::CHUNK > 0) p.epilogue(tot, m0, n0, z, tid, smem + (uint32_t)S * STAGE);
        else p.epilogue(acc, m0, n0, z, tid, smem + (uint32_t)S * STAGE);
        if constexpr (EPI > 0) {
            __syncwarp();                                     // the warp's reads of the buffer are done
            if ((tid & 31) == 0) mbar_arrive(eempty);
            ephase ^= 1u;
        }
    }
}

template <class P>
__global__ void __launch_bounds__(P::TMA ? NTHREADS_TMA : NTHREADS, 1)
    wg_kernel(const P p, const __grid_constant__ TmaArgs ta, int col_fast) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    if constexpr (P::TMA) tma_tiles(p, ta, smem);
    else reg_tile(p, smem, col_fast);
}

// unit block scale for the plain chunked problems
struct NoScale {
    __device__ __forceinline__ float chunk_scale(int, int, int) const { return 1.f; }
};

// Problems with P::TMA run the TMA mainloop; tile(i) names the global source of tensor map i (A tiles, then B tiles): rows x
// cols elements at row stride ld, read in boxes of 128 bytes x box_rows rows, with count > 0 a third dimension of count such
// matrices at stride cstride (elements).  P::produce issues a stage's boxes from the P::NMAPS maps.  The others load through
// registers (P::load).
struct TmaTile {
    const void* base;
    long long rows, cols, ld;
    int box_rows;
    long long count = 0, cstride = 0;
};
// P::produce of the problems whose stage tiles are all K-major boxes of 2-D maps at (k-block, tile row): A tile i from
// map i at row m0, B tile j from map NTA + j at row n0
template <class P>
__device__ __forceinline__ void produce_tiles(const TmaArgs& ta, uint32_t st, uint32_t bar, int it, int m0, int n0) {
    using L = typename P::L;
    constexpr int KE = P::FMT == OP_TF32 ? 32 : 64;          // elements in a 128-byte row
    mbar_expect_tx(bar, L::BYTES);
#pragma unroll
    for (int i = 0; i < L::NTA; ++i) tma_load(st + L::a(i), &ta.map[i], it * KE, m0, bar);
#pragma unroll
    for (int j = 0; j < L::NTB; ++j) tma_load(st + L::b(j), &ta.map[L::NTA + j], it * KE, n0, bar);
}
#define TE_PRODUCE_TILES(P)                                                                                      \
    static constexpr int NMAPS = L::NTA + L::NTB;                                                                \
    __device__ void produce(const TmaArgs& ta, uint32_t st, uint32_t bar, int it, int m0, int n0, int) const { \
        produce_tiles<P>(ta, st, bar, it, m0, n0);                                                               \
    }

// ---- z+ rule, first contraction: S = sd(R, Z) ---------------------------------------------------------------------
// Z two-pass:    x+ W+^T + x- W-^T                        (A tiles x+ / x- transformed on load, B = W+ / W-)
// Z single-pass: ((y - bias) + |x| |W|^T) / 2             (the saved forward output y = x W^T + bias)
// The inhibitor half of the alpha-beta rule swaps the weight signs: two-pass with B = W- / W+ (wa / wb), single-pass with
// zsign = -1, Z = ((y - bias) - |x| |W|^T) / 2 == x+ W-^T + x- W+^T.  S leaves as sscale * sd(R, Z) (alpha or -beta; 1 for
// the plain z+ rule).
// OUT: 0 = S as TF32-rounded fp32, 1 = bf16, 2 = hi-only block-scaled fp16 (one 2^-e per row and 128 columns)
enum { ZO_F32 = 0, ZO_BF16 = 1, ZO_F16S = 2 };
template <bool SINGLE, bool BF, int OUT>
struct ZsProb : NoScale {
    static constexpr int BN = 128, CHUNK = 0, FMT = BF ? OP_BF16 : OP_TF32;
    using PRODS = std::conditional_t<SINGLE, One, Prods<Pr<0, 0, 0>, Pr<0, 1, 1>>>;    // two-pass: x+ W+^T, then x- W-^T
    using L = Stage<PRODS, BN>;
    static constexpr bool COL_FAST = true;
    // single-pass: TMA (A = bf16(|x|), or raw x made tf32(|x|) in shared memory); two-pass: x+ / x- formed on load
    static constexpr bool TMA = SINGLE;
    static constexpr int FIX = SINGLE && !BF ? FIX_A : FIX_NONE;
    static constexpr int EPI_MAPS = SINGLE ? 2 : 0;            // R and y, staged by the producer
    int M, N, K;
    const float* x; long long ldx;
    const void* xabs;                       // BF: bf16(|x|) [M, K]
    const void* wa; const void* wb;         // SINGLE: |W| (tf32 or bf16) ; else W+ / W- (tf32) [N, K]
    const float* r; long long ldr; const float* y; long long ldy; const float* bias;
    void* out; long long ldo; float* hs;    // hs: ZO_F16S block scales [M, N / 128]
    float sscale, zsign;                    // S = sscale * sd(R, Z) ; SINGLE: sign of the |x| |W|^T term

    __device__ int kblocks() const { return K / (BF ? 64 : 32); }
    __device__ void fix(uint8_t* st, int wg, int tid) const {
        map_rows(st + L::a(0), 64 * wg, 64, tid & 127, 128, [](float4 v) { return tf32x4(absx4(v)); });
    }
    TE_PRODUCE_TILES(ZsProb)
    TmaTile tile(int i) const {
        if (i == 0) return BF ? TmaTile{xabs, M, K, K, BM} : TmaTile{x, M, K, ldx, BM};
        if (i == 1) return TmaTile{wa, N, K, K, BN};
        return i == 2 ? TmaTile{r, M, N, ldr, BM} : TmaTile{y, M, N, ldy, BM};
    }
    __device__ void load(uint8_t* st, int kb, int m0, int n0, int, int tid) const {
        for_k32(BM, x, ldx, m0, M, kb * 32, K, tid, [&](int rr, int c, float4 v) {
            st4(st + L::a(0), rr, c, tf32x4(posx4(v)));
            st4(st + L::a(1), rr, c, tf32x4(negx4(v)));
        });
        for_k32(BN, (const float*)wa, K, n0, N, kb * 32, K, tid, [&](int rr, int c, float4 v) { st4(st + L::b(0), rr, c, v); });
        for_k32(BN, (const float*)wb, K, n0, N, kb * 32, K, tid, [&](int rr, int c, float4 v) { st4(st + L::b(1), rr, c, v); });
    }
    // Single-pass: R and y come from the epilogue buffer (eb), bias from global memory; the whole fragment's S is computed
    // before the first store.  Two-pass (register mainloop): R from global memory.
    __device__ void epilogue(float (&acc)[1][BN / 2], int m0, int n0, int, int tid, const uint8_t* eb) const {
        float sv[BN / 2];
        float rmax[2] = {0.f, 0.f};
#pragma unroll
        for (int j = 0; j < BN / 2; j += 2) {
            const int row = m0 + frag_row(tid, j), col = n0 + frag_col(tid, j);
            float2 rr = make_float2(0.f, 0.f), z = make_float2(acc[0][j], acc[0][j + 1]);
            if (row < M) {
                rr = SINGLE ? epi_f2(eb, frag_row(tid, j), frag_col(tid, j))
                            : *reinterpret_cast<const float2*>(r + (long long)row * ldr + col);
                if (SINGLE) {
                    const float2 yy = epi_f2(eb + BM * BN * 4, frag_row(tid, j), frag_col(tid, j));
                    const float2 bb = bias ? *reinterpret_cast<const float2*>(bias + col) : make_float2(0.f, 0.f);
                    // x+ W+^T + x- W-^T == (x W^T + |x| |W|^T) / 2 ; a negative result is cancellation noise of a sum of
                    // non-negative terms (zsign = -1: x+ W-^T + x- W+^T == (x W^T - |x| |W|^T) / 2, a sum of non-positive terms)
                    z.x = 0.5f * ((yy.x - bb.x) + zsign * z.x);
                    z.y = 0.5f * ((yy.y - bb.y) + zsign * z.y);
                    z = zsign > 0.f ? make_float2(fmaxf(z.x, 0.f), fmaxf(z.y, 0.f)) : make_float2(fminf(z.x, 0.f), fminf(z.y, 0.f));
                }
            }
            sv[j] = sscale * te_sd(rr.x, z.x);
            sv[j + 1] = sscale * te_sd(rr.y, z.y);
            if (OUT == ZO_F16S) rmax[(j >> 1) & 1] = fmaxf(rmax[(j >> 1) & 1], fmaxf(fabsf(sv[j]), fabsf(sv[j + 1])));
        }
#pragma unroll
        for (int j = 0; j < BN / 2; j += 2) {
            const int row = m0 + frag_row(tid, j), col = n0 + frag_col(tid, j);
            if (row >= M) continue;
            if (OUT == ZO_F32) {
                *reinterpret_cast<float2*>((float*)out + (long long)row * ldo + col) = make_float2(to_tf32(sv[j]), to_tf32(sv[j + 1]));
            } else if (OUT == ZO_BF16) {
                *reinterpret_cast<__nv_bfloat162*>((__nv_bfloat16*)out + (long long)row * ldo + col) = __floats2bfloat162_rn(sv[j], sv[j + 1]);
            }
        }
        if (OUT == ZO_F16S) {
            // the tile's 128 columns of a row are one scale block, held by the 4 lanes of a quad
            float sc[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float m = rmax[h];
                m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
                m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
                float si;
                te_f16_block_scale(m, sc[h], si);
                const int row = m0 + frag_row(tid, 2 * h);
                if ((tid & 3) == 0 && row < M) hs[(long long)row * (N / 128) + n0 / 128] = si;
            }
#pragma unroll
            for (int j = 0; j < BN / 2; j += 2) {
                const int row = m0 + frag_row(tid, j), col = n0 + frag_col(tid, j);
                const float s = sc[(j >> 1) & 1];
                if (row < M) *reinterpret_cast<__half2*>((__half*)out + (long long)row * N + col) = __floats2half2_rn(sv[j] * s, sv[j + 1] * s);
            }
        }
    }
};

// ---- z+ rule, second contraction: R_in = x+ (S W+) + x- (S W-) --------------------------------------------------------
// KIND 0: S and W+-^T TF32 fp32 ; 1: bf16 ; 2: block-scaled fp16 S (scale per row and 128 k) with row-scaled fp16 W+-^T
// The inhibitor half of the alpha-beta rule passes the weights swapped (wp = W-^T, wn = W+^T and their scales) with accum
// set: R_in += x+ (S W-) + x- (S W+).
template <int KIND>
struct ZrProb {
    static constexpr int BN = (KIND == 2) ? 64 : 128, CHUNK = (KIND == 2) ? 2 : 0;
    static constexpr int FMT = KIND == 0 ? OP_TF32 : KIND == 1 ? OP_BF16 : OP_F16;
    using PRODS = Prods<Pr<0, 0, 0>, Pr<1, 0, 1>>;           // S W+ and S W- into their own accumulators
    using L = Stage<PRODS, BN>;
    static constexpr bool TMA = true;
    // x, staged by the producer, except for KIND 0: its 64 KB buffer would cost it one of four 48 KB stages, and the TF32
    // kernel runs faster with the stage and x read from global memory in the epilogue
    static constexpr int FIX = FIX_NONE, EPI_MAPS = KIND == 0 ? 0 : 1;
    int M, N, K;
    const void* s; const void* wp; const void* wn;     // S [M, K] (row stride K), W+^T / W-^T [N, K]
    const float* rs; int rs_ld; const float* cp; const float* cn;   // KIND 2: scales of S, of the rows of W+^T / W-^T
    const float* x; long long ldx; float* out; long long ldo;
    int accum;                                                      // add into out instead of overwriting it

    __device__ int kblocks() const { return K / (KIND ? 64 : 32); }
    TE_PRODUCE_TILES(ZrProb)
    __device__ float chunk_scale(int row, int ch, int) const { return (KIND == 2 && row < M) ? rs[(long long)row * rs_ld + ch] : 1.f; }
    TmaTile tile(int i) const {
        if (i == 0) return TmaTile{s, M, K, K, BM};
        return i < 3 ? TmaTile{i == 1 ? wp : wn, N, K, K, BN} : TmaTile{x, M, N, ldx, BM};
    }
    // x comes from the epilogue buffer (eb), or for KIND 0 from global memory, the column scales from global memory.
    // Accumulating, each thread reads the out elements it then writes, from global memory: out is not staged (it may alias
    // x, and the value read must be the one the previous launch left).  All reads of the fragment are done into acc[0]
    // before the first store.
    __device__ void epilogue(float (&acc)[2][BN / 2], int m0, int n0, int, int tid, const uint8_t* eb) const {
#pragma unroll
        for (int j = 0; j < BN / 2; j += 2) {
            const int row = m0 + frag_row(tid, j), col = n0 + frag_col(tid, j);
            if (row >= M) continue;
            const float2 xv = EPI_MAPS ? epi_f2(eb, frag_row(tid, j), frag_col(tid, j))
                                       : *reinterpret_cast<const float2*>(x + (long long)row * ldx + col);
            float2 ap = make_float2(acc[0][j], acc[0][j + 1]), an = make_float2(acc[1][j], acc[1][j + 1]);
            if (KIND == 2) {
                ap.x *= cp[col]; ap.y *= cp[col + 1];
                an.x *= cn[col]; an.y *= cn[col + 1];
            }
            float2 v = make_float2(fmaxf(xv.x, 0.f) * ap.x + fminf(xv.x, 0.f) * an.x, fmaxf(xv.y, 0.f) * ap.y + fminf(xv.y, 0.f) * an.y);
            if (accum) {
                const float2 prev = *reinterpret_cast<const float2*>(out + (long long)row * ldo + col);
                v = make_float2(prev.x + v.x, prev.y + v.y);
            }
            acc[0][j] = v.x;
            acc[0][j + 1] = v.y;
        }
#pragma unroll
        for (int j = 0; j < BN / 2; j += 2) {
            const int row = m0 + frag_row(tid, j), col = n0 + frag_col(tid, j);
            if (row < M) *reinterpret_cast<float2*>(out + (long long)row * ldo + col) = make_float2(acc[0][j], acc[0][j + 1]);
        }
    }
};

// ---- Linear rule of the layers_lrp library: each half over its own denominator --------------------------------------
// S half:  S = sd(R, x+- W+-^T), TF32-rounded fp32 [M, N] (A = tf32(x+) or tf32(x-) transformed on load, B = W+ / W-).
// Both factors of every product share a sign, so the denominator is a sum of non-negative terms: no cancellation, and it
// is exactly 0 (S = 0) only when every term is.  The inhibitor products of the alpha-beta rule pair x+ with W- and x- with
// W+ (w is a runtime operand; NEG is the sign of x only): sums of non-positive terms, equally well conditioned.
// S leaves scaled by sscale (alpha, -beta, or 1 for the plain rule).
template <bool NEG>
struct LrpSProb : NoScale {
    static constexpr int BN = 128, CHUNK = 0, FMT = OP_TF32;
    using PRODS = One;
    using L = Stage<PRODS, BN>;
    static constexpr bool COL_FAST = true, TMA = false;
    int M, N, K;
    const float* x; long long ldx; const float* w;      // w: W+ or W- (tf32) [N, K]
    const float* r; long long ldr; float* out;           // out: S [M, N], row stride N
    float sscale;
    __device__ int kblocks() const { return K / 32; }
    __device__ void load(uint8_t* st, int kb, int m0, int n0, int, int tid) const {
        for_k32(BM, x, ldx, m0, M, kb * 32, K, tid, [&](int rr, int c, float4 v) { st4(st + L::a(0), rr, c, tf32x4(NEG ? negx4(v) : posx4(v))); });
        for_k32(BN, w, K, n0, N, kb * 32, K, tid, [&](int rr, int c, float4 v) { st4(st + L::b(0), rr, c, v); });
    }
    __device__ void epilogue(float (&acc)[1][BN / 2], int m0, int n0, int, int tid, const uint8_t*) const {
#pragma unroll
        for (int j = 0; j < BN / 2; j += 2) {
            const int row = m0 + frag_row(tid, j), col = n0 + frag_col(tid, j);
            if (row >= M) continue;
            const float2 rr = *reinterpret_cast<const float2*>(r + (long long)row * ldr + col);
            *reinterpret_cast<float2*>(out + (long long)row * N + col) =
                make_float2(to_tf32(sscale * te_sd(rr.x, acc[0][j])), to_tf32(sscale * te_sd(rr.y, acc[0][j + 1])));
        }
    }
};
// R half:  out = x+ * (S W+)  (NEG false),  out += x- * (S W-)  (NEG true).  A = S [M, K], B = W+^T / W-^T [N, K] (W-^T /
// W+^T for the inhibitor products).  accum: the NEG false half adds into out as well (every product after the first).
template <bool NEG>
struct LrpRProb : NoScale {
    static constexpr int BN = 128, CHUNK = 0, FMT = OP_TF32;
    using PRODS = One;
    using L = Stage<PRODS, BN>;
    static constexpr bool TMA = true;
    static constexpr int FIX = FIX_NONE, EPI_MAPS = 1;           // x, staged by the producer
    int M, N, K;
    const float* s; const float* wt;
    const float* x; long long ldx; float* out; long long ldo;
    int accum;
    __device__ int kblocks() const { return K / 32; }
    TE_PRODUCE_TILES(LrpRProb)
    TmaTile tile(int i) const {
        return i == 0 ? TmaTile{s, M, K, K, BM} : i == 1 ? TmaTile{wt, N, K, K, BN} : TmaTile{x, M, N, ldx, BM};
    }
    // x from the epilogue buffer, out read as in ZrProb (accumulating products: global memory, whole fragment first)
    __device__ void epilogue(float (&acc)[1][BN / 2], int m0, int n0, int, int tid, const uint8_t* eb) const {
#pragma unroll
        for (int j = 0; j < BN / 2; j += 2) {
            const int row = m0 + frag_row(tid, j), col = n0 + frag_col(tid, j);
            if (row >= M) continue;
            const float2 xv = epi_f2(eb, frag_row(tid, j), frag_col(tid, j));
            const float2* o = reinterpret_cast<const float2*>(out + (long long)row * ldo + col);
            float2 v;
            if (NEG) {
                const float2 prev = *o;
                v = make_float2(prev.x + fminf(xv.x, 0.f) * acc[0][j], prev.y + fminf(xv.y, 0.f) * acc[0][j + 1]);
            } else if (accum) {
                const float2 prev = *o;
                v = make_float2(prev.x + fmaxf(xv.x, 0.f) * acc[0][j], prev.y + fmaxf(xv.y, 0.f) * acc[0][j + 1]);
            } else {
                v = make_float2(fmaxf(xv.x, 0.f) * acc[0][j], fmaxf(xv.y, 0.f) * acc[0][j + 1]);
            }
            acc[0][j] = v.x;
            acc[0][j + 1] = v.y;
        }
#pragma unroll
        for (int j = 0; j < BN / 2; j += 2) {
            const int row = m0 + frag_row(tid, j), col = n0 + frag_col(tid, j);
            if (row < M) *reinterpret_cast<float2*>(out + (long long)row * ldo + col) = make_float2(acc[0][j], acc[0][j + 1]);
        }
    }
};

// ---- Linear epilogues (ids of te_gemm_tc.h) -----------------------------------------------------------------------
struct LinOut {
    int M, N;
    const float* bias; const float* E; long long lde;
    float* C; long long ldc; float* C2; long long ldc2;
};
// The Linear epilogue of a fragment in two passes: lin_value forms y from the product and the operands read before any
// store (bias; E of GELU_BWD), then lin_store writes y and the second output (gelu(y), or E + y for BIAS_ADD).  e(): the
// fragment's float2 of E (the epilogue buffer on the TMA mainloop).
// v: the product for columns col, col + 1 (already scaled)
template <int EPI, bool FAST_GRAD, class EF>
__device__ __forceinline__ float2 lin_value(const LinOut& o, int col, float v0, float v1, EF e) {
    float2 b = make_float2(0.f, 0.f);
    if ((EPI == TE_TC_EPI_BIAS || EPI == TE_TC_EPI_BIAS_GELU || EPI == TE_TC_EPI_BIAS_ADD || EPI == TE_TC_EPI_BIAS_QUICK_GELU) &&
        o.bias)
        b = *reinterpret_cast<const float2*>(o.bias + col);
    if (EPI == TE_TC_EPI_GELU_BWD) {
        const float2 ev = e();
        if (FAST_GRAD) return make_float2(v0 * te_gelu_grad_fast(ev.x), v1 * te_gelu_grad_fast(ev.y));
        return make_float2(v0 * te_gelu_grad(ev.x), v1 * te_gelu_grad(ev.y));
    }
    if (EPI == TE_TC_EPI_QUICK_GELU_BWD) {
        const float2 ev = e();
        return make_float2(v0 * te_quick_gelu_grad(ev.x), v1 * te_quick_gelu_grad(ev.y));
    }
    return make_float2(v0 + b.x, v1 + b.y);
}
template <int EPI, class EF>
__device__ __forceinline__ void lin_store(const LinOut& o, int row, int col, float2 y, EF e) {
    *reinterpret_cast<float2*>(o.C + (long long)row * o.ldc + col) = y;
    float2 y2 = make_float2(0.f, 0.f);
    if (EPI == TE_TC_EPI_BIAS_GELU) y2 = make_float2(te_gelu(y.x), te_gelu(y.y));
    if (EPI == TE_TC_EPI_BIAS_QUICK_GELU) y2 = make_float2(te_quick_gelu(y.x), te_quick_gelu(y.y));
    if (EPI == TE_TC_EPI_BIAS_ADD) {
        const float2 ev = e();
        y2 = make_float2(ev.x + y.x, ev.y + y.y);
    }
    if (EPI == TE_TC_EPI_BIAS_GELU || EPI == TE_TC_EPI_BIAS_ADD || EPI == TE_TC_EPI_BIAS_QUICK_GELU)
        *reinterpret_cast<float2*>(o.C2 + (long long)row * o.ldc2 + col) = y2;
}

// ---- Linear GEMMs: C = epi(A B^T), B = the weight copy [N, K] K-major --------------------------------------------------
// LIN_3XTF32: fp32 grade, A split on load into tf32 hi / lo, B pre-split; Split3 in chunks of 4 k-blocks.
// LIN_TF32:   single pass (activation-gradient backward): tf32(A) B^T, B rounded once.
// LIN_F16X3:  fp32 grade on block-scaled fp16 operands (te_common.cuh): A and B pre-split into hi / lo, Split3.
// LIN_F16:    single pass on the fp16 hi parts.
// The fp16 forms take one chunk = 128 k = one scale block of A; the columns carry the row scale of B.
enum { LIN_3XTF32 = 0, LIN_TF32 = 1, LIN_F16X3 = 2, LIN_F16 = 3 };
struct LinArgs {
    int K, rs_ld;
    const void* a; const void* a_lo; long long lda;  // fp32 A [M, K] (row stride lda), or the fp16 hi / lo of A (row stride K)
    const void* b; const void* b_lo;                 // tf32 or fp16 hi / lo of B
    const float* rs; const float* cs;                // fp16 forms: the scales of A [M, rs_ld] and of the rows of B [N]
    LinOut o;
};
// with CUDA 12.9, a 136-byte LinArgs made nvcc read the kernel parameter through a generic pointer, at four more registers
// in the 3xTF32 kernels; at 128 bytes it is read like the other problems' parameters
static_assert(sizeof(LinArgs) <= 128, "LinArgs: keep the kernel parameter within 128 bytes");
template <int EPI, int FORM>
struct LinProb : LinArgs {
    static constexpr bool F16 = FORM == LIN_F16X3 || FORM == LIN_F16, SPLIT = FORM == LIN_3XTF32 || FORM == LIN_F16X3;
    // The single-pass TF32 STORE form (one accumulator, no epilogue buffer) takes 256 columns: 48 KB per stage (4 stages)
    // for twice the MMAs of a 32 KB stage at 128, and the tf32(A) fix serves twice the columns.  The others stay at 128:
    // the chunked forms' acc + tot, and GELU_BWD's E buffer, would not fit at 256.  The epilogue guards the columns past N
    // (N a multiple of 128).
    static constexpr int BN = FORM == LIN_TF32 && EPI == TE_TC_EPI_STORE ? 256 : 128;
    static constexpr int CHUNK = F16 ? 2 : SPLIT ? 4 : 0, FMT = F16 ? OP_F16 : OP_TF32;
    using PRODS = std::conditional_t<SPLIT, Split3, One>;
    using L = Stage<PRODS, BN>;
    static constexpr bool COL_FAST = true;
    // the fp16 forms and the single-pass TF32 form (A rounded in shared memory) on TMA; 3xTF32 splits A on load
    static constexpr bool TMA = FORM != LIN_3XTF32;
    static constexpr int FIX = FORM == LIN_TF32 ? FIX_A : FIX_NONE;
    // E of GELU_BWD, staged by the producer on the TMA mainloop.  E of BIAS_ADD (the fp16-split forward, 64 KB stages) is
    // read from global memory before the first store: its 64 KB buffer would cost it one of three stages, and that form
    // runs faster with the stage.
    static constexpr int EPI_MAPS = TMA && (EPI == TE_TC_EPI_GELU_BWD || EPI == TE_TC_EPI_QUICK_GELU_BWD) ? 1 : 0;
    __device__ int kblocks() const { return K / (F16 ? 64 : 32); }
    __device__ float chunk_scale(int row, int ch, int) const {
        if constexpr (F16) return row < o.M ? rs[(long long)row * rs_ld + ch] : 1.f;
        else return 1.f;
    }
    __device__ void fix(uint8_t* st, int wg, int tid) const {
        map_rows(st + L::a(0), 64 * wg, 64, tid & 127, 128, [](float4 v) { return tf32x4(v); });
    }
    TE_PRODUCE_TILES(LinProb)
    TmaTile tile(int i) const {
        if (i < L::NTA) return TmaTile{i == 0 ? a : a_lo, o.M, K, F16 ? K : lda, BM};
        if (i < NMAPS) return TmaTile{i == L::NTA ? b : b_lo, o.N, K, K, BN};
        return TmaTile{o.E, o.M, o.N, o.lde, BM};
    }
    __device__ void load(uint8_t* st, int kb, int m0, int n0, int, int tid) const {
        for_k32(BM, (const float*)a, lda, m0, o.M, kb * 32, K, tid, [&](int r, int c, float4 v) { st_split(st + L::a(0), st + L::a(1), r, c, v); });
        for_k32(BN, (const float*)b, K, n0, o.N, kb * 32, K, tid, [&](int r, int c, float4 v) { st4(st + L::b(0), r, c, v); });
        for_k32(BN, (const float*)b_lo, K, n0, o.N, kb * 32, K, tid, [&](int r, int c, float4 v) { st4(st + L::b(1), r, c, v); });
    }
    // E from the epilogue buffer (eb) when staged, else from global memory; bias, the column scales and an unstaged E of
    // BIAS_ADD from global memory, for the whole fragment before the first store (C2 may alias E)
    __device__ void epilogue(float (&acc)[1][BN / 2], int m0, int n0, int, int tid, const uint8_t* eb) const {
        // the fragment's elements inside the output (at BN = 128 every column is)
        auto inside = [&](int row, int col) { return row < o.M && (BN == 128 || col < o.N); };
        constexpr bool E_FIRST = EPI == TE_TC_EPI_BIAS_ADD && EPI_MAPS == 0;
        float2 ef[E_FIRST ? BN / 4 : 1];
#pragma unroll
        for (int j = 0; j < BN / 2; j += 2) {
            const int row = m0 + frag_row(tid, j), col = n0 + frag_col(tid, j);
            if (!inside(row, col)) continue;
            if constexpr (E_FIRST) ef[j / 2] = efrag(eb, tid, j, row, col);
            auto e = [&] { return efrag(eb, tid, j, row, col); };
            float2 y;
            if constexpr (F16)                                          // exact scaling
                y = lin_value<EPI, false>(o, col, acc[0][j] * cs[col], acc[0][j + 1] * cs[col + 1], e);
            else y = lin_value<EPI, FORM == LIN_TF32>(o, col, acc[0][j], acc[0][j + 1], e);
            acc[0][j] = y.x;
            acc[0][j + 1] = y.y;
        }
#pragma unroll
        for (int j = 0; j < BN / 2; j += 2) {
            const int row = m0 + frag_row(tid, j), col = n0 + frag_col(tid, j);
            if (inside(row, col))
                lin_store<EPI>(o, row, col, make_float2(acc[0][j], acc[0][j + 1]), [&] {
                    if constexpr (E_FIRST) return ef[j / 2];
                    else return efrag(eb, tid, j, row, col);
                });
        }
    }
    __device__ float2 efrag(const uint8_t* eb, int tid, int j, int row, int col) const {
        if constexpr (EPI_MAPS > 0) return epi_f2(eb, frag_row(tid, j), frag_col(tid, j));
        else return *reinterpret_cast<const float2*>(o.E + (long long)row * o.lde + col);
    }
};

// ---- attention-shaped N x N contraction: out[b,h,i,j] = epi(alpha * sum_d A[b*N+i, h*dh+d] B[b*N+j, h*dh+d]) ------------
enum { AT_STORE = 0, AT_MUL = 1, AT_SD = 2, AT_SOFTMAX = 3, AT_RESID = 4 };
template <int EPI, bool SP, int BN_>
struct NnProb : NoScale {
    static constexpr int BN = BN_, CHUNK = 0, FMT = OP_TF32;
    using PRODS = std::conditional_t<SP, One, Split3>;
    using L = Stage<PRODS, BN>;
    // A and B land raw in their (hi) tiles from 2-D maps over the packed [batch * N, H * dh] rows; a 32-column box never
    // leaves head h (dh is 32 or 64).  Rows past a sample's N are the next sample's (zeros past the tensor): they reach only
    // the output rows and columns the epilogue masks.
    static constexpr bool TMA = true;
    static constexpr int FIX = FIX_AB, EPI_MAPS = 0;
    int N, H, dh, ld_out, batch;
    const float* a; long long lda; const float* b; long long ldb;
    const float* E; float* out; float alpha;
    __device__ int kblocks() const { return dh / 32; }
    static constexpr int NMAPS = 2;
    TmaTile tile(int i) const {
        return i == 0 ? TmaTile{a, (long long)batch * N, H * dh, lda, BM} : TmaTile{b, (long long)batch * N, H * dh, ldb, BN};
    }
    __device__ void produce(const TmaArgs& ta, uint32_t st, uint32_t bar, int kb, int m0, int n0, int bh) const {
        const int s = bh / H, k = (bh % H) * dh + kb * 32;
        mbar_expect_tx(bar, TILE128 + BN * 128);
        tma_load(st + L::a(0), &ta.map[0], k, s * N + m0, bar);
        tma_load(st + L::b(0), &ta.map[1], k, s * N + n0, bar);
    }
    __device__ void fix(uint8_t* st, int wg, int tid) const {
        fix_tf32<SP>(st + L::a(0), st + L::a(1), 64 * wg, 64, tid & 127, 128);
        fix_tf32<SP>(st + L::b(0), st + L::b(1), 0, BN, tid, 256);
    }
    __device__ void epilogue(float (&acc)[1][BN / 2], int m0, int n0, int bh, int tid, const uint8_t*) const {
        const int ncols = (N + 3) & ~3;                  // the row padding up to a multiple of 4 is written as zeros
        if constexpr (EPI == AT_SOFTMAX) {
            // softmax(alpha * A B^T) over the key axis: the tile holds every key (N <= BN); a row's values sit in one quad
            float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
            for (int j = 0; j < BN / 2; ++j)
                if (n0 + frag_col(tid, j) < N) mx[(j >> 1) & 1] = fmaxf(mx[(j >> 1) & 1], alpha * acc[0][j]);
            float sum[2] = {0.f, 0.f}, m2[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
                mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
                m2[h] = -mx[h] * 1.4426950408889634f;
            }
            const float a2 = alpha * 1.4426950408889634f;
#pragma unroll
            for (int j = 0; j < BN / 2; ++j) {
                const float e = (n0 + frag_col(tid, j) < N) ? ex2_approx(fmaf(a2, acc[0][j], m2[(j >> 1) & 1])) : 0.f;
                acc[0][j] = e;
                sum[(j >> 1) & 1] += e;
            }
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 1);
                sum[h] += __shfl_xor_sync(0xffffffffu, sum[h], 2);
                sum[h] = 1.0f / sum[h];
            }
#pragma unroll
            for (int j = 0; j < BN / 2; j += 2) {
                const int r = m0 + frag_row(tid, j), col = n0 + frag_col(tid, j);
                if (r >= N || col >= ncols) continue;
                const float inv = sum[(j >> 1) & 1];
                *reinterpret_cast<float2*>(out + ((long long)bh * N + r) * ld_out + col) = make_float2(acc[0][j] * inv, acc[0][j + 1] * inv);
            }
        } else {
        // E of the whole fragment is loaded before the first store, so that its loads are in flight together (out may alias E)
        float2 ef[BN / 4];
#pragma unroll
        for (int j = 0; j < BN / 2; j += 2) {
            const int r = m0 + frag_row(tid, j), col = n0 + frag_col(tid, j);
            ef[j / 2] = (EPI != AT_STORE && r < N && col < ncols)
                            ? *reinterpret_cast<const float2*>(E + ((long long)bh * N + r) * ld_out + col) : make_float2(0.f, 0.f);
        }
#pragma unroll
        for (int j = 0; j < BN / 2; j += 2) {
            const int r = m0 + frag_row(tid, j), col = n0 + frag_col(tid, j);
            if (r >= N || col >= ncols) continue;
            const long long off = ((long long)bh * N + r) * ld_out + col;
            const float2 e = ef[j / 2];
            float v[2] = {alpha * acc[0][j], alpha * acc[0][j + 1]};
            const float ee[2] = {e.x, e.y};
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                if (EPI == AT_MUL) v[u] *= ee[u];
                else if (EPI == AT_SD) v[u] = te_sd_fast(ee[u], v[u]);
                if (col + u >= N) v[u] = 0.f;
            }
            *reinterpret_cast<float2*>(out + off) = make_float2(v[0], v[1]);
        }
        }
    }
};

// ---- token-reduced N x d contraction: out[b, m, h*BN + d] = epi(alpha * sum_k A_h[m,k] X[b, k, h*BN + d]) ----------------
//   AMN 0: A_h[m,k] = map[bh][m][k] (K-major) ; AMN 1: A_h[m,k] = map[bh][k][m] (MN-major, transposed in shared memory)
//   X is MN-major (transposed in shared memory).  a_shared: A indexed by the batch only (dense rollout product, "heads" =
//   column tiles).
// The map is a 3-D tensor map of inner extent N (not NP) at row stride NP, so keys and rows >= N land as zeros in every bh
// and the pad columns are never read; X is one over [batch, N, ld] of inner extent n_pad: tokens >= N and columns >= n_pad
// land as zeros.  The MN-major sources land as 32 x 32 boxes behind the tiles (Stage::land: A's four boxes when AMN, then
// X's BN / 32).
template <int AMN, int EPI, bool SP, int BN_>
struct NkProb : NoScale {
    static constexpr int BN = BN_, CHUNK = SP ? 0 : 4, FMT = OP_TF32;
    using PRODS = std::conditional_t<SP, One, Split3>;
    static constexpr int LAND_A = AMN ? BM * 128 : 0, LAND_X = BN * 128;
    using L = Stage<PRODS, BN, LAND_A + LAND_X>;
    static constexpr bool TMA = true;
    static constexpr int FIX = FIX_AB, EPI_MAPS = 0;
    int N, H, NP, ld_out, n_out, n_pad, a_shared, batch;
    const float* map; const float* X; long long ldx;
    const float* rowscale; const float* E; float* out; float alpha;
    __device__ int kblocks() const { return (N + 31) / 32; }
    static constexpr int NMAPS = 2;
    TmaTile tile(int i) const {
        if (i == 0) return TmaTile{map, N, N, NP, AMN ? 32 : BM, (long long)batch * (a_shared ? 1 : H), (long long)N * NP};
        return TmaTile{X, N, n_pad, ldx, 32, batch, (long long)N * ldx};
    }
    __device__ void produce(const TmaArgs& ta, uint32_t st, uint32_t bar, int kb, int m0, int, int bh) const {
        const int s = bh / H, h = bh % H, za = a_shared ? s : bh;
        mbar_expect_tx(bar, (AMN ? LAND_A : TILE128) + LAND_X);
        if (AMN == 0) tma_load3(st + L::a(0), &ta.map[0], kb * 32, m0, za, bar);
#pragma unroll
        for (int j = 0; j < LAND_A / 4096; ++j) tma_load3(st + L::land() + j * 4096, &ta.map[0], m0 + 32 * j, kb * 32, za, bar);
#pragma unroll
        for (int j = 0; j < LAND_X / 4096; ++j)
            tma_load3(st + L::land() + LAND_A + j * 4096, &ta.map[1], h * BN + 32 * j, kb * 32, s, bar);
    }
    __device__ void fix(uint8_t* st, int wg, int tid) const {
        if (AMN) transpose_rows(st + L::land(), 64 * wg, 64, tid & 127, 128, put_tf32<SP>(st + L::a(0), st + L::a(1)));
        else fix_tf32<SP>(st + L::a(0), st + L::a(1), 64 * wg, 64, tid & 127, 128);
        transpose_rows(st + L::land() + LAND_A, 0, BN, tid, 256, put_tf32<SP>(st + L::b(0), st + L::b(1)));
    }
    __device__ void epilogue(float (&acc)[1][BN / 2], int m0, int, int bh, int tid, const uint8_t*) const {
        const int s = bh / H, h = bh % H;
        // E of the whole fragment is loaded before the first store, so that its loads are in flight together (out may alias E)
        float2 ef[BN / 4];
#pragma unroll
        for (int j = 0; j < BN / 2; j += 2) {
            const int m = m0 + frag_row(tid, j), gcol = h * BN + frag_col(tid, j);
            ef[j / 2] = (EPI != AT_STORE && m < N && gcol < n_pad)
                            ? *reinterpret_cast<const float2*>(E + ((long long)s * N + m) * ld_out + gcol) : make_float2(0.f, 0.f);
        }
#pragma unroll
        for (int j = 0; j < BN / 2; j += 2) {
            const int m = m0 + frag_row(tid, j), gcol = h * BN + frag_col(tid, j);
            if (m >= N || gcol >= n_pad) continue;
            const long long off = ((long long)s * N + m) * ld_out + gcol;
            float v[2] = {alpha * acc[0][j], alpha * acc[0][j + 1]};
            const float2 e = ef[j / 2];
            if (EPI == AT_MUL) {
                v[0] *= e.x; v[1] *= e.y;
            } else if (EPI == AT_RESID) {
                // the identity's share of the rollout step, added in fp32: out = A J + diag(rowscale) J
                const float rsc = rowscale ? rowscale[(long long)s * N + m] : 1.f;
                v[0] += rsc * e.x; v[1] += rsc * e.y;
            }
            if (gcol >= n_out) v[0] = 0.f;
            if (gcol + 1 >= n_out) v[1] = 0.f;
            *reinterpret_cast<float2*>(out + off) = make_float2(v[0], v[1]);
        }
    }
};

// ---- launch ---------------------------------------------------------------------------------------------------------
inline bool a16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

int sm_count() {
    static int sms[64];
    int dev = 0;
    cudaGetDevice(&dev);
    int& n = sms[dev & 63];
    if (n == 0 && cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) n = 1;
    return n;
}

// cuTensorMapEncodeTiled through the runtime's driver entry point (the library links only the runtime)
using EncodeTiled = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                 const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                 CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiled encode_tiled() {
    static const EncodeTiled fn = [] {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            return (EncodeTiled) nullptr;
        return (EncodeTiled)f;
    }();
    return fn;
}
// The map of a source: boxes of 128 bytes (one swizzled row) x box_rows rows (x 1 matrix), 128-byte swizzle (the layout swz()
// and sdesc() describe), rows, columns and matrices past the source filled with zeros.  TMA needs a 16-byte-aligned base and
// strides that are multiples of 16 bytes.
bool encode_tile(CUtensorMap* map, const TmaTile& t, int esize) {
    const EncodeTiled fn = encode_tiled();
    const int rank = t.count > 0 ? 3 : 2;
    if (!fn || ((uintptr_t)t.base & 15u) || (t.ld * esize) % 16 != 0 || (t.cstride * esize) % 16 != 0 || t.rows < 1 || t.cols < 1)
        return false;
    const cuuint64_t dims[3] = {(cuuint64_t)t.cols, (cuuint64_t)t.rows, (cuuint64_t)t.count};
    const cuuint64_t strides[2] = {(cuuint64_t)(t.ld * esize), (cuuint64_t)(t.cstride * esize)};
    const cuuint32_t box[3] = {(cuuint32_t)(128 / esize), (cuuint32_t)t.box_rows, 1}, estr[3] = {1, 1, 1};
    return fn(map, esize == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_UINT16, rank, const_cast<void*>(t.base),
              dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// grid: (m-tiles, column tiles, batches).
// P::TMA problems run min(tiles, SMs) persistent CTAs of 384 threads that walk the tiles batch-major, then column-fastest
// (tma_tiles).
// The others run one CTA of 256 threads per tile.  P::COL_FAST problems are launched with the column tile in blockIdx.x,
// so that consecutively scheduled CTAs share an A panel and the panel is read from HBM about once instead of once per
// column tile; the weights, at most a few tens of MB, stay in L2.  More than 65535 m-tiles do not fit in grid.y: those
// launches keep the m-tile in blockIdx.x, which is why the order is a kernel argument.  The tiles and their arithmetic do
// not change.
template <class P>
int launch(const P& p, dim3 grid, cudaStream_t st) {
    TmaArgs ta;
    memset(&ta, 0, sizeof(ta));
    int col_fast = 0, threads = NTHREADS, smem = 2 * P::L::BYTES + 1024;
    if constexpr (P::TMA) {
        constexpr int ESIZE = P::FMT == OP_TF32 ? 4 : 2;
        static_assert(P::NMAPS + P::EPI_MAPS <= TMA_MAPS, "TmaArgs holds TMA_MAPS tensor maps");
        for (int i = 0; i < P::NMAPS + P::EPI_MAPS; ++i)        // the epilogue operands are fp32
            if (!encode_tile(&ta.map[i], p.tile(i), i < P::NMAPS ? ESIZE : 4)) {
                te_set_last_error("te_tc: cannot encode a TMA tensor map (16-byte-aligned base and strides required)");
                return TE_ERR_ARG;
            }
        const long long tiles = (long long)grid.x * grid.y * grid.z;
        if (tiles > INT32_MAX) { te_set_last_error("te_tc: grid too large for one launch"); return TE_ERR_ARG; }
        ta.mtiles = (int)grid.x;
        ta.ntiles = (int)grid.y;
        ta.nz = (int)grid.z;
        grid = dim3((unsigned)std::min<long long>(tiles, sm_count()));
        threads = NTHREADS_TMA;
        smem = tma_stages(P::L::BYTES, epi_bytes<P>()) * P::L::BYTES + epi_bytes<P>() + 1024;
    } else {
        col_fast = P::COL_FAST && grid.x <= 65535;
        if (col_fast) grid = dim3(grid.y, grid.x, grid.z);
    }
    // cudaFuncAttributeMaxDynamicSharedMemorySize is per device: one bit per device ordinal
    static unsigned long long done = 0;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { te_set_last_error("te_tc: cudaGetDevice failed"); return TE_ERR_CUDA; }
    if (!(done & (1ull << (dev & 63)))) {
        if (cudaFuncSetAttribute(wg_kernel<P>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) {
            te_set_last_error("te_tc: cannot raise dynamic shared memory");
            return TE_ERR_CUDA;
        }
        done |= 1ull << (dev & 63);
    }
    if (grid.y > 65535 || grid.z > 65535) { te_set_last_error("te_tc: grid too large for one launch"); return TE_ERR_ARG; }
    wg_kernel<P><<<grid, threads, smem, st>>>(p, ta, col_fast);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}
inline unsigned mtiles(long long M) { return (unsigned)((M + BM - 1) / BM); }

// ---- weight preparation: W [out,in] -> the derived operand copies of te_gemm_tc.h ------------------------------------
__global__ void prepare_weights_kernel(const float* __restrict__ w, float* __restrict__ d, int out_f, int in_f) {
    const TeDerived<float> dv(d, in_f, out_f);
    __shared__ float tile[32][33];
    const int bx = blockIdx.x * 32, by = blockIdx.y * 32;      // bx: in index, by: out index
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int o = by + i, c = bx + threadIdx.x;
        float v = 0.f;
        if (o < out_f && c < in_f) {
            const long long idx = (long long)o * in_f + c;
            v = w[idx];
            dv.wp[idx] = to_tf32(fmaxf(v, 0.f));
            dv.wn[idx] = to_tf32(fminf(v, 0.f));
            const float hi = to_tf32(v);
            dv.wh[idx] = hi;
            dv.wl[idx] = to_tf32(v - hi);
            dv.wabs[idx] = to_tf32(fabsf(v));
            dv.bf_wabs[idx] = __float2bfloat16_rn(fabsf(v));
        }
        tile[i][threadIdx.x] = v;
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = bx + i, o = by + threadIdx.x;
        if (o < out_f && c < in_f) {
            const float v = tile[threadIdx.x][i];
            const long long idx = (long long)c * out_f + o;
            dv.wpt[idx] = to_tf32(fmaxf(v, 0.f));
            dv.wnt[idx] = to_tf32(fminf(v, 0.f));
            dv.bf_wpt[idx] = __float2bfloat16_rn(fmaxf(v, 0.f));
            dv.bf_wnt[idx] = __float2bfloat16_rn(fminf(v, 0.f));
            const float hi = to_tf32(v);
            dv.wth[idx] = hi;
            dv.wtl[idx] = to_tf32(v - hi);
        }
    }
}

// ---- fp16 split pre-passes ------------------------------------------------------------------------------------------
// Activations: one warp per row, one scale block per warp iteration (128 columns): single pass, one read of x.
__global__ void __launch_bounds__(256) blocksplit_f16_kernel(const float* __restrict__ x, long long ldx, long long rows, int cols,
                                                             __half* __restrict__ hi, __half* __restrict__ lo,
                                                             float* __restrict__ inv) {
    const int lane = threadIdx.x & 31;
    const long long wpb = blockDim.x >> 5;
    const int nblk = (cols + 127) / 128;
    for (long long row = blockIdx.x * wpb + (threadIdx.x >> 5); row < rows; row += (long long)gridDim.x * wpb) {
        const float* xr = x + row * ldx;
#pragma unroll 2
        for (int base = 0; base < cols; base += 128) {
            const int i = base + lane * 4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (i < cols) v = *reinterpret_cast<const float4*>(xr + i);
            float s, si;
            te_f16_block_scale(te_warp_max(te_absmax4(v)), s, si);
            if (i < cols) {
                uint2 h, l;
                te_f16_split4(v, s, h, l);
                *reinterpret_cast<uint2*>(hi + row * cols + i) = h;
                if (lo) *reinterpret_cast<uint2*>(lo + row * cols + i) = l;
            }
            if (lane == 0) inv[row * nblk + base / 128] = si;
        }
    }
}
// Weights: one scale per row of W (two passes over the row; the second hits L1 / L2).
__global__ void __launch_bounds__(256) rowsplit_f16_kernel(const float* __restrict__ x, long long ldx, long long rows, int cols4,
                                                           __half* __restrict__ hi, __half* __restrict__ lo,
                                                           float* __restrict__ inv) {
    const int lane = threadIdx.x & 31;
    const long long wpb = blockDim.x >> 5;
    for (long long row = blockIdx.x * wpb + (threadIdx.x >> 5); row < rows; row += (long long)gridDim.x * wpb) {
        const float4* xr = reinterpret_cast<const float4*>(x + row * ldx);
        float m = 0.f;
#pragma unroll 4
        for (int c = lane; c < cols4; c += 32) m = fmaxf(m, te_absmax4(xr[c]));
        float s, si;
        te_f16_block_scale(te_warp_max(m), s, si);
        uint2* hr = reinterpret_cast<uint2*>(hi + row * (long long)cols4 * 4);
        uint2* lr = reinterpret_cast<uint2*>(lo + row * (long long)cols4 * 4);
#pragma unroll 4
        for (int c = lane; c < cols4; c += 32) {
            uint2 h, l;
            te_f16_split4(xr[c], s, h, l);
            hr[c] = h;
            if (lo) lr[c] = l;
        }
        if (lane == 0) inv[row] = si;
    }
}
// |x| as bf16: the A operand of the bf16 single-pass S kernel.  x rows at stride ldx -> compact [rows, cols].
__global__ void abs_bf16_kernel(const float* __restrict__ x, long long ldx, __nv_bfloat16* __restrict__ out, long long rows, int cols4) {
    const long long total = rows * cols4;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const long long r = t / cols4;
        const int c = (int)(t - r * cols4);
        const float4 v = *reinterpret_cast<const float4*>(x + r * ldx + 4 * c);
        const __nv_bfloat162 a = __floats2bfloat162_rn(fabsf(v.x), fabsf(v.y)), b = __floats2bfloat162_rn(fabsf(v.z), fabsf(v.w));
        uint2 pk;
        pk.x = *reinterpret_cast<const uint32_t*>(&a);
        pk.y = *reinterpret_cast<const uint32_t*>(&b);
        *reinterpret_cast<uint2*>(out + t * 4) = pk;
    }
}
// grid of a grid-stride elementwise pass: at most 16 blocks per SM
unsigned stride_blocks(long long work, int per_block) {
    long long b = (work + per_block - 1) / per_block;
    const long long cap = (long long)sm_count() * 16;
    if (b > cap) b = cap;
    return (unsigned)(b < 1 ? 1 : b);
}

// The Linear GEMM of one operand form with the epilogue epi: the forward epilogues (STORE, BIAS, BIAS_GELU, BIAS_ADD,
// BIAS_QUICK_GELU) when FWD, else the backward ones (STORE, GELU_BWD, QUICK_GELU_BWD).  C [rows, N] = epi(A B^T); bias / e0 /
// y2 as in te_gemm_tc.h.
template <int EPI, int FORM>
int lin_launch(const LinArgs& args, cudaStream_t st) {
    using P = LinProb<EPI, FORM>;
    P p;
    static_cast<LinArgs&>(p) = args;
    return launch(p, dim3(mtiles(args.o.M), (args.o.N + P::BN - 1) / P::BN), st);
}
template <int FORM, bool FWD>
int linear(int K, const void* a, const void* a_lo, long long lda, const void* b, const void* b_lo, const float* rs,
           const float* cs, long long rows, int N, const float* bias, const float* e0, float* y, float* y2, int epi,
           const char* who, cudaStream_t st) {
    LinArgs g;
    g.K = K; g.a = a; g.a_lo = a_lo; g.lda = lda; g.b = b; g.b_lo = b_lo; g.rs = rs; g.rs_ld = (K + 127) / 128; g.cs = cs;
    g.o.M = (int)rows; g.o.N = N; g.o.bias = bias; g.o.E = e0; g.o.lde = N; g.o.C = y; g.o.ldc = N; g.o.C2 = y2; g.o.ldc2 = N;
    switch (epi) {
        case TE_TC_EPI_STORE: return lin_launch<TE_TC_EPI_STORE, FORM>(g, st);
        case TE_TC_EPI_BIAS: if constexpr (FWD) return lin_launch<TE_TC_EPI_BIAS, FORM>(g, st); break;
        case TE_TC_EPI_BIAS_GELU: if constexpr (FWD) return lin_launch<TE_TC_EPI_BIAS_GELU, FORM>(g, st); break;
        case TE_TC_EPI_BIAS_ADD: if constexpr (FWD) return lin_launch<TE_TC_EPI_BIAS_ADD, FORM>(g, st); break;
        case TE_TC_EPI_GELU_BWD: if constexpr (!FWD) return lin_launch<TE_TC_EPI_GELU_BWD, FORM>(g, st); break;
        case TE_TC_EPI_BIAS_QUICK_GELU: if constexpr (FWD) return lin_launch<TE_TC_EPI_BIAS_QUICK_GELU, FORM>(g, st); break;
        case TE_TC_EPI_QUICK_GELU_BWD: if constexpr (!FWD) return lin_launch<TE_TC_EPI_QUICK_GELU_BWD, FORM>(g, st); break;
    }
    te_set_last_error((std::string(who) + ": unsupported epilogue").c_str());
    return TE_ERR_UNSUPPORTED;
}

// S = sd(R, Z) [rows, out] on the z+ S kernel.  Single-pass: wa = |W| (xabs = bf16(|x|) with BF); two-pass: wa / wb = W+ / W-.
// hs: block scales of the ZO_F16S output.
template <bool SINGLE, bool BF, int OUT>
int zs(const float* x, long long ldx, const void* xabs, const void* wa, const void* wb, const float* r, long long ldr,
       const float* y, long long ldy, const float* bias, void* out, float* hs, long long rows, int in_features, int out_features,
       cudaStream_t st, float s_scale, bool inh) {
    ZsProb<SINGLE, BF, OUT> p;
    p.M = (int)rows; p.N = out_features; p.K = in_features;
    p.x = x; p.ldx = ldx; p.xabs = xabs; p.wa = wa; p.wb = wb;
    p.r = r; p.ldr = ldr; p.y = y; p.ldy = ldy; p.bias = bias;
    p.out = out; p.ldo = out_features; p.hs = hs;
    p.sscale = s_scale; p.zsign = inh ? -1.f : 1.f;
    return launch(p, dim3(mtiles(p.M), p.N / 128), st);
}

}  // namespace

// =====================================================================================================================
// public entry points (te_gemm_tc.h)
// =====================================================================================================================
long long te_tc_derived_floats(int in_features, int out_features) { return TeDerived<float>::floats(in_features, out_features); }

int te_tc_prepare_weights(const float* w, float* derived, int in_features, int out_features, cudaStream_t st) {
    dim3 grid((in_features + 31) / 32, (out_features + 31) / 32), block(32, 8);
    prepare_weights_kernel<<<grid, block, 0, st>>>(w, derived, out_features, in_features);
    TE_CUDA_CHECK_LAUNCH();
    const TeDerived<float> dv(derived, in_features, out_features);
    if (in_features % 8 == 0 && in_features >= 8 && a16(w))        // row-scaled fp16 split of W
        TE_TRY(te_tc_rowsplit_f16(w, in_features, out_features, in_features, dv.h_w, dv.l_w, dv.s_w, st));
    if (out_features % 8 == 0 && in_features >= 2) {               // single-pass fp16 operands from the TF32-rounded transposes [in, out]
        TE_TRY(te_tc_rowsplit_f16(dv.wth, out_features, in_features, out_features, dv.h_wt, nullptr, dv.s_wt, st));
        TE_TRY(te_tc_rowsplit_f16(dv.wpt, out_features, in_features, out_features, dv.h_wpt, nullptr, dv.s_wpt, st));
        TE_TRY(te_tc_rowsplit_f16(dv.wnt, out_features, in_features, out_features, dv.h_wnt, nullptr, dv.s_wnt, st));
    }
    return TE_OK;
}

int te_tc_rowsplit_f16(const float* x, long long ldx, long long rows, int cols, void* hi, void* lo, float* scale_inv,
                       cudaStream_t st) {
    if (cols % 4 != 0 || ldx % 4 != 0 || !a16(x) || ((uintptr_t)hi & 7u) || (lo && ((uintptr_t)lo & 7u))) {
        te_set_last_error("te_tc_rowsplit_f16: alignment");
        return TE_ERR_ARG;
    }
    rowsplit_f16_kernel<<<stride_blocks(rows, 8), 256, 0, st>>>(x, ldx, rows, cols / 4, reinterpret_cast<__half*>(hi),
                                                                reinterpret_cast<__half*>(lo), scale_inv);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}

int te_tc_blocksplit_f16(const float* x, long long ldx, long long rows, int cols, float* split, float* scale_inv, cudaStream_t st,
                         bool hi_only) {
    if (cols % 4 != 0 || ldx % 4 != 0 || !a16(x) || !a16(split) || !scale_inv) {
        te_set_last_error("te_tc_blocksplit_f16: alignment");
        return TE_ERR_ARG;
    }
    __half* hi = reinterpret_cast<__half*>(split);
    blocksplit_f16_kernel<<<stride_blocks(rows, 8), 256, 0, st>>>(x, ldx, rows, cols, hi, hi_only ? nullptr : hi + rows * cols,
                                                                  scale_inv);
    TE_CUDA_CHECK_LAUNCH();
    return TE_OK;
}

// ---- z+ rule --------------------------------------------------------------------------------------------------------
bool te_tc_zplus_supported(long long rows, int in_features, int out_features, long long ldx) {
    return rows > 0 && rows < (1LL << 31) && in_features % 128 == 0 && out_features % 128 == 0 && ldx % 4 == 0;
}
int te_tc_zplus_s1(const float* x, long long ldx, float* xabs, const float* derived, const float* r, long long ldr,
                   const float* y, long long ldy, const float* bias, float* s_out, long long rows, int in_features,
                   int out_features, cudaStream_t st, bool bf16, float* s16, float* s16_scale, float s_scale, bool inh) {
    const TeDerived<const float> dv(derived, in_features, out_features);
    if (ldx % 4 != 0 || !a16(x) || !a16(r) || !a16(y) || ldr % 4 != 0 || ldy % 4 != 0) {   // R, y: TMA-encodable
        te_set_last_error("te_tc_zplus_s1: alignment");
        return TE_ERR_ARG;
    }
    void* o = s16 ? (void*)s16 : (void*)s_out;
    auto run = [&](auto zs_fn, const void* wa) {
        return zs_fn(x, ldx, xabs, wa, nullptr, r, ldr, y, ldy, bias, o, s16_scale, rows, in_features, out_features, st, s_scale,
                     inh);
    };
    if (bf16 && in_features % 64 == 0) {
        if (!a16(xabs)) { te_set_last_error("te_tc_zplus_s1: alignment"); return TE_ERR_ARG; }
        abs_bf16_kernel<<<stride_blocks(rows * (in_features / 4), 256), 256, 0, st>>>(
            x, ldx, reinterpret_cast<__nv_bfloat16*>(xabs), rows, in_features / 4);
        TE_CUDA_CHECK_LAUNCH();
        return s16 ? run(zs<true, true, ZO_F16S>, dv.bf_wabs) : run(zs<true, true, ZO_F32>, dv.bf_wabs);
    }
    return s16 ? run(zs<true, false, ZO_F16S>, dv.wabs) : run(zs<true, false, ZO_F32>, dv.wabs);
}

int te_tc_zplus_r(const float* s, const float* derived, const float* x, long long ldx, float* out, long long ld_out,
                  long long rows, int in_features, int out_features, cudaStream_t st, bool inh) {
    const TeDerived<const float> dv(derived, in_features, out_features);
    ZrProb<0> p;
    memset(&p, 0, sizeof(p));
    p.M = (int)rows; p.N = in_features; p.K = out_features;
    p.s = s; p.wp = inh ? dv.wnt : dv.wpt; p.wn = inh ? dv.wpt : dv.wnt; p.x = x; p.ldx = ldx; p.out = out; p.ldo = ld_out;
    p.accum = inh;
    return launch(p, dim3(mtiles(rows), in_features / 128), st);
}

int te_tc_zplus_r16(const float* s, float* split, float* scale, const float* derived, const float* x, long long ldx, float* out,
                    long long ld_out, long long rows, int in_features, int out_features, cudaStream_t st, bool inh) {
    const TeDerived<const float> dv(derived, in_features, out_features);
    if (!a16(split) || !scale || !a16(derived) || !a16(x) || !a16(out) || ldx % 4 != 0 || ld_out % 4 != 0) {
        te_set_last_error("te_tc_zplus_r16: bad operands");
        return TE_ERR_ARG;
    }
    if (s) TE_TRY(te_tc_blocksplit_f16(s, out_features, rows, out_features, split, scale, st, true));
    ZrProb<2> p;
    p.M = (int)rows; p.N = in_features; p.K = out_features;
    p.s = split; p.wp = inh ? dv.h_wnt : dv.h_wpt; p.wn = inh ? dv.h_wpt : dv.h_wnt;
    p.rs = scale; p.rs_ld = (out_features + 127) / 128; p.cp = inh ? dv.s_wnt : dv.s_wpt; p.cn = inh ? dv.s_wpt : dv.s_wnt;
    p.x = x; p.ldx = ldx; p.out = out; p.ldo = ld_out; p.accum = inh;
    return launch(p, dim3(mtiles(rows), in_features / 64), st);
}

namespace {
// One half of the z+ / alpha-beta rule: S = s_scale * sd(R, Z) into s_scratch, then out = x+ (S W+) + x- (S W-); the inhibitor
// half (inh) swaps the weight signs in both contractions and adds into out.
int zplus_half(const float* x, long long ldx, const float* derived, const float* r, long long ldr, float* out, float* s_scratch,
               long long rows, int in_features, int out_features, cudaStream_t st, const float* y, long long ldy,
               const float* bias, ZplusVariant zv, long long ld_out, float* xabs, float s_scale, bool inh) {
    const TeDerived<const float> dv(derived, in_features, out_features);
    const bool single = y && a16(y) && ldy % 4 == 0 && (!bias || a16(bias));
    const bool rb = zv.r_bf16 && (out_features % 64 == 0);          // S as bf16, R kernel with bf16 operands
    if (!rb && single && xabs && a16(xabs)) {
        if (zv.r_f16 && te_tc_fwd16_supported(rows, out_features, in_features, out_features)) {
            // second contraction on block-scaled fp16: S leaves the S kernel in that format, straight into s_scratch
            // ([rows, out] fp16, then the [rows, out/128] scales: rows*out floats hold both)
            float* s16_scale = s_scratch + ((rows * out_features / 2 + 63) & ~63LL);
            TE_TRY(te_tc_zplus_s1(x, ldx, xabs, derived, r, ldr, y, ldy, bias, nullptr, rows, in_features, out_features, st,
                                  zv.s1_bf16, s_scratch, s16_scale, s_scale, inh));
            return te_tc_zplus_r16(nullptr, s_scratch, s16_scale, derived, x, ldx, out, ld_out, rows, in_features, out_features, st,
                                   inh);
        }
        TE_TRY(te_tc_zplus_s1(x, ldx, xabs, derived, r, ldr, y, ldy, bias, s_scratch, rows, in_features, out_features, st,
                              zv.s1_bf16, nullptr, nullptr, s_scale, inh));
        return te_tc_zplus_r(s_scratch, derived, x, ldx, out, ld_out, rows, in_features, out_features, st, inh);
    }
    // S = s_scale * sd(R, Z) [rows, out]: single-pass from y, or two-pass
    auto run = [&](auto zs_fn) {
        return single ? zs_fn(x, ldx, nullptr, dv.wabs, nullptr, r, ldr, y, ldy, bias, s_scratch, nullptr, rows,
                              in_features, out_features, st, s_scale, inh)
                      : zs_fn(x, ldx, nullptr, inh ? dv.wn : dv.wp, inh ? dv.wp : dv.wn, r, ldr, nullptr, 0, nullptr, s_scratch,
                              nullptr, rows, in_features, out_features, st, s_scale, inh);
    };
    if (single) TE_TRY(rb ? run(zs<true, false, ZO_BF16>) : run(zs<true, false, ZO_F32>));
    else TE_TRY(rb ? run(zs<false, false, ZO_BF16>) : run(zs<false, false, ZO_F32>));
    if (rb) {
        ZrProb<1> p;
        memset(&p, 0, sizeof(p));
        p.M = (int)rows; p.N = in_features; p.K = out_features;
        p.s = s_scratch; p.wp = inh ? dv.bf_wnt : dv.bf_wpt; p.wn = inh ? dv.bf_wpt : dv.bf_wnt;
        p.x = x; p.ldx = ldx; p.out = out; p.ldo = ld_out; p.accum = inh;
        return launch(p, dim3(mtiles(rows), in_features / 128), st);
    }
    return te_tc_zplus_r(s_scratch, derived, x, ldx, out, ld_out, rows, in_features, out_features, st, inh);
}
}  // namespace

int te_tc_zplus_linear_relprop(const float* x, long long ldx, const float* derived, const float* r, long long ldr,
                               float* out, float* s_scratch, long long rows, int in_features, int out_features, cudaStream_t st,
                               const float* y, long long ldy, const float* bias, ZplusVariant zv, long long ld_out, float* xabs,
                               float alpha) {
    if (ld_out == 0) ld_out = in_features;
    if (!a16(x) || !a16(derived) || !a16(r) || !a16(out) || !a16(s_scratch)) {
        te_set_last_error("te_gemm_tc: operands must be 16-byte aligned");
        return TE_ERR_ARG;
    }
    // activator (alpha = 1: the z+ rule, S unscaled), then for beta != 0 the inhibitor through the same S buffer
    const float beta = alpha - 1.f;
    TE_TRY(zplus_half(x, ldx, derived, r, ldr, out, s_scratch, rows, in_features, out_features, st, y, ldy, bias, zv, ld_out, xabs,
                      alpha, false));
    if (beta == 0.f) return TE_OK;
    return zplus_half(x, ldx, derived, r, ldr, out, s_scratch, rows, in_features, out_features, st, y, ldy, bias, zv, ld_out, xabs,
                      -beta, true);
}

namespace {
// one product of the layers_lrp rule: x+ (NEG false) or x- (NEG true) with the weight w (w [out, in], wt its transpose);
// S = s_scale * sd(R, x+- w^T), out (+)= x+- * (S w)
template <bool NEG>
int lrp_half(const float* x, long long ldx, const float* w, const float* wt, const float* r, long long ldr, float* out,
             long long ld_out, float* s, long long rows, int in_features, int out_features, cudaStream_t st, float s_scale,
             bool accum) {
    LrpSProb<NEG> ps;
    ps.M = (int)rows; ps.N = out_features; ps.K = in_features;
    ps.x = x; ps.ldx = ldx; ps.w = w; ps.r = r; ps.ldr = ldr; ps.out = s; ps.sscale = s_scale;
    TE_TRY(launch(ps, dim3(mtiles(rows), out_features / 128), st));
    LrpRProb<NEG> pr;
    pr.M = (int)rows; pr.N = in_features; pr.K = out_features;
    pr.s = s; pr.wt = wt; pr.x = x; pr.ldx = ldx; pr.out = out; pr.ldo = ld_out; pr.accum = accum;
    return launch(pr, dim3(mtiles(rows), in_features / 128), st);
}
}  // namespace

int te_tc_lrp_linear_relprop(const float* x, long long ldx, const float* derived, const float* r, long long ldr, float* out,
                             long long ld_out, float* s_scratch, long long rows, int in_features, int out_features,
                             cudaStream_t st, float alpha) {
    if (!a16(x) || !a16(derived) || !a16(r) || !a16(out) || !a16(s_scratch) || ldx % 4 != 0 || ldr % 4 != 0 || ld_out % 4 != 0) {
        te_set_last_error("te_tc_lrp_linear_relprop: operands must be 16-byte aligned");
        return TE_ERR_ARG;
    }
    const TeDerived<const float> dv(derived, in_features, out_features);
    // the products in sequence through the one S buffer: x+ W+ first (writes out), then x- W- (adds to it); for beta != 0
    // the inhibitor's x+ W-, x- W+ add to it as well, S scaled by alpha for the activator and -beta for the inhibitor
    const float beta = alpha - 1.f;
    TE_TRY(lrp_half<false>(x, ldx, dv.wp, dv.wpt, r, ldr, out, ld_out, s_scratch, rows, in_features, out_features, st, alpha, false));
    TE_TRY(lrp_half<true>(x, ldx, dv.wn, dv.wnt, r, ldr, out, ld_out, s_scratch, rows, in_features, out_features, st, alpha, true));
    if (beta == 0.f) return TE_OK;
    TE_TRY(lrp_half<false>(x, ldx, dv.wn, dv.wnt, r, ldr, out, ld_out, s_scratch, rows, in_features, out_features, st, -beta, true));
    return lrp_half<true>(x, ldx, dv.wp, dv.wpt, r, ldr, out, ld_out, s_scratch, rows, in_features, out_features, st, -beta, true);
}

// ---- Linear GEMMs ---------------------------------------------------------------------------------------------------
bool te_tc_gemm3x_supported(long long rows, int K, int N, long long lda) {
    return rows > 0 && rows < (1LL << 31) && K % 32 == 0 && N % 128 == 0 && lda % 4 == 0;
}

int te_tc_linear_fwd(const float* x, long long ldx, const float* derived, int in_features, int out_features, const float* bias,
                     float* y, float* y2, const float* e0, long long rows, int epi, cudaStream_t st) {
    if (!a16(x) || !a16(derived) || !a16(y) || (y2 && !a16(y2)) || (e0 && !a16(e0)) || (bias && !a16(bias))) {
        te_set_last_error("te_tc_linear_fwd: operands must be 16-byte aligned");
        return TE_ERR_ARG;
    }
    const TeDerived<const float> dv(derived, in_features, out_features);
    return linear<LIN_3XTF32, true>(in_features, x, nullptr, ldx, dv.wh, dv.wl, nullptr, nullptr, rows, out_features, bias, e0, y,
                                    y2, epi, "te_tc_linear_fwd", st);
}

int te_tc_linear_bwd(const float* dy, const float* derived, int in_features, int out_features, float* dx, const float* e0,
                     long long rows, int epi, cudaStream_t st) {
    if (!a16(dy) || !a16(derived) || !a16(dx) || (e0 && !a16(e0))) {
        te_set_last_error("te_tc_linear_bwd: operands must be 16-byte aligned");
        return TE_ERR_ARG;
    }
    const TeDerived<const float> dv(derived, in_features, out_features);
    return linear<LIN_3XTF32, false>(out_features, dy, nullptr, out_features, dv.wth, dv.wtl, nullptr, nullptr, rows, in_features,
                                     nullptr, e0, dx, nullptr, epi, "te_tc_linear_bwd", st);
}

int te_tc_linear_bwd_tf32(const float* dy, long long lddy, const float* derived, int in_features, int out_features, float* dx,
                          const float* e0, long long rows, int epi, cudaStream_t st) {
    if (!a16(dy) || lddy % 4 != 0 || !a16(derived) || !a16(dx) || (e0 && !a16(e0))) {
        te_set_last_error("te_tc_linear_bwd_tf32: operands must be 16-byte aligned");
        return TE_ERR_ARG;
    }
    const TeDerived<const float> dv(derived, in_features, out_features);
    return linear<LIN_TF32, false>(out_features, dy, nullptr, lddy, dv.wth, nullptr, nullptr, nullptr, rows, in_features, nullptr,
                                   e0, dx, nullptr, epi, "te_tc_linear_bwd_tf32", st);
}

bool te_tc_fwd16_supported(long long rows, int K, int N, long long lda) {
    return rows > 0 && rows < (1LL << 31) && K % 64 == 0 && N % 128 == 0 && lda % 4 == 0;
}

int te_tc_linear_fwd16(const float* x, long long ldx, float* split, float* scale, const float* derived, int in_features,
                       int out_features, const float* bias, float* y, float* y2, const float* e0, long long rows, int epi,
                       cudaStream_t st, float* split_out, float* scale_out) {
    if (!a16(split) || !scale || !a16(derived) || !a16(y) || (y2 && !a16(y2)) || (e0 && !a16(e0)) || (bias && !a16(bias)) ||
        (split_out && (!a16(split_out) || !scale_out || !y2 || (epi != TE_TC_EPI_BIAS_GELU && epi != TE_TC_EPI_BIAS_QUICK_GELU)))) {
        te_set_last_error("te_tc_linear_fwd16: bad operands");
        return TE_ERR_ARG;
    }
    const __half* ah = reinterpret_cast<const __half*>(split);
    const __half* al = ah + rows * in_features;
    if (x) TE_TRY(te_tc_blocksplit_f16(x, ldx, rows, in_features, split, scale, st));
    const TeDerived<const float> dv(derived, in_features, out_features);
    TE_TRY((linear<LIN_F16X3, true>(in_features, ah, al, in_features, dv.h_w, dv.l_w, scale, dv.s_w, rows, out_features, bias, e0,
                                    y, y2, epi, "te_tc_linear_fwd16", st)));
    // the next Linear's A operand (BIAS_GELU / BIAS_QUICK_GELU only): the block-scaled split of y2 = gelu(y) / quick_gelu(y)
    if (split_out) return te_tc_blocksplit_f16(y2, out_features, rows, out_features, split_out, scale_out, st);
    return TE_OK;
}

int te_tc_linear_bwd16(const float* dy, long long lddy, float* split, float* scale, const float* derived, int in_features,
                       int out_features, float* dx, const float* e0, long long rows, int epi, cudaStream_t st) {
    if (!a16(split) || !scale || !a16(derived) || !a16(dx) || (e0 && !a16(e0))) {
        te_set_last_error("te_tc_linear_bwd16: bad operands");
        return TE_ERR_ARG;
    }
    if (dy) TE_TRY(te_tc_blocksplit_f16(dy, lddy, rows, out_features, split, scale, st, true));
    const TeDerived<const float> dv(derived, in_features, out_features);
    return linear<LIN_F16, false>(out_features, split, nullptr, out_features, dv.h_wt, nullptr, scale, dv.s_wt, rows, in_features,
                                  nullptr, e0, dx, nullptr, epi, "te_tc_linear_bwd16", st);
}

// ---- attention-shaped contractions -------------------------------------------------------------------------------------
bool te_tc_attn_supported(int N, int dh, long long lda, long long ldb, int ld_out) {
    return N >= 1 && (dh == 32 || dh == 64) && lda % 4 == 0 && ldb % 4 == 0 && ld_out % 4 == 0;
}
bool te_tc_attn_nk_supported(int N, int dh, int NP, long long ldx, long long ld_out) {
    return N >= 1 && dh == 64 && NP % 4 == 0 && ldx % 4 == 0 && ld_out % 4 == 0;
}
bool te_tc_bmm_nk_supported(int N, int ld) { return N >= 1 && ld % 4 == 0 && ld >= N; }

namespace {
template <int EPI, bool SP, int BN>
int nn(const float* A, long long lda, const float* B, long long ldb, int batch, int H, int N, int dh, float* out, int ld_out,
       const float* E, float alpha, cudaStream_t st) {
    NnProb<EPI, SP, BN> p;
    p.N = N; p.H = H; p.dh = dh; p.ld_out = ld_out; p.batch = batch;
    p.a = A; p.lda = lda; p.b = B; p.ldb = ldb; p.E = E; p.out = out; p.alpha = alpha;
    return launch(p, dim3(mtiles(N), (unsigned)((N + BN - 1) / BN), (unsigned)(batch * H)), st);
}
template <int AMN, int EPI, bool SP, int BN>
int nk(const float* map, int NP, const float* X, long long ldx, int batch, int H, int N, float* out, int ld_out, int n_out,
       int n_pad, int a_shared, const float* rowscale, const float* E, float alpha, cudaStream_t st) {
    NkProb<AMN, EPI, SP, BN> p;
    p.N = N; p.H = H; p.NP = NP; p.ld_out = ld_out; p.n_out = n_out; p.n_pad = n_pad; p.a_shared = a_shared; p.batch = batch;
    p.map = map; p.X = X; p.ldx = ldx; p.rowscale = rowscale; p.E = E; p.out = out; p.alpha = alpha;
    return launch(p, dim3(mtiles(N), 1, (unsigned)(batch * H)), st);
}
}  // namespace

// out[b,h,i,j] = epi(alpha * sum_d A[b*N+i, h*dh+d] * B[b*N+j, h*dh+d]);  out / E are [batch,H,N,ld_out]
int te_tc_attn_nn(const float* A, long long lda, const float* B, long long ldb, int batch, int H, int N, int dh,
                  float* out, int ld_out, const float* E, float alpha, int epi, cudaStream_t st, bool single_pass) {
#define TE_NN(EPI, SP, BN) nn<EPI, SP, BN>(A, lda, B, ldb, batch, H, N, dh, out, ld_out, E, alpha, st)
    if (single_pass && epi == TE_TC_ATTN_STORE) return TE_NN(AT_STORE, true, 128);
    if (single_pass && epi == TE_TC_ATTN_MUL) return TE_NN(AT_MUL, true, 128);
    switch (epi) {
        case TE_TC_ATTN_STORE: return TE_NN(AT_STORE, false, 128);
        case TE_TC_ATTN_MUL: return TE_NN(AT_MUL, false, 128);
        case TE_TC_ATTN_SD: return TE_NN(AT_SD, false, 128);
        case TE_TC_ATTN_SOFTMAX:
            if (N > 256) break;                       // the whole key axis must sit in one tile
            return TE_NN(AT_SOFTMAX, false, 256);
    }
#undef TE_NN
    te_set_last_error("te_gemm_tc: unsupported attention epilogue");
    return TE_ERR_UNSUPPORTED;
}

// out[b, m, h, :] = epi(alpha * sum_k A_h[m,k] X[b,k,h,:]) ; A_h = map[b,h] (amn = 0) or its transpose (amn = 1);
// X, out, E: packed activations [batch, N, ld] (head h at columns h*64..); epi: TE_TC_ATTN_STORE / TE_TC_ATTN_MUL
int te_tc_attn_nk(const float* map, int NP, int amn, const float* X, long long ldx, int batch, int H, int N, float* out,
                  int ld_out, const float* E, float alpha, int epi, cudaStream_t st, bool single_pass) {
#define TE_NK(AMN, EPI, SP) nk<AMN, EPI, SP, 64>(map, NP, X, ldx, batch, H, N, out, ld_out, H * 64, H * 64, 0, nullptr, E, alpha, st)
    if (epi == TE_TC_ATTN_STORE) {
        if (single_pass) return amn ? TE_NK(1, AT_STORE, true) : TE_NK(0, AT_STORE, true);
        return amn ? TE_NK(1, AT_STORE, false) : TE_NK(0, AT_STORE, false);
    }
    if (epi == TE_TC_ATTN_MUL) {
        if (single_pass) return amn ? TE_NK(1, AT_MUL, true) : TE_NK(0, AT_MUL, true);
        return amn ? TE_NK(1, AT_MUL, false) : TE_NK(0, AT_MUL, false);
    }
#undef TE_NK
    te_set_last_error("te_gemm_tc: unsupported attention nk epilogue");
    return TE_ERR_UNSUPPORTED;
}

// One step of the rollout chain in residual form: out[b] = A[b] * J[b] + diag(rowscale[b]) * J[b], all [batch, N, ld]
// (fp32-grade 3xTF32).  The padding columns of out are zeroed so that it can be the next J.
int te_tc_bmm_nk_resid(const float* A, const float* J, const float* rowscale, float* out, int batch, int N, int ld,
                       cudaStream_t st) {
    return nk<0, AT_RESID, false, 128>(A, ld, J, ld, batch, (ld + 127) / 128, N, out, ld, N, ld, 1, rowscale, J, 1.f, st);
}
