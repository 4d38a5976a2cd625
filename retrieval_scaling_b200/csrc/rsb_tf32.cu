// rsb_tf32.cu -- fp32-accurate inner-product scores on the Hopper tensor cores: S[M,N] = A[M,K] . B[N,K]^T with
// A, B fp32, computed as the error-compensated 3xTF32 product
//        A.B ~= Ah.Bh + Ah.Bl + Al.Bh        (x = xh + xl, xh = tf32(x), xl = tf32(x - xh); the dropped Al.Bl term
// is ~2^-22 relative) accumulated in fp32 registers.  Used for Flat search over fp32 rows.
//
// 128 x 128 output tiles, TMA tensor loads (128B swizzle, 32 fp32 = one swizzle row per K step) -> 3-stage
// shared-memory ring of {Ah, Al, Bh, Bl} tiles filled by one producer thread -> two consumer warpgroups that take the
// tiles of a persistent CTA in turn, each issuing 24 wgmma.m64n128k8.tf32 per stage (4 K-slices x 3 products x 2
// row halves) -> epilogue from the accumulator registers while the other warpgroup runs the next tile's MMAs.
//
// fp16 forms (F16 = true).  Each row of an fp32 operand is scaled by a power of two s that puts its largest
// |element| in [2^14, 2^15) (exact), and split into fp16 hi = fp16(x s), lo = fp16(x s - hi) (split_f16_kernel).
// 64 fp16 = one swizzle row per K step, so a stage carries twice the K of the tf32 form in the same 64 KB.
//  * B exact (Flat indexes with fp16 storage): B is the database as stored, so no split copy of it exists; per
//    16-wide K-slice two wgmma.m64n128k16.f16 (lo.B, then hi.B) share the B tile; the epilogue multiplies by
//    inv_a[row] = 1 / s.
//  * B split (the IVF coarse quantizer: queries against the centroids, split once when the index gets them): per
//    16-wide K-slice three wgmma.m64n128k16.f16 in 3xTF32's order, Al.Bh, Ah.Bl, Ah.Bh; the epilogue multiplies by
//    inv_b[col], then inv_a[row] (powers of two: exact unless a product leaves the normal fp32 range).
//    Error per product a b, in scaled units (a = x s of one operand row, b of the other), u = 2^-11 the fp16 unit
//    round-off, d = 2^-25 half the fp16 subnormal spacing: a = Ah + Al + ea with
//      |Al| <= u (1 + u) |a| + d,  |ea| <= u^2 |a| + d      (|a - Ah| <= u |a|; Al rounds that remainder to 11
//                                                             significant bits, or to the subnormal grid below 2^-14)
//      a b - (Ah Bh + Ah Bl + Al Bh) = Al Bl + a eb + ea b - ea eb
//      |a b - (Ah Bh + Ah Bl + Al Bh)| <= (3 u^2 + 2 u^3 + 2 u^4) |a b| + d (1 + u + 2 u^2) (|a| + |b|) + 2 d^2.
//    The relative term is about 3 * 2^-22 (3xTF32: the same 3 u^2 with u = 2^-11); the absolute term is below 2^-39
//    of the row maxima (each row's largest |a| is >= 2^14), so a lo that goes subnormal costs nothing measurable.
//    Each fp16 product is exact in fp32; the accumulators add them in the 3xTF32 form's order.
//    tests/test_coarse_f16_split_cpu.py restates the split and this bound in fp64.
//    Exactness: the coarse stage keeps the top kc = nprobe + 8 of these scores (the fused filter below is exact with
//    respect to them) and re-scores the kc candidates in fp32 (refine_exact_kernel).  A column of the exact top
//    nprobe can only be missed if kc columns score at least as high in S~, so with eps the largest score error of the
//    row (the bound above summed over K, plus the fp32 accumulation) at least 8 columns outside the exact top nprobe
//    come within 2 eps of it: the result is the exact fp32 top nprobe unless the exact scores at ranks
//    nprobe and nprobe + 8 lie within 2 eps -- the same boundary caveat as the 3xTF32 form.
// All forms share the mainloop ring and the epilogues below (score tile, or the fused top-8 candidate + bound filter).
#include "rsb_common.cuh"
#include "rsb_internal.h"
#include "rsb_tc.cuh"

#include <algorithm>
#include <math.h>
#include <stdlib.h>
#include <type_traits>

namespace rsb {

using namespace rsbtc;

constexpr int T_BM = 128, T_BN = 128, T_BK = 32, T_BK16 = 64, T_STAGES = 3;
constexpr int T_THREADS = 384;                                // warpgroup 0: TMA producer, warpgroups 1-2: MMA + epilogue
constexpr int T_TILE_BYTES = 128 * T_BK * 4;                  // 16 KB
constexpr int T_STAGE_BYTES = 4 * T_TILE_BYTES;               // Ah, Al, Bh, Bl (fp16 form: Ah, Al, B)
constexpr int T_SMEM = T_STAGES * T_STAGE_BYTES + 1024 + 256;

__global__ void split_tf32_kernel(const float* __restrict__ x, size_t n, float* __restrict__ hi, float* __restrict__ lo) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        const float v = x[i];
        uint32_t h, l;
        asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(v));
        const float r = v - __uint_as_float(h);      // exact in fp32
        asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(l) : "f"(r));
        hi[i] = __uint_as_float(h);
        lo[i] = __uint_as_float(l);
    }
}

void launch_split_tf32(const float* x, size_t n, float* hi, float* lo, cudaStream_t st) {
    if (n == 0) return;
    const int blocks = (int)((n + 255) / 256 < 8192 ? (n + 255) / 256 : 8192);
    split_tf32_kernel<<<blocks, 256, 0, st>>>(x, n, hi, lo);
}

// one block of 128 threads per query row: scale to the top of the fp16 range, split into hi + lo
__global__ __launch_bounds__(128)
void split_f16_kernel(const float* __restrict__ q, int K, __half* __restrict__ hi, __half* __restrict__ lo,
                      float* __restrict__ inv) {
    __shared__ float s_max[4];
    const float* row = q + (size_t)blockIdx.x * K;
    float m = 0.f;
    for (int c = threadIdx.x; c < K; c += 128) m = fmaxf(m, fabsf(row[c]));
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = m;
    __syncthreads();
    m = fmaxf(fmaxf(s_max[0], s_max[1]), fmaxf(s_max[2], s_max[3]));
    int e = 0;
    frexpf(m, &e);                                            // m = f 2^e, f in [0.5, 1)
    const int sh = m > 0.f && isfinite(m) ? min(126, max(-126, 15 - e)) : 0;
    const float s = ldexpf(1.f, sh);
    for (int c = threadIdx.x; c < K; c += 128) {
        const float v = row[c] * s;
        const __half h = __float2half_rn(v);
        hi[(size_t)blockIdx.x * K + c] = h;
        lo[(size_t)blockIdx.x * K + c] = __float2half_rn(v - __half2float(h));   // v - h is exact in fp32
    }
    if (threadIdx.x == 0) inv[blockIdx.x] = ldexpf(1.f, -sh);
}

void launch_split_f16(const float* q, int M, int K, void* hi, void* lo, float* inv, cudaStream_t st) {
    if (M <= 0) return;
    split_f16_kernel<<<M, 128, 0, st>>>(q, K, static_cast<__half*>(hi), static_cast<__half*>(lo), inv);
}

// Persistent, warp-specialised: every CTA walks the tiles blockIdx.x, blockIdx.x + gridDim.x, ... of tile_coords' order.
// Warpgroup 0 (one thread) streams the {A, B} k-blocks of all of them through the ring without draining it between
// tiles; consumer warpgroups 1 and 2 take the CTA's tiles in turn (ping-pong) and each computes a whole 128 x 128 tile
// (two m64n128 accumulators), so one warpgroup's epilogue runs while the other one's MMAs keep the tensor cores busy.
// The k-blocks of consecutive tiles pass through the ring in order, so warpgroup w starts waiting on the stages of its
// tile only once the other warpgroup has seen every stage of the previous tile filled (mdone): a stage's full barrier
// is then never more than one phase behind the parity waited for.
//
// FUSED = false: the score tile goes to C.  FUSED = true: the score tile never goes to HBM.  Every row of the tile
// keeps its 9 largest scores in the total order (score descending, column ascending) -- the order a sequential strict
// insertion in column order realises; the top 8 are emitted as candidates (64 B per row per 128-column tile) together
// with the 9th as a bound: an element the filter dropped is <= the 9th largest of its tile, so if the kc-th best
// CANDIDATE of a row is strictly greater than the maximum of these bounds over the row, no dropped element can belong
// to the row's top kc -- select_cands_kernel checks exactly that and flags the (rare) rows for which it fails; those
// are re-done exhaustively in fp32 by exact_rows_kernel.  The result is therefore the exact top-kc of the 3xTF32
// scores without writing and re-reading nq x nlist x 4 bytes.
// F16: fp16 operands, scores multiplied by inv_b[col] (B split; tmBl unused when inv_b is null) and inv_a[row] before
// either epilogue.

// tile t -> (query tile, column tile): bands of `band` query tiles; inside a band the query tile runs fastest, so the
// CTAs in flight share a few column tiles and the band's query operand stays L2-resident while it sweeps all columns
__device__ __forceinline__ void tile_coords(int t, int tiles_m, int tiles_n, int band, int& tm, int& tn) {
    const int per_band = band * tiles_n;
    const int b = t / per_band;
    const int rows = min(band, tiles_m - b * band);
    const int local = t - b * per_band;
    tm = b * band + local % rows;
    tn = local / rows;
}

// (x, cx) ranks before (y, cy): higher score, or the same score and the lower column; empty entries (-inf, -1) last
__device__ __forceinline__ bool top9_before(float x, int cx, float y, int cy) {
    return x > y || (x == y && (unsigned)cx < (unsigned)cy);
}
// Insert (x, cx) into the sorted list where it ranks before entry i (p[i]), dropping the last entry; nothing changes
// if it ranks before none.  The list is sorted, so p is false up to the insertion point and true from there on, and
// every entry takes its new value from the old list alone: a branch-free step whose 9 lanes are independent, instead
// of a chain of 8 dependent compare-and-swaps.  The epilogue of a 128 x 128 tile runs 4 x 32 of these per lane plus
// the merges, and with one warp per scheduler their latency is not hidden.
// COL_ORDER: fed in ascending column order, so (x, cx) ranks before entry i iff x > v[i] (strict: ties keep the
// lower column, the one already in the list).
template <bool COL_ORDER>
__device__ __forceinline__ void top9_insert(float (&v)[9], int (&c)[9], float x, int cx) {
    bool p[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) p[i] = COL_ORDER ? x > v[i] : top9_before(x, cx, v[i], c[i]);
#pragma unroll
    for (int i = 8; i > 0; --i) {                             // descending: v[i - 1] is still the old entry
        v[i] = p[i - 1] ? v[i - 1] : p[i] ? x : v[i];
        c[i] = p[i - 1] ? c[i - 1] : p[i] ? cx : c[i];
    }
    v[0] = p[0] ? x : v[0];
    c[0] = p[0] ? cx : c[0];
}
// merge the list of lane ^ off into this lane's: both lanes end with the top 9 of the union in the total order
__device__ __forceinline__ void top9_merge(float (&v)[9], int (&c)[9], int off) {
    float pv[9];
    int pc[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) {
        pv[i] = __shfl_xor_sync(0xffffffffu, v[i], off);
        pc[i] = __shfl_xor_sync(0xffffffffu, c[i], off);
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) top9_insert<false>(v, c, pv[k], pc[k]);
}

template <bool F16, bool FUSED>
__global__ __launch_bounds__(T_THREADS, 1)
void gemm_ip_tc_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
                       const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl,
                       const float* __restrict__ inv, const float* __restrict__ inv_b, float* __restrict__ C, int ldc,
                       u64* __restrict__ cand, unsigned* __restrict__ xbound, int M, int N, int K, unsigned col_base,
                       int band) {
    constexpr int BK = F16 ? T_BK16 : T_BK;                   // K elements per stage: one 128-byte swizzle row
    const bool b_split = !F16 || inv_b != nullptr;            // B has a lo part (uniform over the grid)
    const int stage_tx = (b_split ? 4 : 3) * T_TILE_BYTES;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + T_STAGES * T_STAGE_BYTES);
    uint64_t* empty = full + T_STAGES;
    uint64_t* mdone = empty + T_STAGES;                       // [w]: warpgroup w has seen all stages of its tile filled

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
    const int tiles_m = (M + T_BM - 1) / T_BM, tiles_n = (N + T_BN - 1) / T_BN;
    const int ntiles = tiles_m * tiles_n;
    const int nk = (K + BK - 1) / BK;                         // columns past K read as zero

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmAh)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmAl)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmBh)) : "memory");
        if (b_split) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmBl)) : "memory");
        for (int s = 0; s < T_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4); }   // 4 warps of one consumer
        mbar_init(&mdone[0], 1);
        mbar_init(&mdone[1], 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
        if (threadIdx.x == 0) {
            int g = 0;                                        // k-block counter over all tiles of this CTA
            for (int t = blockIdx.x; t < ntiles; t += gridDim.x) {
                int tm, tn;
                tile_coords(t, tiles_m, tiles_n, band, tm, tn);
                for (int kb = 0; kb < nk; ++kb, ++g) {
                    const int s = g % T_STAGES;
                    mbar_wait(&empty[s], ((g / T_STAGES) & 1) ^ 1);   // the first pass over the ring falls through
                    unsigned char* base = smem + s * T_STAGE_BYTES;
                    mbar_expect_tx(&full[s], stage_tx);
                    tma_load_2d(base + 0 * T_TILE_BYTES, &tmAh, &full[s], kb * BK, tm * T_BM);   // rows past M / N read as zero
                    tma_load_2d(base + 1 * T_TILE_BYTES, &tmAl, &full[s], kb * BK, tm * T_BM);
                    tma_load_2d(base + 2 * T_TILE_BYTES, &tmBh, &full[s], kb * BK, tn * T_BN);
                    if (b_split) tma_load_2d(base + 3 * T_TILE_BYTES, &tmBl, &full[s], kb * BK, tn * T_BN);
                }
            }
        }
        return;
    }
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");

    const int cw = wg - 1;                                    // consumer warpgroup: local tiles cw, cw + 2, ...
    const int r_lo = (warp & 3) * 16 + (lane >> 2);           // rows of acc[h][4 j + c]: 64 h + r_lo; acc[h][4 j + 2 + c]: + 8
    const int c_lo = 2 * (lane & 3);                          // column of acc[h][4 j + c]: 8 j + c_lo + c
    float acc[2][64];
    for (int i = cw;; i += 2) {
        const int t = blockIdx.x + i * gridDim.x;
        if (t >= ntiles) break;
        int tm, tn;
        tile_coords(t, tiles_m, tiles_n, band, tm, tn);
        const int m0 = tm * T_BM, n0 = tn * T_BN;
#pragma unroll
        for (int e = 0; e < 64; ++e) { acc[0][e] = 0.f; acc[1][e] = 0.f; }
        if (i > 0) mbar_wait(&mdone[(i - 1) & 1], ((i - 1) >> 1) & 1);
        int g = i * nk;
        // one copy of the k-loop per B form, so that no branch sits between the MMAs of a stage
        auto mainloop = [&](auto split) {
            constexpr bool SPLIT = decltype(split)::value;
            for (int kb = 0; kb < nk; ++kb, ++g) {
                const int s = g % T_STAGES;
                mbar_wait(&full[s], (g / T_STAGES) & 1);
                const uint32_t base = smem_u32(smem + s * T_STAGE_BYTES);
                const uint64_t ah = make_sw128_kmajor_desc(base);
                const uint64_t al = make_sw128_kmajor_desc(base + T_TILE_BYTES);
                const uint64_t bh = make_sw128_kmajor_desc(base + 2 * T_TILE_BYTES);
                const uint64_t bl = make_sw128_kmajor_desc(base + 3 * T_TILE_BYTES);
                constexpr uint64_t LOWER = (64 * 128) >> 4;   // rows 64..127: 64 swizzle rows further in the A tiles
                acc_fence(acc[0]);
                acc_fence(acc[1]);
                wgmma_fence();
                // per output element, per K slice: the small term(s) first, the dominant hi product last
                if constexpr (F16 && SPLIT) {
#pragma unroll
                    for (int k4 = 0; k4 < T_BK16 / 16; ++k4) {  // K = 16 fp16 = 32 bytes: +2 in the (addr >> 4) field
                        const uint64_t o = (uint64_t)(k4 * 2);
                        wgmma_f16_n128(acc[0], al + o, bh + o);
                        wgmma_f16_n128(acc[1], al + LOWER + o, bh + o);
                        wgmma_f16_n128(acc[0], ah + o, bl + o);
                        wgmma_f16_n128(acc[1], ah + LOWER + o, bl + o);
                        wgmma_f16_n128(acc[0], ah + o, bh + o);
                        wgmma_f16_n128(acc[1], ah + LOWER + o, bh + o);
                    }
                } else if constexpr (F16) {
#pragma unroll
                    for (int k4 = 0; k4 < T_BK16 / 16; ++k4) {
                        const uint64_t o = (uint64_t)(k4 * 2);
                        wgmma_f16_n128(acc[0], al + o, bh + o);
                        wgmma_f16_n128(acc[1], al + LOWER + o, bh + o);
                        wgmma_f16_n128(acc[0], ah + o, bh + o);
                        wgmma_f16_n128(acc[1], ah + LOWER + o, bh + o);
                    }
                } else {
#pragma unroll
                    for (int k4 = 0; k4 < T_BK / 8; ++k4) {     // K = 8 tf32 = 32 bytes: +2 in the (addr >> 4) field
                        const uint64_t o = (uint64_t)(k4 * 2);
                        wgmma_tf32_n128(acc[0], al + o, bh + o);
                        wgmma_tf32_n128(acc[1], al + LOWER + o, bh + o);
                        wgmma_tf32_n128(acc[0], ah + o, bl + o);
                        wgmma_tf32_n128(acc[1], ah + LOWER + o, bl + o);
                        wgmma_tf32_n128(acc[0], ah + o, bh + o);
                        wgmma_tf32_n128(acc[1], ah + LOWER + o, bh + o);
                    }
                }
                wgmma_commit();
                acc_fence(acc[0]);
                acc_fence(acc[1]);
                wgmma_wait<1>();                              // the previous k-block's MMAs have retired: free its stage
                if (kb > 0) {
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty[(g - 1) % T_STAGES]);
                }
            }
        };
        if (b_split) mainloop(std::true_type{});
        else mainloop(std::false_type{});
        if (threadIdx.x % 128 == 0) mbar_arrive(&mdone[cw]);  // the other warpgroup may start on the next tile's stages
        wgmma_wait<0>();
        acc_fence(acc[0]);
        acc_fence(acc[1]);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[(g - 1) % T_STAGES]);
        if (F16 && b_split) {                                 // undo the per-column scale (a power of two: exact)
#pragma unroll
            for (int j = 0; j < 16; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const int col = n0 + 8 * j + c_lo + e;
                    const float sb = col < N ? inv_b[col] : 0.f;
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        acc[0][4 * j + 2 * h + e] *= sb;
                        acc[1][4 * j + 2 * h + e] *= sb;
                    }
                }
        }

        if (!FUSED) {
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int row = m0 + 64 * hh + r_lo + 8 * h;
                    if (row >= M) continue;
                    const float s = F16 ? inv[row] : 1.f;     // undo the per-row query scale (a power of two: exact)
                    float* dst = C + (size_t)row * ldc + n0;
#pragma unroll
                    for (int j = 0; j < 16; ++j) {
                        const int col = 8 * j + c_lo;
                        float x0 = acc[hh][4 * j + 2 * h], x1 = acc[hh][4 * j + 2 * h + 1];
                        if (F16) { x0 *= s; x1 *= s; }
                        if (n0 + col + 1 < N) *reinterpret_cast<float2*>(dst + col) = make_float2(x0, x1);
                        else if (n0 + col < N) dst[col] = x0;
                    }
                }
            continue;
        }

        // fused epilogue, straight from the accumulators: a row of the tile lives in the 4 lanes of a quad (lane & 3),
        // 32 columns each.  Each lane keeps its columns' top 9 (fed in column order), then two butterfly merges give
        // every lane of the quad the row's top 9 of the total order -- the same 9 as one sequential pass over the row.
        const int nhalf = 2 * ((N + 255) / 256);              // 128-column candidate items per row
        const int q = lane & 3;
        const int nrows = m0 + 64 < M ? 4 : 2;               // tile rows 64..127 hold no query: skip them
#pragma unroll 1
        for (int rr = 0; rr < nrows; ++rr) {                  // tile row 64 (rr >> 1) + r_lo + 8 (rr & 1)
            const int hh = rr >> 1, h = rr & 1;
            const int row = m0 + 64 * hh + r_lo + 8 * h;
            const float s = F16 ? (row < M ? inv[row] : 0.f) : 1.f;
            float v[9];
            int c[9];
#pragma unroll
            for (int e = 0; e < 9; ++e) { v[e] = -INFINITY; c[e] = -1; }
#pragma unroll
            for (int j = 0; j < 16; ++j)
#pragma unroll
                for (int e = 0; e < 2; ++e) {
                    const float a0 = h ? acc[0][4 * j + 2 + e] : acc[0][4 * j + e];
                    const float a1 = h ? acc[1][4 * j + 2 + e] : acc[1][4 * j + e];
                    float x = hh ? a1 : a0;
                    if (F16) x *= s;
                    const int col = 8 * j + c_lo + e;
                    if (n0 + col < N) top9_insert<true>(v, c, x, n0 + col);
                }
            top9_merge(v, c, 1);
            top9_merge(v, c, 2);
            if (row >= M) continue;
            u64 k0 = 0ull, k1 = 0ull;                         // this lane writes candidates 2 q, 2 q + 1
#pragma unroll
            for (int e = 0; e < 4; ++e)
                if (q == e) {
                    k0 = c[2 * e] >= 0 ? ((static_cast<u64>(ord_f32(v[2 * e])) << 32) |
                                          static_cast<u64>(0xFFFFFFFFu - (col_base + (unsigned)c[2 * e])))
                                       : 0ull;
                    k1 = c[2 * e + 1] >= 0 ? ((static_cast<u64>(ord_f32(v[2 * e + 1])) << 32) |
                                              static_cast<u64>(0xFFFFFFFFu - (col_base + (unsigned)c[2 * e + 1])))
                                           : 0ull;
                }
            const size_t item = (size_t)row * nhalf + (size_t)tn;
            reinterpret_cast<ulonglong2*>(cand + item * 8)[q] = make_ulonglong2(k0, k1);
            if (q == 0) xbound[item] = c[8] >= 0 ? ord_f32(v[8]) : 0u;
            if (tn + 1 < nhalf && tn + 1 == tiles_n) {        // the empty second half of the last 256-column group
                reinterpret_cast<ulonglong2*>(cand + (item + 1) * 8)[q] = make_ulonglong2(0ull, 0ull);
                if (q == 0) xbound[item + 1] = 0u;
            }
        }
    }
}

static bool make_maps(CUtensorMap (&m)[4], const float* Ah, const float* Al, int M, const float* Bh, const float* Bl, int N, int K) {
    return make_map_2d(&m[0], Ah, (uint64_t)M, (uint64_t)K, T_BM, 4) && make_map_2d(&m[1], Al, (uint64_t)M, (uint64_t)K, T_BM, 4) &&
           make_map_2d(&m[2], Bh, (uint64_t)N, (uint64_t)K, T_BN, 4) && make_map_2d(&m[3], Bl, (uint64_t)N, (uint64_t)K, T_BN, 4);
}

// candidates kept per row per call: 8 per 128-column tile, counted in pairs of tiles (256 columns)
size_t fused_cand_per_row(int N) { return (size_t)((N + 255) / 256) * 2 * 8; }

static int device_l2_bytes() {
    static int l2[64] = {};
    int& b = l2[current_device_slot()];
    if (!b) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&b, cudaDevAttrL2CacheSize, dev);
        if (b <= 0) b = 50 << 20;
    }
    return b;
}

// query tiles per band of the tile order: the band's hi + lo query operand takes about a third of L2, which leaves
// room for the column tiles in flight (the CTAs of one wave share them) and for what else the stream keeps there
static int tile_band(int M, int K, int elem_bytes) {
    const int tiles_m = (M + T_BM - 1) / T_BM;
    const size_t a_tile = (size_t)T_BM * K * elem_bytes * 2;
    const size_t band = (size_t)device_l2_bytes() / 3 / a_tile;
    return (int)std::max<size_t>(1, std::min<size_t>(band, (size_t)tiles_m));
}

// FUSED: cand / xbound (C unused); else C (cand / xbound unused)
template <bool F16, bool FUSED>
static void launch_gemm(const CUtensorMap (&m)[4], const float* inv, const float* inv_b, int M, int N, int K, float* C,
                        int ldc, unsigned col_base, u64* cand, unsigned* xbound, cudaStream_t st) {
    static PerDeviceSize configured;
    if (configured.raise(T_SMEM))
        cudaFuncSetAttribute(gemm_ip_tc_kernel<F16, FUSED>, cudaFuncAttributeMaxDynamicSharedMemorySize, T_SMEM);
    const int ntiles = ((M + T_BM - 1) / T_BM) * ((N + T_BN - 1) / T_BN);
    const int grid = std::min(ntiles, device_num_sms());     // one CTA per SM (shared memory), persistent
    gemm_ip_tc_kernel<F16, FUSED><<<grid, T_THREADS, T_SMEM, st>>>(m[0], m[1], m[2], m[3], inv, inv_b, C, ldc, cand, xbound,
                                                                   M, N, K, col_base, tile_band(M, K, F16 ? 2 : 4));
}

// Ah/Al [M,K], Bh/Bl [N,K] fp32 (already split).  cand [M, fused_cand_per_row(N)] u64 keys (score order high word,
// 0xFFFFFFFF - (col_base + column) low word, 0 = empty), xbound [M, fused_cand_per_row(N) / 8] (ordered score of the
// best dropped element of each 128-column tile, 0 = none).  Returns false if the path cannot run (caller falls back).
bool launch_gemm_tf32x3_topt(const float* Ah, const float* Al, int M, const float* Bh, const float* Bl, int N, int K,
                             unsigned col_base, u64* cand, unsigned* xbound, cudaStream_t st) {
    if (M <= 0 || N <= 0) return true;
    if (K % T_BK) return false;
    CUtensorMap m[4];
    if (!make_maps(m, Ah, Al, M, Bh, Bl, N, K)) return false;
    launch_gemm<false, true>(m, nullptr, nullptr, M, N, K, nullptr, 0, col_base, cand, xbound, st);
    return true;
}

bool tf32_path_available() { return get_encode() != nullptr; }

// Ah/Al [M,K], Bh/Bl [N,K] fp32 (already split), C [M, ldc] fp32.  K % 32 == 0, ldc % 4 == 0.  Returns false if
// the tensor maps cannot be encoded (caller falls back to launch_sgemm_nt -- still CUDA, never the CPU).
bool launch_gemm_tf32x3(const float* Ah, const float* Al, int M, const float* Bh, const float* Bl, int N, int K,
                        float* C, int ldc, cudaStream_t st) {
    if (M <= 0 || N <= 0) return true;
    if (K % T_BK) return false;
    CUtensorMap m[4];
    if (!make_maps(m, Ah, Al, M, Bh, Bl, N, K)) return false;
    launch_gemm<false, false>(m, nullptr, nullptr, M, N, K, C, ldc, 0u, nullptr, nullptr, st);
    return true;
}

// Ah/Al [M,K] fp16 (launch_split_f16), inv [M].  B [N,K] fp16: the rows as stored (Bl and inv_b null), or Bh/Bl and
// inv_b [N] of launch_split_f16.  K % 8 == 0 (16-byte rows; a partial last K step reads zeros).  Returns false if
// the tensor maps cannot be encoded; there is no CUDA-core fp16 path to fall back to (the caller reports an error).
static bool make_maps_f16(CUtensorMap (&m)[4], const void* Ah, const void* Al, int M, const void* Bh, const void* Bl,
                          int N, int K) {
    if (!(make_map_2d(&m[0], Ah, (uint64_t)M, (uint64_t)K, T_BM, 2) && make_map_2d(&m[1], Al, (uint64_t)M, (uint64_t)K, T_BM, 2) &&
          make_map_2d(&m[2], Bh, (uint64_t)N, (uint64_t)K, T_BN, 2)))
        return false;
    if (!Bl) {
        m[3] = m[2];                                          // unused by the kernel
        return true;
    }
    return make_map_2d(&m[3], Bl, (uint64_t)N, (uint64_t)K, T_BN, 2);
}

bool launch_gemm_f16(const void* Ah, const void* Al, const float* inv, int M, const void* Bh, const void* Bl,
                     const float* inv_b, int N, int K, float* C, int ldc, cudaStream_t st) {
    if (M <= 0 || N <= 0) return true;
    if (K % 8 || (!Bl && K % T_BK16) || !Bl != !inv_b) return false;
    CUtensorMap m[4];
    if (!make_maps_f16(m, Ah, Al, M, Bh, Bl, N, K)) return false;
    launch_gemm<true, false>(m, inv, inv_b, M, N, K, C, ldc, 0u, nullptr, nullptr, st);
    return true;
}

bool launch_gemm_f16_topt(const void* Ah, const void* Al, const float* inv, int M, const void* Bh, const void* Bl,
                          const float* inv_b, int N, int K, unsigned col_base, u64* cand, unsigned* xbound,
                          cudaStream_t st) {
    if (M <= 0 || N <= 0) return true;
    if (K % 8 || (!Bl && K % T_BK16) || !Bl != !inv_b) return false;
    CUtensorMap m[4];
    if (!make_maps_f16(m, Ah, Al, M, Bh, Bl, N, K)) return false;
    launch_gemm<true, true>(m, inv, inv_b, M, N, K, nullptr, 0, col_base, cand, xbound, st);
    return true;
}

}  // namespace rsb
