// rsb_tf32.cu -- fp32-accurate inner-product scores on the Hopper tensor cores: S[M,N] = A[M,K] . B[N,K]^T with
// A, B fp32, computed as the error-compensated 3xTF32 product
//        A.B ~= Ah.Bh + Ah.Bl + Al.Bh        (x = xh + xl, xh = tf32(x), xl = tf32(x - xh); the dropped Al.Bl term
// is ~2^-22 relative) accumulated in fp32 registers.  Used for the IVF coarse quantizer (the IndexFlatIP the reference
// builds at src/indicies/ivf_flat.py:142, ivf_pq.py:145).
//
// Same pipeline as the encoder GEMM (rsb_bert.cu): 128 x 128 output tile per CTA, TMA tensor loads (128B swizzle,
// 32 fp32 = one swizzle row per K step) -> 3-stage shared-memory ring of {Ah, Al, Bh, Bl} tiles filled by one
// producer thread -> two consumer warpgroups, each issuing 12 wgmma.m64n128k8.tf32 per stage (4 K-slices x 3
// products) on its 64 rows -> epilogue from the accumulator registers.
//
// fp16 form (F16 = true; Flat indexes with fp16 storage): B is the database as stored (fp16 rows, exact), so no split
// copy of it exists.  Each query row is scaled by a power of two s that puts its largest |element| in [2^14, 2^15)
// (exact), and split into fp16 hi = fp16(q s), lo = fp16(q s - hi): 22 significant bits, as many as the 3xTF32 query
// split; there is no lo.lo term because B is exact.  Per stage two wgmma.m64n128k16.f16 per 16-wide K-slice (lo.B,
// then hi.B) share the B tile, 64 fp16 = one swizzle row per K step; the epilogue multiplies by 1 / s.  Both forms
// share the mainloop ring and the epilogues below (score tile, or the fused top-8 candidate + bound filter).
#include "rsb_common.cuh"
#include "rsb_internal.h"
#include "rsb_tc.cuh"

#include <math.h>
#include <stdlib.h>

namespace rsb {

using namespace rsbtc;

constexpr int T_BM = 128, T_BN = 128, T_BK = 32, T_BK16 = 64, T_STAGES = 3;
constexpr int T_THREADS = 384;                                // warpgroup 0: TMA producer, warpgroups 1-2: MMA + epilogue
constexpr int T_TILE_BYTES = 128 * T_BK * 4;                  // 16 KB
constexpr int T_STAGE_BYTES = 4 * T_TILE_BYTES;               // Ah, Al, Bh, Bl (fp16 form: Ah, Al, B)
constexpr int T_SMEM = T_STAGES * T_STAGE_BYTES + 1024 + 256;
constexpr int T_LDS = T_BN + 1;                               // row stride of the fused epilogue's staged tile (floats)
static_assert(T_BM * T_LDS * 4 + T_BM * 9 * 8 <= T_STAGES * T_STAGE_BYTES, "staged tile must fit in the ring");

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

// FUSED = false: the 128 x 128 score tile goes to C.  FUSED = true: the score tile never goes to HBM.  Every row of
// the tile keeps its 9 largest scores (sorted insertion in column order, strict comparisons => ties keep the lower
// column); the top 8 are emitted as candidates (64 B per row per 128-column tile) together with the 9th as a bound:
// an element the filter dropped is <= the 9th largest of its tile, so if the kc-th best CANDIDATE of a row is
// strictly greater than the maximum of these bounds over the row, no dropped element can belong to the row's top kc
// -- select_cands_kernel checks exactly that and flags the (rare) rows for which it fails; those are re-done
// exhaustively in fp32 by exact_rows_kernel.  The result is therefore the exact top-kc of the 3xTF32 scores without
// writing and re-reading nq x nlist x 4 bytes.
// F16: fp16 operands (tmBl unused), scores multiplied by inv[row] before either epilogue.
template <bool F16, bool FUSED>
__global__ __launch_bounds__(T_THREADS, 1)
void gemm_ip_tc_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
                       const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl,
                       const float* __restrict__ inv, float* __restrict__ C, int ldc, u64* __restrict__ cand,
                       unsigned* __restrict__ xbound, int M, int N, int K, unsigned col_base, int m_fastest) {
    constexpr int BK = F16 ? T_BK16 : T_BK;                   // K elements per stage: one 128-byte swizzle row
    constexpr int STAGE_TX = (F16 ? 3 : 4) * T_TILE_BYTES;
    extern __shared__ unsigned char smem_dyn[];
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + T_STAGES * T_STAGE_BYTES);
    uint64_t* empty = full + T_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
    int tm = blockIdx.y, tn = blockIdx.x;
    const int nhalf = 2 * ((N + 255) / 256);                  // 128-column candidate items per row (FUSED)
    if (FUSED) {
        // tile order: m fastest = consecutive tiles share one B (centroid) tile and sweep the query tiles, which stay
        // L2-resident -- n fastest re-reads the whole centroid matrix per query tile
        const int tiles_m = (M + T_BM - 1) / T_BM;
        tm = m_fastest ? (int)blockIdx.x % tiles_m : (int)blockIdx.x / nhalf;
        tn = m_fastest ? (int)blockIdx.x / tiles_m : (int)blockIdx.x % nhalf;
    }
    const int m0 = tm * T_BM, n0 = tn * T_BN;
    const int nk = K / BK;
    if (FUSED && n0 >= N) {                                   // the empty second half of a 256-column group: no candidates
        const int row = m0 + (int)threadIdx.x;
        if (threadIdx.x < T_BM && row < M) {
            const size_t item = (size_t)row * nhalf + (size_t)tn;
            ulonglong2* dst = reinterpret_cast<ulonglong2*>(cand + item * 8);
#pragma unroll
            for (int i = 0; i < 4; ++i) dst[i] = make_ulonglong2(0ull, 0ull);
            xbound[item] = 0u;
        }
        return;
    }

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmAh)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmAl)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmBh)) : "memory");
        if (!F16) asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmBl)) : "memory");
        for (int s = 0; s < T_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }   // 8 consumer warps
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        if (threadIdx.x == 0) {
            for (int kb = 0; kb < nk; ++kb) {
                const int s = kb % T_STAGES;
                mbar_wait(&empty[s], ((kb / T_STAGES) & 1) ^ 1);   // the first pass over the ring falls through
                unsigned char* base = smem + s * T_STAGE_BYTES;
                mbar_expect_tx(&full[s], STAGE_TX);
                tma_load_2d(base + 0 * T_TILE_BYTES, &tmAh, &full[s], kb * BK, m0);   // rows past M / N read as zero
                tma_load_2d(base + 1 * T_TILE_BYTES, &tmAl, &full[s], kb * BK, m0);
                tma_load_2d(base + 2 * T_TILE_BYTES, &tmBh, &full[s], kb * BK, n0);
                if (!F16) tma_load_2d(base + 3 * T_TILE_BYTES, &tmBl, &full[s], kb * BK, n0);
            }
        }
        return;
    }

    const int cw = wg - 1;                                    // consumer warpgroup: tile rows 64 cw .. 64 cw + 63
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < nk; ++kb) {
        const int s = kb % T_STAGES;
        mbar_wait(&full[s], (kb / T_STAGES) & 1);
        const uint32_t base = smem_u32(smem + s * T_STAGE_BYTES);
        const uint64_t ah = make_sw128_kmajor_desc(base + cw * 64 * 128);
        const uint64_t al = make_sw128_kmajor_desc(base + T_TILE_BYTES + cw * 64 * 128);
        const uint64_t bh = make_sw128_kmajor_desc(base + 2 * T_TILE_BYTES);
        const uint64_t bl = make_sw128_kmajor_desc(base + 3 * T_TILE_BYTES);
        acc_fence(acc);
        wgmma_fence();
        if (F16) {
#pragma unroll
            for (int k4 = 0; k4 < T_BK16 / 16; ++k4) {        // K = 16 fp16 = 32 bytes: +2 in the (addr >> 4) field
                const uint64_t o = (uint64_t)(k4 * 2);
                wgmma_f16_n128(acc, al + o, bh + o);          // the small term first, then the dominant hi.B product
                wgmma_f16_n128(acc, ah + o, bh + o);
            }
        } else {
#pragma unroll
            for (int k4 = 0; k4 < T_BK / 8; ++k4) {           // K = 8 tf32 = 32 bytes: +2 in the (addr >> 4) field
                const uint64_t o = (uint64_t)(k4 * 2);
                wgmma_tf32_n128(acc, al + o, bh + o);         // small terms first, the dominant Ah.Bh product last
                wgmma_tf32_n128(acc, ah + o, bl + o);
                wgmma_tf32_n128(acc, ah + o, bh + o);
            }
        }
        wgmma_commit();
        acc_fence(acc);
        wgmma_wait<1>();                                      // the previous k-block's MMAs have retired: free its stage
        if (kb > 0) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[(kb - 1) % T_STAGES]);
        }
    }
    wgmma_wait<0>();
    acc_fence(acc);

    const int r_lo = cw * 64 + (warp & 3) * 16 + (lane >> 2);   // tile row of acc[4 j + c]; acc[4 j + 2 + c]: r_lo + 8
    const int c_lo = 2 * (lane & 3);                            // tile column of acc[4 j]: 8 j + c_lo
    if (F16) {                                                  // undo the per-row query scale (a power of two: exact)
        const float s0 = m0 + r_lo < M ? inv[m0 + r_lo] : 0.f;
        const float s1 = m0 + r_lo + 8 < M ? inv[m0 + r_lo + 8] : 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            acc[4 * j] *= s0; acc[4 * j + 1] *= s0;
            acc[4 * j + 2] *= s1; acc[4 * j + 3] *= s1;
        }
    }
    if (!FUSED) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = m0 + r_lo + 8 * h;
            if (row >= M) continue;
            float* dst = C + (size_t)row * ldc + n0;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
                const int col = 8 * j + c_lo;
                if (n0 + col + 1 < N) *reinterpret_cast<float2*>(dst + col) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                else if (n0 + col < N) dst[col] = acc[4 * j + 2 * h];
            }
        }
        return;
    }

    // fused epilogue: both consumer warpgroups are done with the ring -> stage the 128 x 128 tile there.  Every row is
    // split between the warpgroups: each selects the 9 largest scores of its 64 columns in column order, then the
    // second half's list (sorted, ties in column order) goes through the same strict-comparison insertion into the
    // first half's -- the result is exactly that of one sequential pass over the 128 columns.
    named_sync(1, 256);
    float* S = reinterpret_cast<float*>(smem);
#pragma unroll
    for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            S[(r_lo + 8 * h) * T_LDS + 8 * j + c_lo] = acc[4 * j + 2 * h];
            S[(r_lo + 8 * h) * T_LDS + 8 * j + c_lo + 1] = acc[4 * j + 2 * h + 1];
        }
    named_sync(1, 256);
    const int r = (int)threadIdx.x & 127;                     // tile row
    const int half = cw;                                      // columns 64 half .. 64 half + 63
    const int row = m0 + r;
    float v[9];
    int c[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) { v[i] = -INFINITY; c[i] = -1; }
    auto insert = [&](float x, int col) {
        if (x > v[8]) {
            v[8] = x; c[8] = col;
#pragma unroll
            for (int i = 8; i > 0; --i) {
                if (v[i] > v[i - 1]) {
                    const float tv = v[i]; v[i] = v[i - 1]; v[i - 1] = tv;
                    const int tc = c[i]; c[i] = c[i - 1]; c[i - 1] = tc;
                }
            }
        }
    };
    const float* srow = S + r * T_LDS;
    const int ncol = N - n0 < T_BN ? N - n0 : T_BN;
    const int e1 = ncol < 64 * (half + 1) ? ncol : 64 * (half + 1);
#pragma unroll 4
    for (int e = 64 * half; e < e1; ++e) insert(srow[e], n0 + e);
    float* hv = S + T_BM * T_LDS;                             // second half's lists: [128][9] scores, [128][9] columns
    int* hc = reinterpret_cast<int*>(hv + T_BM * 9);
    if (half == 1) {
#pragma unroll
        for (int i = 0; i < 9; ++i) { hv[r * 9 + i] = v[i]; hc[r * 9 + i] = c[i]; }
    }
    named_sync(1, 256);
    if (half == 1 || row >= M) return;
#pragma unroll
    for (int i = 0; i < 9; ++i) insert(hv[r * 9 + i], hc[r * 9 + i]);
    const size_t item = (size_t)row * nhalf + (size_t)tn;
    u64 keys[8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
        keys[i] = c[i] >= 0 ? ((static_cast<u64>(ord_f32(v[i])) << 32) | static_cast<u64>(0xFFFFFFFFu - (col_base + (unsigned)c[i])))
                            : 0ull;
    ulonglong2* dst = reinterpret_cast<ulonglong2*>(cand + item * 8);
#pragma unroll
    for (int i = 0; i < 4; ++i) dst[i] = make_ulonglong2(keys[2 * i], keys[2 * i + 1]);
    xbound[item] = c[8] >= 0 ? ord_f32(v[8]) : 0u;
}

static bool make_maps(CUtensorMap (&m)[4], const float* Ah, const float* Al, int M, const float* Bh, const float* Bl, int N, int K) {
    return make_map_2d(&m[0], Ah, (uint64_t)M, (uint64_t)K, T_BM, 4) && make_map_2d(&m[1], Al, (uint64_t)M, (uint64_t)K, T_BM, 4) &&
           make_map_2d(&m[2], Bh, (uint64_t)N, (uint64_t)K, T_BN, 4) && make_map_2d(&m[3], Bl, (uint64_t)N, (uint64_t)K, T_BN, 4);
}

// candidates kept per row per call: 8 per 128-column tile, counted in pairs of tiles (256 columns)
size_t fused_cand_per_row(int N) { return (size_t)((N + 255) / 256) * 2 * 8; }

template <bool F16>
static void launch_gemm_topt(const CUtensorMap (&m)[4], const float* inv, int M, int N, int K, unsigned col_base, u64* cand,
                             unsigned* xbound, cudaStream_t st) {
    static PerDeviceSize configured;
    if (configured.raise(T_SMEM))
        cudaFuncSetAttribute(gemm_ip_tc_kernel<F16, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, T_SMEM);
    const int ntiles = ((M + T_BM - 1) / T_BM) * (int)(fused_cand_per_row(N) / 8);
    static const int m_fastest = getenv("RSB_COARSE_N_FASTEST") ? 0 : 1;
    gemm_ip_tc_kernel<F16, true><<<ntiles, T_THREADS, T_SMEM, st>>>(m[0], m[1], m[2], m[3], inv, nullptr, 0, cand, xbound,
                                                                    M, N, K, col_base, m_fastest);
}

template <bool F16>
static void launch_gemm_scores(const CUtensorMap (&m)[4], const float* inv, int M, int N, int K, float* C, int ldc,
                               cudaStream_t st) {
    static PerDeviceSize configured;
    if (configured.raise(T_SMEM))
        cudaFuncSetAttribute(gemm_ip_tc_kernel<F16, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, T_SMEM);
    dim3 grid((N + T_BN - 1) / T_BN, (M + T_BM - 1) / T_BM);
    gemm_ip_tc_kernel<F16, false><<<grid, T_THREADS, T_SMEM, st>>>(m[0], m[1], m[2], m[3], inv, C, ldc, nullptr, nullptr,
                                                                   M, N, K, 0u, 0);
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
    launch_gemm_topt<false>(m, nullptr, M, N, K, col_base, cand, xbound, st);
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
    launch_gemm_scores<false>(m, nullptr, M, N, K, C, ldc, st);
    return true;
}

// Ah/Al [M,K] fp16 (launch_split_f16), inv [M], B [N,K] fp16 rows as stored.  K % 64 == 0.  Returns false if the
// tensor maps cannot be encoded; there is no CUDA-core fp16 path to fall back to (the caller reports an error).
static bool make_maps_f16(CUtensorMap (&m)[4], const void* Ah, const void* Al, int M, const void* B, int N, int K) {
    if (!(make_map_2d(&m[0], Ah, (uint64_t)M, (uint64_t)K, T_BM, 2) && make_map_2d(&m[1], Al, (uint64_t)M, (uint64_t)K, T_BM, 2) &&
          make_map_2d(&m[2], B, (uint64_t)N, (uint64_t)K, T_BN, 2)))
        return false;
    m[3] = m[2];                                              // unused by the fp16 kernel
    return true;
}

bool launch_gemm_f16x2(const void* Ah, const void* Al, const float* inv, int M, const void* B, int N, int K, float* C,
                       int ldc, cudaStream_t st) {
    if (M <= 0 || N <= 0) return true;
    if (K % T_BK16) return false;
    CUtensorMap m[4];
    if (!make_maps_f16(m, Ah, Al, M, B, N, K)) return false;
    launch_gemm_scores<true>(m, inv, M, N, K, C, ldc, st);
    return true;
}

bool launch_gemm_f16x2_topt(const void* Ah, const void* Al, const float* inv, int M, const void* B, int N, int K,
                            unsigned col_base, u64* cand, unsigned* xbound, cudaStream_t st) {
    if (M <= 0 || N <= 0) return true;
    if (K % T_BK16) return false;
    CUtensorMap m[4];
    if (!make_maps_f16(m, Ah, Al, M, B, N, K)) return false;
    launch_gemm_topt<true>(m, inv, M, N, K, col_base, cand, xbound, st);
    return true;
}

}  // namespace rsb
