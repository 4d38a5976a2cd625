// rsb_bert.cu -- BERT-base query encoder forward (reference: `Contriever.forward`, contriever/src/contriever.py:17-55,
// called from src/search.py:83-96 with the model in fp16) on variable-length (un-padded) token streams.
//
//   embed_ln_kernel      word + position + token-type gather, LayerNorm(eps)                    -> H  [T,768]  f16
//                        (<true>: RoBERTa positions, padding_idx + count of non-pad ids, for rsb_roberta_create)
//   gemm_tn_kernel       Y = X . W^T (+bias [+GELU | +residual]) on the Hopper tensor cores: TMA (cp.async.bulk.tensor,
//                        128B swizzle) -> shared-memory ring -> wgmma.mma_async f16 (fp32 accumulate in registers) ->
//                        epilogue from the registers.  Warp-specialised producer / consumer warpgroups synchronised
//                        with mbarriers.
//   attention_mma32_kernel / attention_flash_kernel   softmax(QK^T / sqrt(64)) V per (sequence, head) on mma.sync:
//                        one warp per (sequence, head) up to 32 tokens, flash-style blocks of 128 queries beyond
//                        (collect_long_kernel lists those sequences once per forward)
//   layernorm_rows_kernel  LayerNorm over 768 (fp32 statistics), persistent warps with the next row prefetched
//   pool_kernel          masked mean over the valid tokens (all tokens of an un-padded sequence) or CLS row
//
// The same handle runs a T5 encoder (rsb_t5_create; sentence-transformers' GTR-T5, reference src/search.py:49-61 and
// src/embed.py:25-40): embed_gather_kernel, then per pre-norm block layernorm_rows_kernel<true> (RMS norm + HF's fp16
// clamp), the GEMMs with zero biases and the ReLU / inf-flagging residual epilogues, and the T5 form of both attention
// kernels (relative-position bias, no scaling).  Either architecture can end in the sentence-transformers head:
// pool_kernel -> Dense on gemm_tn_kernel -> l2normalize_rows_kernel.
#include "../../include/rsb.h"

#include "rsb_dtype.cuh"
#include "rsb_internal.h"
#include "rsb_tc.cuh"

#include <cuda_fp16.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <type_traits>
#include <vector>

namespace {

using namespace rsbtc;

// ---------------------------------------------------------------------------------------------------------
// GEMM  C[M,N] = A[M,K] . B[N,K]^T  (A = activations, B = nn.Linear weight: both K-major), f16 in, f32 accumulate, on
// the Hopper tensor cores.  CTA tile 128 x 128, K step 64 (= one 128-byte swizzle row), 4-stage ring of TMA loads
// (cp.async.bulk.tensor, 128B swizzle) signalled through mbarriers.  384 threads: warpgroup 0 = producer (one thread
// issues the TMA loads), warpgroups 1-2 = consumers: each issues wgmma.m64n128k16 on its 64 rows of the tile and
// applies the epilogue (+bias [+GELU | +residual]) straight from its accumulator registers.
// ---------------------------------------------------------------------------------------------------------
constexpr int G_BM = 128, G_BN = 128, G_BK = 64, G_STAGES = 4, G_THREADS = 384;
constexpr int G_TILE_BYTES = 128 * G_BK * 2;                            // 16 KB
constexpr int G_STAGE_BYTES = 2 * G_TILE_BYTES;                         // A and B tiles
constexpr int G_SMEM = G_STAGES * G_STAGE_BYTES + 1024 /*align*/ + 256; // ring + barriers

// EPI_BIAS_RELU: T5's DenseReluDense (wi -> ReLU).  EPI_BIAS_RESIDUAL_INF: the T5 residual add, which also raises
// *inf_flag when it writes +-inf -- the condition of HF T5Block's fp16 clamp, read by the next RMS norm.
enum { EPI_BIAS = 0, EPI_BIAS_GELU = 1, EPI_BIAS_RESIDUAL = 2, EPI_BIAS_RELU = 3, EPI_BIAS_RESIDUAL_INF = 4 };

#ifdef RSB_EXACT_ERF
// HF BERT's "gelu" with CUDA's erff (-DRSB_EXACT_ERF; the default is the restatement gelu_erf_pair below)
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }
#endif

// fp32 pairs packed in 64-bit registers.  Hopper has no packed fp32 arithmetic: each pair operation is two scalar
// round-to-nearest operations (never contracted), the same rounding as a packed instruction.
__device__ __forceinline__ unsigned long long f2pack(float lo, float hi) {
    unsigned long long r;
    asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
    return r;
}
__device__ __forceinline__ void f2unpack(unsigned long long v, float& lo, float& hi) {
    asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ unsigned long long f2fma(unsigned long long a, unsigned long long b, unsigned long long c) {
    float a0, a1, b0, b1, c0, c1;
    f2unpack(a, a0, a1); f2unpack(b, b0, b1); f2unpack(c, c0, c1);
    return f2pack(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ unsigned long long f2mul(unsigned long long a, unsigned long long b) {
    float a0, a1, b0, b1;
    f2unpack(a, a0, a1); f2unpack(b, b0, b1);
    return f2pack(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ unsigned long long f2splat(float v) { return f2pack(v, v); }

// GELU restated as relu(x) + 0.5|x| (erf(|x|/sqrt 2) - 1): one multiply-add onto max(x, 0) instead of 1 - p, copysign
// and 0.5 x (1 + e); with z' = |x| sqrt(log2(e)/2) the exponent is just -z'^2 (negation folded into the MUFU operand)
// and every scale factor is folded into the polynomial's coefficients, with no cancellation for x < 0 (numpy
// restatement: max 1 fp16 ulp from the fp64 erf form, tests/test_gelu_restatement.py).
__device__ __forceinline__ unsigned long long gelu_erf_pair(unsigned long long X) {
    float x0, x1;
    f2unpack(X, x0, x1);
#ifdef RSB_EXACT_ERF
    return f2pack(gelu_erf(x0), gelu_erf(x1));
#else
    const unsigned long long Z = f2mul(f2pack(fabsf(x0), fabsf(x1)), f2splat(0.8493218003f));   // |x| sqrt(log2(e) / 2)
    float d0, d1;
    f2unpack(f2fma(Z, f2splat(0.2727374809f), f2splat(1.f)), d0, d1);                          // 1 + 0.3275911 |x| / sqrt 2
    float t0, t1;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t0) : "f"(d0));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t1) : "f"(d1));
    const unsigned long long T = f2pack(t0, t1);
    // -(0.5 / 0.8493218) (a1 t + ... + a5 t^5), Abramowitz-Stegun 7.1.26
    unsigned long long P = f2fma(T, f2splat(-0.624854695f), f2splat(0.8554778804f));
    P = f2fma(P, T, f2splat(-0.8367933924f));
    P = f2fma(P, T, f2splat(0.1674846542f));
    P = f2fma(P, T, f2splat(-0.1500194578f));
    P = f2mul(f2mul(P, T), Z);                                                                 // 0.5 |x| (erf - 1) e^{+z^2}
    float a0, a1;
    f2unpack(f2mul(Z, Z), a0, a1);
    float e0, e1;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e0) : "f"(-a0));
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e1) : "f"(-a1));
    return f2fma(P, f2pack(e0, e1), f2pack(fmaxf(x0, 0.f), fmaxf(x1, 0.f)));
#endif
}

// T = __half (every epilogue) or __nv_bfloat16 (EPI_BIAS / _GELU / _RESIDUAL, the reader's): A, B, bias, residual and
// C in T, fp32 accumulation, the epilogue rounding to T where the fp16 one rounds to half.
template <int EPI, typename T = __half>
__global__ __launch_bounds__(G_THREADS, 1)
void gemm_tn_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    T* __restrict__ C, const T* __restrict__ bias, const T* __restrict__ residual,
                    int M, int N, int K, int m_rev, int* __restrict__ inf_flag) {
    static_assert(std::is_same<T, __half>::value || EPI == EPI_BIAS || EPI == EPI_BIAS_GELU || EPI == EPI_BIAS_RESIDUAL,
                  "bf16 epilogues: bias, GELU and residual only");
    extern __shared__ unsigned char smem_dyn[];
    // 1024-byte alignment required by the 128B swizzle atom
    unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + G_STAGES * G_STAGE_BYTES);
    uint64_t* empty = full + G_STAGES;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
    const int tm = m_rev ? (int)(gridDim.y - 1 - blockIdx.y) : (int)blockIdx.y;
    const int m0 = tm * G_BM, n0 = blockIdx.x * G_BN;
    const int nk = K / G_BK;

    if (threadIdx.x == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmA)) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmB)) : "memory");
        for (int s = 0; s < G_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 8); }   // 8 consumer warps
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        if (threadIdx.x == 0) {
            for (int kb = 0; kb < nk; ++kb) {
                const int s = kb % G_STAGES;
                mbar_wait(&empty[s], ((kb / G_STAGES) & 1) ^ 1);   // the first pass over the ring falls through
                unsigned char* a_dst = smem + s * G_STAGE_BYTES;
                mbar_expect_tx(&full[s], G_STAGE_BYTES);
                tma_load_2d(a_dst, &tmA, &full[s], kb * G_BK, m0);                 // rows past M are zero-filled by TMA
                tma_load_2d(a_dst + G_TILE_BYTES, &tmB, &full[s], kb * G_BK, n0);
            }
        }
        return;
    }

    const int cw = wg - 1;                                    // consumer warpgroup: tile rows 64 cw .. 64 cw + 63
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < nk; ++kb) {
        const int s = kb % G_STAGES;
        mbar_wait(&full[s], (kb / G_STAGES) & 1);
        const uint32_t a_addr = smem_u32(smem + s * G_STAGE_BYTES);
        const uint64_t adesc = make_sw128_kmajor_desc(a_addr + cw * 64 * 128);
        const uint64_t bdesc = make_sw128_kmajor_desc(a_addr + G_TILE_BYTES);
        acc_fence(acc);
        wgmma_fence();
#pragma unroll
        for (int k4 = 0; k4 < G_BK / 16; ++k4)   // advance 16 K-elements = 32 bytes inside the swizzle row: +2 in the (addr >> 4) field
            if constexpr (std::is_same<T, __half>::value)
                wgmma_f16_n128(acc, adesc + (uint64_t)(k4 * 2), bdesc + (uint64_t)(k4 * 2));
            else
                wgmma_bf16_n128(acc, adesc + (uint64_t)(k4 * 2), bdesc + (uint64_t)(k4 * 2));
        wgmma_commit();
        acc_fence(acc);
        wgmma_wait<1>();                                      // the previous k-block's MMAs have retired: free its stage
        if (kb > 0) {
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[(kb - 1) % G_STAGES]);
        }
    }
    wgmma_wait<0>();
    acc_fence(acc);

    // epilogue: acc[4 j + 2 h + c] is row r_lo + 8 h, column 8 j + 2 (lane % 4) + c of this warpgroup's 64 x 128 block.
    // Bias added in fp32, GELU on the fp32 sum, rounded to half; the residual is added in half precision after the
    // rounding, which is also the order of HF BertSelfOutput / BertOutput (dense -> fp16, then + input).
    const int r_lo = m0 + cw * 64 + (warp & 3) * 16 + (lane >> 2);
    const int c_lo = n0 + 2 * (lane & 3);
    float2 bj[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) bj[j] = rsbdt::to_f2(*reinterpret_cast<const rsbdt::pair_t<T>*>(bias + c_lo + 8 * j));
    bool wrote_inf = false;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int row = r_lo + 8 * h;
        if (row >= M) continue;
        T* dst = C + (size_t)row * N + c_lo;
        const T* res = residual + (size_t)row * N + c_lo;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            float x0 = __fadd_rn(acc[4 * j + 2 * h], bj[j].x), x1 = __fadd_rn(acc[4 * j + 2 * h + 1], bj[j].y);
            if (EPI == EPI_BIAS_GELU) f2unpack(gelu_erf_pair(f2pack(x0, x1)), x0, x1);
            if (EPI == EPI_BIAS_RELU) { x0 = x0 < 0.f ? 0.f : x0; x1 = x1 < 0.f ? 0.f : x1; }   // NaN passes, as torch.relu
            rsbdt::pair_t<T> o = rsbdt::from_f2<T>(x0, x1);
            if (EPI == EPI_BIAS_RESIDUAL || EPI == EPI_BIAS_RESIDUAL_INF) o = __hadd2(o, *reinterpret_cast<const rsbdt::pair_t<T>*>(res + 8 * j));
            if constexpr (EPI == EPI_BIAS_RESIDUAL_INF) wrote_inf |= __hisinf(__low2half(o)) != 0 || __hisinf(__high2half(o)) != 0;
            *reinterpret_cast<rsbdt::pair_t<T>*>(dst + 8 * j) = o;
        }
    }
    if (EPI == EPI_BIAS_RESIDUAL_INF && wrote_inf) *inf_flag = 1;   // every writer stores the same value
}

// ---------------------------------------------------------------------------------------------------------
// small kernels
// ---------------------------------------------------------------------------------------------------------
constexpr int HID = 768;  // one warp per row: 24 values per lane = 3 x (8 halves)

__device__ __forceinline__ void warp_layernorm_store(float (&x)[24], const __half* gamma, const __half* beta, float eps,
                                                     __half* out, int lane) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 24; ++i) s += x[i];
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s * (1.f / HID);
    float v = 0.f;
#pragma unroll
    for (int i = 0; i < 24; ++i) { const float dlt = x[i] - mean; v = fmaf(dlt, dlt, v); }
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const float rstd = rsqrtf(v * (1.f / HID) + eps);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int col = c * 256 + lane * 8;
        const uint4 gv = *reinterpret_cast<const uint4*>(gamma + col);
        const uint4 bv = *reinterpret_cast<const uint4*>(beta + col);
        const __half2* g2 = reinterpret_cast<const __half2*>(&gv);
        const __half2* b2 = reinterpret_cast<const __half2*>(&bv);
        uint4 ov;
        __half2* o2 = reinterpret_cast<__half2*>(&ov);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float y0 = (x[c * 8 + e * 2] - mean) * rstd * __low2float(g2[e]) + __low2float(b2[e]);
            const float y1 = (x[c * 8 + e * 2 + 1] - mean) * rstd * __high2float(g2[e]) + __high2float(b2[e]);
            o2[e] = __floats2half2_rn(y0, y1);
        }
        *reinterpret_cast<uint4*>(out + col) = ov;
    }
}

__device__ __forceinline__ void load_row24(const __half* row, int lane, float (&x)[24], bool accumulate) {
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const uint4 v = *reinterpret_cast<const uint4*>(row + c * 256 + lane * 8);
        const __half2* h2 = reinterpret_cast<const __half2*>(&v);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = __half22float2(h2[e]);
            if (accumulate) { x[c * 8 + e * 2] += f.x; x[c * 8 + e * 2 + 1] += f.y; }
            else { x[c * 8 + e * 2] = f.x; x[c * 8 + e * 2 + 1] = f.y; }
        }
    }
}

// RoBERTa position of the token at offset p of the sequence starting at seq (modeling_roberta.py
// create_position_ids_from_input_ids): padding_idx for a pad id, otherwise padding_idx + the number of non-pad ids in
// seq[0..p].  Called by the whole warp (p is warp-uniform): 32 ids per ballot, ceil((p + 1) / 32) coalesced loads.
__device__ __forceinline__ int roberta_position(const int* __restrict__ seq, int p, int id, int padding_idx, int lane) {
    if (id == padding_idx) return padding_idx;
    int n = 0;
    for (int j0 = 0; j0 <= p; j0 += 32) {
        const int j = j0 + lane;
        n += __popc(__ballot_sync(0xffffffffu, j <= p && seq[j] != padding_idx));
    }
    return padding_idx + n;
}

// ROBERTA = false: BERT, position = offset in the sequence.  ROBERTA = true: roberta_position (the host has refused any
// sequence whose positions would pass max_pos).  In both forms the position is clamped to the table, which only
// matters for a caller that passes a max_seqlen below its longest sequence.
template <bool ROBERTA>
__global__ void embed_ln_kernel(const int* __restrict__ input_ids, const int* __restrict__ type_ids,
                                const int* __restrict__ cu_seqlens, int B, int T, const __half* __restrict__ word,
                                const __half* __restrict__ pos, const __half* __restrict__ type,
                                const __half* __restrict__ gamma, const __half* __restrict__ beta, float eps,
                                int vocab, int max_pos, __half* __restrict__ out, int padding_idx) {
    const int lane = threadIdx.x & 31;
    const int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= T) return;
    int lo = 0, hi = B;   // sequence b with cu[b] <= t < cu[b+1]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (cu_seqlens[mid] <= t) lo = mid; else hi = mid;
    }
    int p = t - cu_seqlens[lo];
    if constexpr (ROBERTA) p = roberta_position(input_ids + cu_seqlens[lo], p, input_ids[t], padding_idx, lane);
    p = p < max_pos ? p : max_pos - 1;
    int id = input_ids[t];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    const int tt = type_ids ? (type_ids[t] != 0) : 0;
    float x[24];
    load_row24(word + (size_t)id * HID, lane, x, false);
    load_row24(type + (size_t)tt * HID, lane, x, true);
    load_row24(pos + (size_t)p * HID, lane, x, true);
    warp_layernorm_store(x, gamma, beta, eps, out + (size_t)t * HID, lane);
}

__global__ void layernorm_kernel(const __half* __restrict__ in, int T, const __half* __restrict__ gamma,
                                 const __half* __restrict__ beta, float eps, __half* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= T) return;
    float x[24];
    load_row24(in + (size_t)t * HID, lane, x, false);
    warp_layernorm_store(x, gamma, beta, eps, out + (size_t)t * HID, lane);
}

// Persistent form for the two LayerNorms of a layer: a warp walks rows gw, gw + nw, ... with the raw 1.5 KB of its NEXT
// row already requested while it reduces and stores the current one.  Inside a forward (clock lowered by the power
// cap after a GEMM) a warp that loads, reduces and stores one row and exits is bound by its own latency chain, not by
// HBM; the one-row-per-warp kernel was slower there than in isolation (RSB_BERT_PROFILE).  Same arithmetic, same order of operations per row (RSB_LN_V1=1: the first form, A/B).
//
// RMS = true is T5LayerNorm in fp16: fp32 x rsqrt(mean(x^2) + eps), rounded to half, times the half weight (beta is
// unused).  It first applies HF T5Block's fp16 clamp to its input: when *clamp_flag is set (a residual add of the
// previous GEMM wrote +-inf anywhere in the batch) every row is clamped to +-(65504 - 1000) -- rounded to half, that
// is +-64512 -- and the clamped row is written back to the residual stream `in` before it is normalised.  Without the
// flag the clamp to +-65504 leaves the finite rows unchanged.  The kernel boundary is the batch-wide barrier that
// HF's `torch.isinf(hidden_states).any()` implies.
template <bool RMS>
__global__ __launch_bounds__(256, 3)
void layernorm_rows_kernel(const __half* __restrict__ in, int T, const __half* __restrict__ gamma,
                           const __half* __restrict__ beta, float eps, __half* __restrict__ out,
                           const int* __restrict__ clamp_flag) {
    const int lane = threadIdx.x & 31;
    const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
    if (gw >= T) return;
    uint4 cur[3], nxt[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        cur[c] = *reinterpret_cast<const uint4*>(in + (size_t)gw * HID + c * 256 + lane * 8);
        nxt[c] = cur[c];
    }
    for (int t = gw; t < T; t += nw) {
        if (t + nw < T) {
#pragma unroll
            for (int c = 0; c < 3; ++c) nxt[c] = *reinterpret_cast<const uint4*>(in + (size_t)(t + nw) * HID + c * 256 + lane * 8);
        }
        float x[24];
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const __half2* h2 = reinterpret_cast<const __half2*>(&cur[c]);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 f = __half22float2(h2[e]);
                x[c * 8 + e * 2] = f.x;
                x[c * 8 + e * 2 + 1] = f.y;
            }
        }
        if constexpr (RMS) {
            if (clamp_flag && *clamp_flag) {
#pragma unroll
                for (int c = 0; c < 3; ++c) {
                    uint4 cv;
                    __half2* c2 = reinterpret_cast<__half2*>(&cv);
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        float& a = x[c * 8 + e * 2];
                        float& b = x[c * 8 + e * 2 + 1];
                        a = a > 64504.f ? 64504.f : (a < -64504.f ? -64504.f : a);   // NaN passes, as torch.clamp
                        b = b > 64504.f ? 64504.f : (b < -64504.f ? -64504.f : b);
                        c2[e] = __floats2half2_rn(a, b);
                        a = __low2float(c2[e]);
                        b = __high2float(c2[e]);
                    }
                    *reinterpret_cast<uint4*>(const_cast<__half*>(in) + (size_t)t * HID + c * 256 + lane * 8) = cv;
                }
            }
#pragma unroll
            for (int i = 0; i < 24; ++i) s = fmaf(x[i], x[i], s);
            for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
            const float rstd = rsqrtf(s * (1.f / HID) + eps);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const uint4 gv = *reinterpret_cast<const uint4*>(gamma + c * 256 + lane * 8);
                const __half2* g2 = reinterpret_cast<const __half2*>(&gv);
                uint4 ov;
                __half2* o2 = reinterpret_cast<__half2*>(&ov);
#pragma unroll
                for (int e = 0; e < 4; ++e)
                    o2[e] = __hmul2(__floats2half2_rn(x[c * 8 + e * 2] * rstd, x[c * 8 + e * 2 + 1] * rstd), g2[e]);
                *reinterpret_cast<uint4*>(out + (size_t)t * HID + c * 256 + lane * 8) = ov;
            }
        } else {
#pragma unroll
        for (int i = 0; i < 24; ++i) s += x[i];
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        const float mean = s * (1.f / HID);
        float v = 0.f;
#pragma unroll
        for (int i = 0; i < 24; ++i) { const float dlt = x[i] - mean; v = fmaf(dlt, dlt, v); }
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        const float rstd = rsqrtf(v * (1.f / HID) + eps);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const uint4 gv = *reinterpret_cast<const uint4*>(gamma + c * 256 + lane * 8);   // L1-resident after the first row
            const uint4 bv = *reinterpret_cast<const uint4*>(beta + c * 256 + lane * 8);
            const __half2* g2 = reinterpret_cast<const __half2*>(&gv);
            const __half2* b2 = reinterpret_cast<const __half2*>(&bv);
            uint4 ov;
            __half2* o2 = reinterpret_cast<__half2*>(&ov);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float y0 = (x[c * 8 + e * 2] - mean) * rstd * __low2float(g2[e]) + __low2float(b2[e]);
                const float y1 = (x[c * 8 + e * 2 + 1] - mean) * rstd * __high2float(g2[e]) + __high2float(b2[e]);
                o2[e] = __floats2half2_rn(y0, y1);
            }
            *reinterpret_cast<uint4*>(out + (size_t)t * HID + c * 256 + lane * 8) = ov;
        }
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) cur[c] = nxt[c];
    }
}

// T5 embedding (modeling_t5.py T5Stack: embed_tokens only, not scaled, no position embedding): one warp per token
__global__ void embed_gather_kernel(const int* __restrict__ input_ids, int T, const __half* __restrict__ word, int vocab,
                                    __half* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int t = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (t >= T) return;
    int id = input_ids[t];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
#pragma unroll
    for (int c = 0; c < 3; ++c)
        *reinterpret_cast<uint4*>(out + (size_t)t * HID + c * 256 + lane * 8) =
            *reinterpret_cast<const uint4*>(word + (size_t)id * HID + c * 256 + lane * 8);
}

// sentence-transformers Normalize on a half tensor (torch.nn.functional.normalize): x / max(||x||_2, 1e-12), the norm
// accumulated in fp32 and rounded to half, the quotient rounded to half.  One warp per row, in place.
__global__ void l2normalize_rows_kernel(__half* __restrict__ x, int B) {
    const int lane = threadIdx.x & 31;
    const int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (b >= B) return;
    float v[24];
    load_row24(x + (size_t)b * HID, lane, v, false);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 24; ++i) s = fmaf(v[i], v[i], s);
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float d = fmaxf(__half2float(__float2half_rn(sqrtf(s))), 1e-12f);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        uint4 ov;
        __half2* o2 = reinterpret_cast<__half2*>(&ov);
#pragma unroll
        for (int e = 0; e < 4; ++e) o2[e] = __floats2half2_rn(__fdiv_rn(v[c * 8 + e * 2], d), __fdiv_rn(v[c * 8 + e * 2 + 1], d));
        *reinterpret_cast<uint4*>(x + (size_t)b * HID + c * 256 + lane * 8) = ov;
    }
}

// T5 relative-position bias per head and relative position r = key - query in [-511, 511]: relb[h][r + 511] =
// weight[bucket[r + 511]][h], with the bucket of every r computed on the host by HF's fp32 expression
// (T5Attention._relative_position_bucket).  Run once when both tables have been loaded.
constexpr int T5_REL = 1023;
__global__ void t5_bias_expand_kernel(const int* __restrict__ bucket, const __half* __restrict__ weight, int heads,
                                      float* __restrict__ relb) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= heads * T5_REL) return;
    const int h = i / T5_REL, k = i % T5_REL;
    relb[i] = __half2float(weight[bucket[k] * heads + h]);
}

// T5 attention score (modeling_t5.py T5Attention, fp16): scores = fp16(q.k) with no 1/sqrt(d) scaling, then
// scores = fp16(scores + bias), the sum taken in fp32 as torch does for two half tensors
__device__ __forceinline__ float t5_score(float qk, float bias) {
    return __half2float(__float2half_rn(__half2float(__float2half_rn(qk)) + bias));
}

constexpr int ATT_HD = 64, ATT_PADH = 72, ATT_MAXS = 512;

// ---------------------------------------------------------------------------------------------------------
// attention for query-length sequences (S <= 32): ONE WARP per (sequence, head), QK^T and PV on the tensor cores
// with mma.sync.m16n8k16 (a 32x32x64 problem is far too small for a wgmma tile), softmax on the accumulator
// fragments in registers.  Q and K fragments are read straight from global memory as 32-bit words (row-major
// [token, 64] slices are exactly the A / "col" B fragment layouts); V is staged per warp in shared memory and
// read with ldmatrix.trans.  ~64 MMAs per (sequence, head) instead of ~10k scalar instructions.
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
    const __half2 h = __floats2half2_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&h);
}

constexpr int ATT32_WARP_BYTES = 3 * 32 * ATT_PADH * 2;      // Q, K, V tiles of one (sequence, head)
constexpr int ATT32_T5_BIAS_BYTES = 64 * 4;                   // T5: the head's bias for r = -31..31, per warp

// T5 = true: T5 attention (t5_score, scale 1) with the head's relative-position bias from relb (t5_bias_expand_kernel)
template <bool T5>
__global__ __launch_bounds__(128)
void attention_mma32_kernel(const __half* __restrict__ qkv, const int* __restrict__ cu_seqlens, __half* __restrict__ ctx,
                            float scale, int heads, int B, int rev, const float* __restrict__ relb) {
    extern __shared__ __align__(16) unsigned char att32_smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    // blocks run last sequence first: the QKV tensor (188 MB at 41k tokens) is larger than the L2 and the GEMM wrote its
    // last rows most recently
    const int w = (rev ? (int)(gridDim.x - 1 - blockIdx.x) : (int)blockIdx.x) * 4 + wib;
    if (w >= B * heads) return;                         // warp-uniform
    const int b = w / heads, h = w % heads;
    const int t0 = cu_seqlens[b];
    const int S = cu_seqlens[b + 1] - t0;
    if (S > 32 || S <= 0) return;                        // longer sequences belong to attention_flash_kernel
    const int g = lane >> 2, t = lane & 3;
    const __half* base = qkv + (size_t)t0 * (3 * HID) + h * ATT_HD;   // Q of token 0; K at +HID, V at +2*HID
    typedef __half (*Tile)[ATT_PADH];
    Tile Qs = reinterpret_cast<Tile>(att32_smem + wib * ATT32_WARP_BYTES);
    Tile Ks = Qs + 32, Vs = Qs + 64;
    float* bsm = nullptr;                               // T5: bsm[r + 31] = bias of relative position r
    if constexpr (T5) {
        bsm = reinterpret_cast<float*>(att32_smem + 4 * ATT32_WARP_BYTES) + wib * 64;
        bsm[lane] = relb[h * T5_REL + 511 - 31 + lane];
        if (lane < 31) bsm[32 + lane] = relb[h * T5_REL + 511 + 1 + lane];
    }

    // (A persistent variant that prefetched the next item's tiles with cp.async into a second buffer was slower: the
    // double buffer halves the resident warps and the kernel is bound by the dependent-instruction latency of each warp.)
    // stage Q, K, V (rows >= S zero-filled): 8 lanes cover one 128-byte row, a warp instruction covers 4 whole rows --
    // every sector that is fetched is used (32-bit fragment loads straight from global memory would touch 32 sectors per
    // instruction for 128 useful bytes)
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int idx = lane + 32 * i, j = idx >> 3, c = idx & 7;
        uint4 qv = make_uint4(0, 0, 0, 0), kv = qv, vv = qv;
        if (j < S) {
            const __half* src = base + (size_t)j * (3 * HID) + c * 8;
            qv = *reinterpret_cast<const uint4*>(src);
            kv = *reinterpret_cast<const uint4*>(src + HID);
            vv = *reinterpret_cast<const uint4*>(src + 2 * HID);
        }
        *reinterpret_cast<uint4*>(&Qs[j][c * 8]) = qv;
        *reinterpret_cast<uint4*>(&Ks[j][c * 8]) = kv;
        *reinterpret_cast<uint4*>(&Vs[j][c * 8]) = vv;
    }
    __syncwarp();

    // S = Q K^T (fp32 accumulators): 2 m-tiles (query rows 0-15, 16-31) x 4 n-tiles (keys 8 each).  Fragments come from
    // ldmatrix.x4: one instruction per Q m-tile and per PAIR of key tiles (row stride 144 B: the 8 rows of a matrix fall
    // in 8 disjoint groups of 4 banks).
    const int ntm = (S + 7) >> 3;                        // key tiles of 8 that hold at least one valid key (NQ queries: 3 of 4)
    float sacc[2][4][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) sacc[mt][nt][e] = 0.f;
    // lane -> row/column of the 8x8 matrix whose row address it supplies
    const uint32_t q_lane = smem_u32(&Qs[(lane & 7) + ((lane >> 3) & 1) * 8][(lane >> 4) * 8]);   // A: (r, k), (r+8, k), (r, k+8), (r+8, k+8)
    const uint32_t k_lane = smem_u32(&Ks[(lane & 7) + ((lane >> 4) & 1) * 8][((lane >> 3) & 1) * 8]); // B: tile nt (k, k+8), tile nt+1 (k, k+8)
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
        uint32_t qa[2][4], kb[4][2];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
            asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                         : "=r"(qa[mt][0]), "=r"(qa[mt][1]), "=r"(qa[mt][2]), "=r"(qa[mt][3])
                         : "r"(q_lane + (uint32_t)((mt * 16 * ATT_PADH + ks * 16) * 2)));
#pragma unroll
        for (int np = 0; np < 2; ++np) {
            if (np * 2 < ntm) {                          // warp-uniform: key tiles past the sequence end are skipped
                asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                             : "=r"(kb[np * 2][0]), "=r"(kb[np * 2][1]), "=r"(kb[np * 2 + 1][0]), "=r"(kb[np * 2 + 1][1])
                             : "r"(k_lane + (uint32_t)((np * 16 * ATT_PADH + ks * 16) * 2)));
#pragma unroll
                for (int mt = 0; mt < 2; ++mt) mma_16816(sacc[mt][np * 2], qa[mt], kb[np * 2]);
                if (np * 2 + 1 < ntm) {
#pragma unroll
                    for (int mt = 0; mt < 2; ++mt) mma_16816(sacc[mt][np * 2 + 1], qa[mt], kb[np * 2 + 1]);
                }
            }
        }
    }

    // softmax over keys: thread holds rows (mt*16 + g) [elements 0,1] and (mt*16 + g + 8) [elements 2,3], key columns
    // nt*8 + 2t + {0,1}; a row is spread over the 4 lanes of a quad.  exp((s - max) scale) = 2^(s c - max c) with
    // c = scale log2(e): one FFMA + one MUFU per element.  Every row sees at least one valid key (S >= 1), so the row
    // maximum is finite and the sum positive.  The probabilities are normalised BEFORE they are rounded to half -- the
    // order of HF BERT (softmax -> fp16 probabilities -> P V) -- which also halves the scaling work (32 instead of 64
    // multiplies per lane).
    const float cexp = scale * 1.4426950408889634f;
    uint32_t pa[2][2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
        float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            if (nt < ntm) {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int col = nt * 8 + 2 * t + (e & 1);
                    float s;
                    if constexpr (T5) s = col < S ? t5_score(sacc[mt][nt][e], bsm[col - (mt * 16 + g + (e >> 1) * 8) + 31]) : -INFINITY;
                    else s = col < S ? sacc[mt][nt][e] : -INFINITY;
                    sacc[mt][nt][e] = s;
                    if (e < 2) mx0 = fmaxf(mx0, s); else mx1 = fmaxf(mx1, s);
                }
            }
        }
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
        const float m0c = -mx0 * cexp, m1c = -mx1 * cexp;
        float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) {
            if (nt < ntm) {                              // skipped tiles keep their zeros = probability 0
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    float p;
                    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(p) : "f"(fmaf(sacc[mt][nt][e], cexp, e < 2 ? m0c : m1c)));   // 2^(-inf) = 0
                    sacc[mt][nt][e] = p;
                    if (e < 2) sum0 += p; else sum1 += p;
                }
            }
        }
        sum0 += __shfl_xor_sync(0xffffffffu, sum0, 1); sum0 += __shfl_xor_sync(0xffffffffu, sum0, 2);
        sum1 += __shfl_xor_sync(0xffffffffu, sum1, 1); sum1 += __shfl_xor_sync(0xffffffffu, sum1, 2);
        const float inv0 = __fdividef(1.f, sum0), inv1 = __fdividef(1.f, sum1);
        // probabilities as the A operand of P.V: k-step kk covers keys 16kk..16kk+15 = n-tiles 2kk, 2kk+1
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {
            pa[mt][kk][0] = pack_half2(sacc[mt][2 * kk][0] * inv0, sacc[mt][2 * kk][1] * inv0);
            pa[mt][kk][1] = pack_half2(sacc[mt][2 * kk][2] * inv1, sacc[mt][2 * kk][3] * inv1);
            pa[mt][kk][2] = pack_half2(sacc[mt][2 * kk + 1][0] * inv0, sacc[mt][2 * kk + 1][1] * inv0);
            pa[mt][kk][3] = pack_half2(sacc[mt][2 * kk + 1][2] * inv1, sacc[mt][2 * kk + 1][3] * inv1);
        }
    }
    // O = P V : 2 m-tiles x 8 n-tiles (head dims 8 each); V^T fragments of both 16-key steps through ONE ldmatrix.x4.trans
    // (rows = keys 0..31 of this lane, zero-filled past the sequence end)
    const uint32_t v_lane = smem_u32(&Vs[lane][0]);
    const bool two_steps = S > 16;                       // warp-uniform: a 16-key step without valid keys adds nothing
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
        float o[2][4] = {{0.f, 0.f, 0.f, 0.f}, {0.f, 0.f, 0.f, 0.f}};
        uint32_t vb[2][2];
        asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
                     : "=r"(vb[0][0]), "=r"(vb[0][1]), "=r"(vb[1][0]), "=r"(vb[1][1])
                     : "r"(v_lane + (uint32_t)(nt * 8 * 2)));
        mma_16816(o[0], pa[0][0], vb[0]);
        mma_16816(o[1], pa[1][0], vb[0]);
        if (two_steps) {
            mma_16816(o[0], pa[0][1], vb[1]);
            mma_16816(o[1], pa[1][1], vb[1]);
        }
        // the output tile goes back through this warp's Q tile (all Q fragments were consumed before the first P.V
        // MMA; program order inside the warp + the __syncwarp below make the reuse safe) so that it can be written
        // with whole 128-byte rows instead of 4-byte pieces
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            const int r0 = mt * 16 + g, col = nt * 8 + 2 * t;
            *reinterpret_cast<__half2*>(&Qs[r0][col]) = __floats2half2_rn(o[mt][0], o[mt][1]);
            *reinterpret_cast<__half2*>(&Qs[r0 + 8][col]) = __floats2half2_rn(o[mt][2], o[mt][3]);
        }
    }
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int idx = lane + 32 * i, j = idx >> 3, c = idx & 7;
        if (j < S)
            *reinterpret_cast<uint4*>(ctx + (size_t)(t0 + j) * HID + h * ATT_HD + c * 8) = *reinterpret_cast<const uint4*>(&Qs[j][c * 8]);
    }
}


// sequences longer than `threshold` tokens -> list (order irrelevant) + count; once per forward
__global__ void collect_long_kernel(const int* __restrict__ cu_seqlens, int B, int threshold, int* __restrict__ list,
                                    int* __restrict__ count) {
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < B; b += gridDim.x * blockDim.x)
        if (cu_seqlens[b + 1] - cu_seqlens[b] > threshold) list[atomicAdd(count, 1)] = b;
}

// ---------------------------------------------------------------------------------------------------------
// attention for longer sequences (33..512 tokens: the passage side, reference src/embed.py:24-94 at batch 512):
// flash-style on the tensor cores.  One block = 4 warps = 128 consecutive query rows of one (sequence, head); a warp
// owns 32 query rows (Q fragments stay in registers) and walks the keys in blocks of 32 that the whole block stages
// in shared memory once: S = Q K^T with mma.sync.m16n8k16, online softmax on the accumulator fragments (running row
// maximum / sum, output rescaled when the maximum moves), O += P V with V^T fragments through ldmatrix.trans.
// Same arithmetic as attention_mma32_kernel for a single key block.
// ---------------------------------------------------------------------------------------------------------
template <bool T5>
__global__ __launch_bounds__(128)
void attention_flash_kernel(const __half* __restrict__ qkv, const int* __restrict__ cu_seqlens, __half* __restrict__ ctx,
                            float scale, const int* __restrict__ long_list, const int* __restrict__ long_count, int heads,
                            int nqb, const float* __restrict__ relb) {
    __shared__ __align__(16) __half Ks[32][ATT_PADH];
    __shared__ __align__(16) __half Vs[32][ATT_PADH];
    float* Bs = nullptr;                                 // T5: Bs[r + 511] = bias of relative position r for this item's head
    if constexpr (T5) {
        __shared__ float t5_bias[T5_REL];
        Bs = t5_bias;
    }
    // work items (long sequence, head, block of 128 queries) in a grid-stride loop over the list that collect_long_kernel
    // wrote once for this forward.  A batch of queries holds one or two sequences beyond 32 tokens: walking all
    // B x heads x nqb candidates every layer would keep the side stream busy and slow the short-sequence kernel it
    // overlaps with.
    const int n_items = *long_count * heads * nqb;
    for (int item = blockIdx.x; item < n_items; item += gridDim.x) {
    const int qblk = item % nqb, h = (item / nqb) % heads, b = long_list[item / (nqb * heads)];
    const int t0 = cu_seqlens[b];
    const int S = cu_seqlens[b + 1] - t0;
    const int q0 = qblk * 128;
    if (q0 >= S) continue;                               // block-uniform
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int g = lane >> 2, t = lane & 3;
    const int qw = q0 + wib * 32;                        // first query row of this warp
    const bool active = qw < S;                          // warp-uniform; idle warps still stage K / V and hit the barriers
    const __half* base = qkv + (size_t)t0 * (3 * HID) + h * ATT_HD;
    if constexpr (T5) {                                  // visible after the first barrier of the key loop
        for (int i = threadIdx.x; i < T5_REL; i += 128) Bs[i] = relb[h * T5_REL + i];
    }

    uint32_t qa[4][2][4];
#pragma unroll
    for (int ks = 0; ks < 4; ++ks)
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            const int r0 = qw + mt * 16 + g, c = ks * 16 + 2 * t;
            const __half* p0 = base + (size_t)r0 * (3 * HID) + c;
            const __half* p1 = base + (size_t)(r0 + 8) * (3 * HID) + c;
            qa[ks][mt][0] = r0 < S ? *reinterpret_cast<const uint32_t*>(p0) : 0u;
            qa[ks][mt][1] = r0 + 8 < S ? *reinterpret_cast<const uint32_t*>(p1) : 0u;
            qa[ks][mt][2] = r0 < S ? *reinterpret_cast<const uint32_t*>(p0 + 8) : 0u;
            qa[ks][mt][3] = r0 + 8 < S ? *reinterpret_cast<const uint32_t*>(p1 + 8) : 0u;
        }
    float o[2][8][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) o[mt][nt][e] = 0.f;
    float m_run[2][2] = {{-INFINITY, -INFINITY}, {-INFINITY, -INFINITY}};
    float l_run[2][2] = {{0.f, 0.f}, {0.f, 0.f}};       // per-lane partial row sums (quad-reduced at the end)

    const int nkb = (S + 31) >> 5;
    for (int kb = 0; kb < nkb; ++kb) {
        __syncthreads();                                 // the previous key block has been consumed by every warp
#pragma unroll
        for (int i = 0; i < 2; ++i) {                    // 32 rows x 8 uint4 for K and for V: 2 + 2 per thread
            const int idx = threadIdx.x + 128 * i, j = idx >> 3, c = idx & 7;
            const int key = kb * 32 + j;
            uint4 kv = make_uint4(0, 0, 0, 0), vv = make_uint4(0, 0, 0, 0);
            if (key < S) {
                const __half* src = base + (size_t)key * (3 * HID) + c * 8;
                kv = *reinterpret_cast<const uint4*>(src + HID);
                vv = *reinterpret_cast<const uint4*>(src + 2 * HID);
            }
            *reinterpret_cast<uint4*>(&Ks[j][c * 8]) = kv;
            *reinterpret_cast<uint4*>(&Vs[j][c * 8]) = vv;
        }
        __syncthreads();
        if (!active) continue;
        float sacc[2][4][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) sacc[mt][nt][e] = 0.f;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            uint32_t kbf[4][2];
#pragma unroll
            for (int nt = 0; nt < 4; ++nt) {
                const int j = nt * 8 + g, c = ks * 16 + 2 * t;
                kbf[nt][0] = *reinterpret_cast<const uint32_t*>(&Ks[j][c]);
                kbf[nt][1] = *reinterpret_cast<const uint32_t*>(&Ks[j][c + 8]);
            }
#pragma unroll
            for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                for (int nt = 0; nt < 4; ++nt) mma_16816(sacc[mt][nt], qa[ks][mt], kbf[nt]);
        }
        uint32_t pa[2][2][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
            float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int col = kb * 32 + nt * 8 + 2 * t + (e & 1);
                    float sv;
                    if constexpr (T5) sv = col < S ? t5_score(sacc[mt][nt][e], Bs[col - (qw + mt * 16 + g + (e >> 1) * 8) + 511]) : -INFINITY;
                    else sv = col < S ? sacc[mt][nt][e] * scale : -INFINITY;
                    sacc[mt][nt][e] = sv;
                    if (e < 2) mx0 = fmaxf(mx0, sv); else mx1 = fmaxf(mx1, sv);
                }
            mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1)); mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
            mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1)); mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
            // every key block holds at least one valid key, so the new maxima are finite
            const float mn0 = fmaxf(m_run[mt][0], mx0), mn1 = fmaxf(m_run[mt][1], mx1);
            const float cr0 = __expf(m_run[mt][0] - mn0), cr1 = __expf(m_run[mt][1] - mn1);   // exp(-inf) = 0 on the first block
            m_run[mt][0] = mn0; m_run[mt][1] = mn1;
            float sum0 = 0.f, sum1 = 0.f;
#pragma unroll
            for (int nt = 0; nt < 4; ++nt)
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float sv = sacc[mt][nt][e];
                    const float pv = (sv == -INFINITY) ? 0.f : __expf(sv - (e < 2 ? mn0 : mn1));
                    sacc[mt][nt][e] = pv;
                    if (e < 2) sum0 += pv; else sum1 += pv;
                }
            l_run[mt][0] = l_run[mt][0] * cr0 + sum0;
            l_run[mt][1] = l_run[mt][1] * cr1 + sum1;
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                o[mt][nt][0] *= cr0; o[mt][nt][1] *= cr0;
                o[mt][nt][2] *= cr1; o[mt][nt][3] *= cr1;
            }
#pragma unroll
            for (int kk = 0; kk < 2; ++kk) {
                pa[mt][kk][0] = pack_half2(sacc[mt][2 * kk][0], sacc[mt][2 * kk][1]);
                pa[mt][kk][1] = pack_half2(sacc[mt][2 * kk][2], sacc[mt][2 * kk][3]);
                pa[mt][kk][2] = pack_half2(sacc[mt][2 * kk + 1][0], sacc[mt][2 * kk + 1][1]);
                pa[mt][kk][3] = pack_half2(sacc[mt][2 * kk + 1][2], sacc[mt][2 * kk + 1][3]);
            }
        }
#pragma unroll
        for (int nt = 0; nt < 8; ++nt)
#pragma unroll
            for (int kk = 0; kk < 2; ++kk) {
                uint32_t vb[2];
                const uint32_t addr = smem_u32(&Vs[kk * 16 + (lane & 15)][nt * 8]);
                asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(vb[0]), "=r"(vb[1]) : "r"(addr));
                mma_16816(o[0][nt], pa[0][kk], vb);
                mma_16816(o[1][nt], pa[1][kk], vb);
            }
    }
    if (active) {
#pragma unroll
    for (int mt = 0; mt < 2; ++mt) {
        float l0 = l_run[mt][0], l1 = l_run[mt][1];
        l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
        l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
        const float i0 = l0 > 0.f ? 1.f / l0 : 0.f, i1 = l1 > 0.f ? 1.f / l1 : 0.f;
        const int r0 = qw + mt * 16 + g;
#pragma unroll
        for (int nt = 0; nt < 8; ++nt) {
            const int col = h * ATT_HD + nt * 8 + 2 * t;
            if (r0 < S)
                *reinterpret_cast<__half2*>(ctx + (size_t)(t0 + r0) * HID + col) = __floats2half2_rn(o[mt][nt][0] * i0, o[mt][nt][1] * i0);
            if (r0 + 8 < S)
                *reinterpret_cast<__half2*>(ctx + (size_t)(t0 + r0 + 8) * HID + col) = __floats2half2_rn(o[mt][nt][2] * i1, o[mt][nt][3] * i1);
        }
    }
    }
    __syncthreads();                                     // K / V tiles are re-staged by the next item
    }
}

// pooling: one block per sequence; mode 0 = mean over tokens (contriever.py:45-49), 1 = CLS row (:50-51)
__global__ void pool_kernel(const __half* __restrict__ H, const int* __restrict__ cu_seqlens, int mode,
                            __half* __restrict__ out) {
    const int b = blockIdx.x;
    const int t0 = cu_seqlens[b], t1 = cu_seqlens[b + 1];
    for (int c = threadIdx.x; c < HID; c += blockDim.x) {
        float s = 0.f;
        if (mode == 1 || t1 <= t0) {
            s = t1 > t0 ? __half2float(H[(size_t)t0 * HID + c]) : 0.f;
        } else {
            for (int t = t0; t < t1; ++t) s += __half2float(H[(size_t)t * HID + c]);
            s /= (float)(t1 - t0);
        }
        out[(size_t)b * HID + c] = __float2half_rn(s);
    }
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
thread_local std::string g_berr;
int bfail(int code, const char* fmt, const char* a = "", long b = 0) {
    char buf[512];
    snprintf(buf, sizeof buf, fmt, a, b);
    g_berr = buf;
    return code;
}

bool make_map(CUtensorMap* m, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows, bool bf16 = false) {
    return rsbtc::make_map_2d(m, base, rows, cols, box_rows, 2, bf16);
}

struct Linear {
    __half* w = nullptr;   // [N, K]
    __half* b = nullptr;   // [N]
    int N = 0, K = 0;
    CUtensorMap map;       // box 128 rows
    bool map_ok = false;
};

struct Layer {
    Linear qkv, attn_out, ffn1, ffn2;
    __half *ln1_g = nullptr, *ln1_b = nullptr, *ln2_g = nullptr, *ln2_b = nullptr;
};

}  // namespace

struct rsb_bert {
    int hidden = 768, layers = 12, heads = 12, inter = 3072, vocab = 30522, max_pos = 512, type_vocab = 2;
    float eps = 1e-12f;
    int padding_idx = -1;                                // >= 0: a RoBERTa handle (rsb_roberta_create), its position rule
    __half *word = nullptr, *pos = nullptr, *type = nullptr, *emb_g = nullptr, *emb_b = nullptr;
    std::vector<Layer> L;
    // T5 encoder (rsb_t5_create): pre-norm blocks, RMS norms ln1_g / ln2_g, no biases (the Linear biases stay zero)
    bool t5 = false;
    int num_buckets = 0, max_distance = 0;
    int* bucket = nullptr;                               // [T5_REL] bucket of r = -511..511
    __half* rel_w = nullptr;                             // [num_buckets, heads] relative_attention_bias.weight
    float* relb = nullptr;                               // [heads, T5_REL] expanded by t5_bias_expand_kernel
    bool bucket_loaded = false, rel_w_loaded = false;
    __half* final_g = nullptr;                           // encoder.final_layer_norm.weight
    // sentence-transformers Dense head (both architectures): 768 -> 768, bias zero unless loaded
    Linear dense;
    bool dense_loaded = false;
    long launches = 0;
    // the two attention kernels of a layer work on disjoint sequences (<= 32 tokens / longer): the long-sequence one runs
    // on a side stream so that it overlaps the other instead of adding its latency to every layer
    cudaStream_t side = nullptr;
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    int* long_list = nullptr;                            // sequences > 32 tokens of the current forward; [long_cap] = their count
    int long_cap = 0;
};

namespace {

int alloc_linear(Linear& l, int N, int K) {
    l.N = N; l.K = K;
    if (cudaMalloc(&l.w, (size_t)N * K * 2) != cudaSuccess) return RSB_ERR_OOM;
    if (cudaMalloc(&l.b, (size_t)N * 2) != cudaSuccess) return RSB_ERR_OOM;
    cudaMemset(l.w, 0, (size_t)N * K * 2);
    cudaMemset(l.b, 0, (size_t)N * 2);
    l.map_ok = make_map(&l.map, l.w, N, K, G_BN);
    return l.map_ok ? RSB_OK : RSB_ERR_CUDA;
}
void free_linear(Linear& l) { cudaFree(l.w); cudaFree(l.b); }

// m_rev: visit the row tiles last-to-first.  The FFN intermediate (251 MB at 41k tokens) is twice the L2: FFN2 starts with the
// rows FFN1 wrote last, which are still cached (RSB_NO_SNAKE=1 disables, A/B).
// T = __nv_bfloat16: lin.w / lin.b hold bf16 and lin.map is a BFLOAT16 map.
template <int EPI, typename T = __half>
int launch_gemm(const T* A, int M, const Linear& lin, typename std::common_type<T>::type* C,
                const typename std::common_type<T>::type* residual, cudaStream_t st, bool m_rev = false,
                int* inf_flag = nullptr) {
    constexpr bool bf16 = std::is_same<T, __nv_bfloat16>::value;
    CUtensorMap tmA;
    if (!lin.map_ok || !make_map(&tmA, A, (uint64_t)M, (uint64_t)lin.K, G_BM, bf16)) return RSB_ERR_CUDA;
    static rsb::PerDeviceFlag configured;                    // attributes are per (function, device)
    if (configured.first()) cudaFuncSetAttribute(gemm_tn_kernel<EPI, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, G_SMEM);
    static const bool no_snake = getenv("RSB_NO_SNAKE") != nullptr;
    dim3 grid(lin.N / G_BN, (M + G_BM - 1) / G_BM);              // consecutive CTAs share one row tile of A
    gemm_tn_kernel<EPI, T><<<grid, G_THREADS, G_SMEM, st>>>(tmA, lin.map, C, reinterpret_cast<const T*>(lin.b), residual,
                                                            M, lin.N, lin.K, (m_rev && !no_snake) ? 1 : 0, inf_flag);
    return RSB_OK;
}

// Per-forward set-up of the attention step: the kernels' shared-memory attributes, the side stream and its events, and
// -- when max_seqlen > 32 -- the list of sequences the flash kernel takes (collect_long_kernel), built once and read by
// every layer's launch_attention.
int prepare_attention(rsb_bert* h, const int* cu_seqlens, int B, int max_seqlen, cudaStream_t st) {
    static rsb::PerDeviceFlag att_configured;
    if (att_configured.first()) {
        cudaFuncSetAttribute(attention_mma32_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * ATT32_WARP_BYTES);
        cudaFuncSetAttribute(attention_mma32_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             4 * (ATT32_WARP_BYTES + ATT32_T5_BIAS_BYTES));
    }
    if (!h->side) {
        cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking);
        cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming);
        cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming);
    }
    if (max_seqlen > 32) {                               // list of the sequences the flash kernel has to take, once per forward
        if (h->long_cap < B) {
            cudaFree(h->long_list);
            h->long_list = nullptr;
            h->long_cap = 0;
            if (cudaMalloc(&h->long_list, ((size_t)B + 1) * sizeof(int)) != cudaSuccess) return bfail(RSB_ERR_OOM, "long-sequence list");
            h->long_cap = B;
        }
        cudaMemsetAsync(h->long_list + h->long_cap, 0, sizeof(int), st);          // the count lives behind the list
        collect_long_kernel<<<(B + 255) / 256, 256, 0, st>>>(cu_seqlens, B, 32, h->long_list, h->long_list + h->long_cap);
        h->launches++;
    }
    return RSB_OK;
}

// One attention step, ctx [T, 768] from qkv [T, 2304], after prepare_attention with the same cu_seqlens / B / max_seqlen.
// Sequences of <= 32 tokens (queries): warp-per-(sequence, head) tensor-core kernel; longer ones (passages, the odd long
// query): flash-style kernel on a side stream -- the two work on disjoint sequences of the same buffers -- joined
// before the caller's next launch on st.
void launch_attention(rsb_bert* h, const __half* qkv_p, const int* cu_seqlens, int B, int max_seqlen, __half* ctx_p,
                      cudaStream_t st) {
    const float scale = h->t5 ? 1.f : 0.125f;
    const bool have_long = max_seqlen > 32;
    if (have_long) {
        cudaEventRecord(h->ev_fork, st);
        cudaStreamWaitEvent(h->side, h->ev_fork, 0);
        const int nqb = (max_seqlen + 127) / 128;
        const long items = (long)B * h->heads * nqb;
        const int fgrid = (int)std::min<long>(items, 2L * rsb::device_num_sms());   // 194 registers: two resident blocks per SM
        if (h->t5)
            attention_flash_kernel<true><<<fgrid, 128, 0, h->side>>>(qkv_p, cu_seqlens, ctx_p, scale, h->long_list,
                                                                     h->long_list + h->long_cap, h->heads, nqb, h->relb);
        else
            attention_flash_kernel<false><<<fgrid, 128, 0, h->side>>>(qkv_p, cu_seqlens, ctx_p, scale, h->long_list,
                                                                      h->long_list + h->long_cap, h->heads, nqb, nullptr);
        cudaEventRecord(h->ev_join, h->side);
        h->launches++;
    }
    const int nwarps = B * h->heads;
    static const bool no_snake = getenv("RSB_NO_SNAKE") != nullptr;
    if (h->t5)
        attention_mma32_kernel<true><<<(nwarps + 3) / 4, 128, 4 * (ATT32_WARP_BYTES + ATT32_T5_BIAS_BYTES), st>>>(
            qkv_p, cu_seqlens, ctx_p, scale, h->heads, B, no_snake ? 0 : 1, h->relb);
    else
        attention_mma32_kernel<false><<<(nwarps + 3) / 4, 128, 4 * ATT32_WARP_BYTES, st>>>(
            qkv_p, cu_seqlens, ctx_p, scale, h->heads, B, no_snake ? 0 : 1, nullptr);
    h->launches++;
    if (have_long) cudaStreamWaitEvent(st, h->ev_join, 0);   // join before the attention-output GEMM
}

}  // namespace

extern "C" const char* rsb_bert_last_error(void) { return g_berr.c_str(); }

extern "C" int rsb_bert_create(int hidden, int layers, int heads, int inter, int vocab, int max_pos, int type_vocab,
                               float ln_eps, rsb_bert_t** out) {
    if (!out) return bfail(RSB_ERR_INVALID, "out is NULL");
    *out = nullptr;
    if (hidden != 768 || heads != 12 || inter % G_BN || inter % G_BK || layers <= 0 || vocab <= 0 || max_pos <= 0 || type_vocab <= 0)
        return bfail(RSB_ERR_UNSUPPORTED, "only BERT-base geometry (hidden 768, 12 heads, FFN multiple of 128) is implemented");
    if (!get_encode()) return bfail(RSB_ERR_CUDA, "cuTensorMapEncodeTiled is not available from this driver");
    rsb_bert* h = new rsb_bert();
    h->hidden = hidden; h->layers = layers; h->heads = heads; h->inter = inter; h->vocab = vocab;
    h->max_pos = max_pos; h->type_vocab = type_vocab; h->eps = ln_eps;
    bool ok = true;
    ok &= cudaMalloc(&h->word, (size_t)vocab * hidden * 2) == cudaSuccess;
    ok &= cudaMalloc(&h->pos, (size_t)max_pos * hidden * 2) == cudaSuccess;
    ok &= cudaMalloc(&h->type, (size_t)std::max(type_vocab, 2) * hidden * 2) == cudaSuccess;
    ok &= cudaMalloc(&h->emb_g, hidden * 2) == cudaSuccess;
    ok &= cudaMalloc(&h->emb_b, hidden * 2) == cudaSuccess;
    ok &= alloc_linear(h->dense, hidden, hidden) == RSB_OK;
    if (ok) cudaMemset(h->type, 0, (size_t)std::max(type_vocab, 2) * hidden * 2);
    h->L.resize(layers);
    for (auto& l : h->L) {
        ok &= alloc_linear(l.qkv, 3 * hidden, hidden) == RSB_OK;
        ok &= alloc_linear(l.attn_out, hidden, hidden) == RSB_OK;
        ok &= alloc_linear(l.ffn1, inter, hidden) == RSB_OK;
        ok &= alloc_linear(l.ffn2, hidden, inter) == RSB_OK;
        ok &= cudaMalloc(&l.ln1_g, hidden * 2) == cudaSuccess;
        ok &= cudaMalloc(&l.ln1_b, hidden * 2) == cudaSuccess;
        ok &= cudaMalloc(&l.ln2_g, hidden * 2) == cudaSuccess;
        ok &= cudaMalloc(&l.ln2_b, hidden * 2) == cudaSuccess;
    }
    if (!ok) { rsb_bert_free(h); return bfail(RSB_ERR_OOM, "allocating encoder weights failed"); }
    *out = h;
    return RSB_OK;
}

// Replaces `SentenceTransformer(name)`'s T5 module (src/search.py:49-61, src/embed.py:25-40): HF T5EncoderModel with
// d_model 768, 12 heads of 64 and a ReLU feed-forward of d_ff.
extern "C" int rsb_t5_create(int layers, int d_ff, int vocab, int num_buckets, int max_distance, float eps,
                             rsb_bert_t** out) {
    if (!out) return bfail(RSB_ERR_INVALID, "out is NULL");
    *out = nullptr;
    if (layers <= 0 || d_ff <= 0 || d_ff % G_BN || vocab <= 0 || num_buckets < 2 || max_distance <= 0)
        return bfail(RSB_ERR_UNSUPPORTED, "only T5 encoders with d_model 768, 12 heads of 64 and a ReLU feed-forward of a "
                                          "multiple of 128 are implemented%s (got d_ff %ld)", "", (long)d_ff);
    rsb_bert_t* h = nullptr;
    const int rc = rsb_bert_create(768, layers, 12, d_ff, vocab, ATT_MAXS, 1, eps, &h);
    if (rc != RSB_OK) return rc;
    h->t5 = true;
    h->num_buckets = num_buckets;
    h->max_distance = max_distance;
    bool ok = true;
    ok &= cudaMalloc(&h->bucket, T5_REL * sizeof(int)) == cudaSuccess;
    ok &= cudaMalloc(&h->rel_w, (size_t)num_buckets * h->heads * 2) == cudaSuccess;
    ok &= cudaMalloc(&h->relb, (size_t)h->heads * T5_REL * sizeof(float)) == cudaSuccess;
    ok &= cudaMalloc(&h->final_g, h->hidden * 2) == cudaSuccess;
    if (!ok) { rsb_bert_free(h); return bfail(RSB_ERR_OOM, "allocating encoder weights failed"); }
    *out = h;
    return RSB_OK;
}

// Replaces `AutoModel.from_pretrained(name)` + `last_hidden_state[:, 0, :]` for RoBERTa checkpoints such as
// DRAGON-RoBERTa's query and context encoders (src/search.py:241-243 and :93-94, src/embed.py:123-126 and :74-78):
// HF RobertaModel = BERT-base layers behind RoBERTa's embedding positions.
extern "C" int rsb_roberta_create(int layers, int inter, int vocab, int max_pos, int type_vocab, float ln_eps,
                                  int padding_idx, rsb_bert_t** out) {
    if (!out) return bfail(RSB_ERR_INVALID, "out is NULL");
    *out = nullptr;
    if (padding_idx < 0 || padding_idx + 2 > max_pos)
        return bfail(RSB_ERR_INVALID, "padding_idx %s%ld leaves no position for a token below max_pos", "", (long)padding_idx);
    if (type_vocab != 1 && type_vocab != 2)
        return bfail(RSB_ERR_UNSUPPORTED, "RoBERTa with type_vocab_size %s%ld: only 1 or 2 are implemented", "", (long)type_vocab);
    rsb_bert_t* h = nullptr;
    const int rc = rsb_bert_create(768, layers, 12, inter, vocab, max_pos, type_vocab, ln_eps, &h);
    if (rc != RSB_OK) return rc;
    h->padding_idx = padding_idx;
    *out = h;
    return RSB_OK;
}

extern "C" int rsb_bert_free(rsb_bert_t* h) {
    if (!h) return RSB_OK;
    cudaFree(h->word); cudaFree(h->pos); cudaFree(h->type); cudaFree(h->emb_g); cudaFree(h->emb_b);
    cudaFree(h->bucket); cudaFree(h->rel_w); cudaFree(h->relb); cudaFree(h->final_g);
    free_linear(h->dense);
    if (h->side) cudaStreamDestroy(h->side);
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    if (h->ev_join) cudaEventDestroy(h->ev_join);
    cudaFree(h->long_list);
    for (auto& l : h->L) {
        free_linear(l.qkv); free_linear(l.attn_out); free_linear(l.ffn1); free_linear(l.ffn2);
        cudaFree(l.ln1_g); cudaFree(l.ln1_b); cudaFree(l.ln2_g); cudaFree(l.ln2_b);
    }
    delete h;
    return RSB_OK;
}

// HF T5EncoderModel keys.  relative_position_bucket is int32 [1023]: the bucket of r = key - query = -511..511.
template <class Put>
static int t5_load(rsb_bert* h, const std::string& s, const void* dev_ptr, int64_t n, cudaStream_t st, Put put) {
    const int H = h->hidden;
    auto expand = [&]() -> int {                         // once both bias tables are present
        if (h->bucket_loaded && h->rel_w_loaded) {
            t5_bias_expand_kernel<<<(h->heads * T5_REL + 255) / 256, 256, 0, st>>>(h->bucket, h->rel_w, h->heads, h->relb);
            if (cudaPeekAtLastError() != cudaSuccess) return bfail(RSB_ERR_CUDA, "bias table expansion failed");
        }
        return RSB_OK;
    };
    if (s == "shared.weight" || s == "encoder.embed_tokens.weight") return put(h->word, (int64_t)h->vocab * H);
    if (s == "encoder.final_layer_norm.weight") return put(h->final_g, H);
    if (s == "relative_position_bucket") {
        if (n != T5_REL) return bfail(RSB_ERR_INVALID, "relative_position_bucket needs 1023 int32 entries%s (got %ld)", "", (long)n);
        std::vector<int> hb(T5_REL);
        if (cudaMemcpyAsync(hb.data(), dev_ptr, T5_REL * sizeof(int), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
            cudaStreamSynchronize(st) != cudaSuccess)
            return bfail(RSB_ERR_CUDA, "copy of relative_position_bucket failed");
        for (int v : hb)
            if (v < 0 || v >= h->num_buckets) return bfail(RSB_ERR_INVALID, "relative_position_bucket entry %s%ld is outside [0, num_buckets)", "", (long)v);
        if (cudaMemcpyAsync(h->bucket, hb.data(), T5_REL * sizeof(int), cudaMemcpyHostToDevice, st) != cudaSuccess ||
            cudaStreamSynchronize(st) != cudaSuccess)
            return bfail(RSB_ERR_CUDA, "copy of relative_position_bucket failed");
        h->bucket_loaded = true;
        return expand();
    }
    int li = -1;
    char rest[128] = {0};
    if (sscanf(s.c_str(), "encoder.block.%d.%127s", &li, rest) == 2 && li >= 0 && li < h->layers) {
        Layer& l = h->L[li];
        std::string r(rest);
        const int64_t HH = (int64_t)H * H;
        if (r == "layer.0.SelfAttention.q.weight") return put(l.qkv.w, HH);
        if (r == "layer.0.SelfAttention.k.weight") return put(l.qkv.w + HH, HH);
        if (r == "layer.0.SelfAttention.v.weight") return put(l.qkv.w + 2 * HH, HH);
        if (r == "layer.0.SelfAttention.o.weight") return put(l.attn_out.w, HH);
        if (r == "layer.0.layer_norm.weight") return put(l.ln1_g, H);
        if (r == "layer.1.DenseReluDense.wi.weight") return put(l.ffn1.w, (int64_t)h->inter * H);
        if (r == "layer.1.DenseReluDense.wo.weight") return put(l.ffn2.w, (int64_t)h->inter * H);
        if (r == "layer.1.layer_norm.weight") return put(l.ln2_g, H);
        if (li == 0 && r == "layer.0.SelfAttention.relative_attention_bias.weight") {   // layer 0's table serves every layer
            const int rc = put(h->rel_w, (int64_t)h->num_buckets * h->heads);
            if (rc != RSB_OK) return rc;
            h->rel_w_loaded = true;
            return expand();
        }
    }
    return bfail(RSB_ERR_INVALID, "unknown weight name %s", s.c_str());
}

// name = HF BertModel state_dict key (SURVEY.md App. B), data = fp16 device pointer, n = element count.
extern "C" int rsb_bert_load(rsb_bert_t* h, const char* name, const void* dev_ptr, int64_t n, rsb_stream_t stream) {
    if (!h || !name || !dev_ptr) return bfail(RSB_ERR_INVALID, "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    const int H = h->hidden;
    auto put = [&](void* dst, int64_t expect) -> int {
        if (n != expect) return bfail(RSB_ERR_INVALID, "weight %s has the wrong size (%ld elements)", name, (long)n);
        return cudaMemcpyAsync(dst, dev_ptr, (size_t)n * 2, cudaMemcpyDeviceToDevice, st) == cudaSuccess
                   ? RSB_OK : bfail(RSB_ERR_CUDA, "copy of %s failed", name);
    };
    std::string s(name);
    if (s == "dense.weight") {
        const int rc = put(h->dense.w, (int64_t)H * H);
        if (rc == RSB_OK) h->dense_loaded = true;
        return rc;
    }
    if (s == "dense.bias") return put(h->dense.b, H);
    if (h->t5) return t5_load(h, s, dev_ptr, n, st, put);
    if (s == "embeddings.word_embeddings.weight") return put(h->word, (int64_t)h->vocab * H);
    if (s == "embeddings.position_embeddings.weight") return put(h->pos, (int64_t)h->max_pos * H);
    if (s == "embeddings.token_type_embeddings.weight") return put(h->type, (int64_t)h->type_vocab * H);
    if (s == "embeddings.LayerNorm.weight") return put(h->emb_g, H);
    if (s == "embeddings.LayerNorm.bias") return put(h->emb_b, H);
    int li = -1;
    char rest[128] = {0};
    if (sscanf(name, "encoder.layer.%d.%127s", &li, rest) == 2 && li >= 0 && li < h->layers) {
        Layer& l = h->L[li];
        std::string r(rest);
        const int64_t HH = (int64_t)H * H;
        if (r == "attention.self.query.weight") return put(l.qkv.w, HH);
        if (r == "attention.self.key.weight") return put(l.qkv.w + HH, HH);
        if (r == "attention.self.value.weight") return put(l.qkv.w + 2 * HH, HH);
        if (r == "attention.self.query.bias") return put(l.qkv.b, H);
        if (r == "attention.self.key.bias") return put(l.qkv.b + H, H);
        if (r == "attention.self.value.bias") return put(l.qkv.b + 2 * H, H);
        if (r == "attention.output.dense.weight") return put(l.attn_out.w, HH);
        if (r == "attention.output.dense.bias") return put(l.attn_out.b, H);
        if (r == "attention.output.LayerNorm.weight") return put(l.ln1_g, H);
        if (r == "attention.output.LayerNorm.bias") return put(l.ln1_b, H);
        if (r == "intermediate.dense.weight") return put(l.ffn1.w, (int64_t)h->inter * H);
        if (r == "intermediate.dense.bias") return put(l.ffn1.b, h->inter);
        if (r == "output.dense.weight") return put(l.ffn2.w, (int64_t)h->inter * H);
        if (r == "output.dense.bias") return put(l.ffn2.b, H);
        if (r == "output.LayerNorm.weight") return put(l.ln2_g, H);
        if (r == "output.LayerNorm.bias") return put(l.ln2_b, H);
    }
    return bfail(RSB_ERR_INVALID, "unknown weight name %s", name);
}

static size_t bert_ws_layout(const rsb_bert* h, int T, size_t off[7]) {
    auto al = [](size_t x) { return (x + 1023) / 1024 * 1024; };   // TMA global addresses: 16 B is enough; keep 1 KB
    const size_t Tp = (size_t)((T + 127) / 128 * 128);
    size_t o = 0;
    off[0] = o; o += al(Tp * h->hidden * 2);        // H (T5: the RMS-normed rows)
    off[1] = o; o += al(Tp * 3 * h->hidden * 2);    // QKV
    off[2] = o; o += al(Tp * h->hidden * 2);        // CTX (after the last layer: the pooled rows the Dense head reads)
    off[3] = o; o += al(Tp * h->hidden * 2);        // TMP (pre-LN sums; T5: the residual stream)
    off[4] = o; o += al(Tp * h->inter * 2);         // FFN intermediate
    off[5] = o; if (h->t5) o += al((size_t)2 * h->layers * sizeof(int));   // T5: one clamp flag per residual add
    off[6] = o;
    return o;
}
extern "C" size_t rsb_bert_workspace_bytes(rsb_bert_t* h, int total_tokens) {
    if (!h) return 0;
    size_t off[7];
    return bert_ws_layout(h, std::max(total_tokens, 1), off);
}

// input_ids / token_type_ids [T] int32 (token_type_ids may be NULL), cu_seqlens [B+1] int32 (all device), out [B, 768] f16
extern "C" int rsb_bert_forward(rsb_bert_t* h, const int32_t* input_ids, const int32_t* token_type_ids,
                                const int32_t* cu_seqlens, int B, int T, int max_seqlen, int pooling, void* out_f16,
                                void* ws, size_t ws_bytes, rsb_stream_t stream) {
    if (!h || !input_ids || !cu_seqlens || !out_f16) return bfail(RSB_ERR_INVALID, "null argument");
    if (B <= 0 || T <= 0) return bfail(RSB_ERR_INVALID, "empty batch");
    if (pooling & ~(RSB_POOL_CLS | RSB_POOL_DENSE | RSB_POOL_NORMALIZE | RSB_POOL_TOKENS)) return bfail(RSB_ERR_INVALID, "unknown pooling bits%s %ld", "", (long)pooling);
    if ((pooling & RSB_POOL_TOKENS) && pooling != RSB_POOL_TOKENS)
        return bfail(RSB_ERR_INVALID, "RSB_POOL_TOKENS cannot be combined with other pooling bits%s (got %ld)", "", (long)pooling);
    if ((pooling & RSB_POOL_DENSE) && !h->dense_loaded) return bfail(RSB_ERR_STATE, "pooling asks for the Dense head but dense.weight was not loaded");
    if (h->t5 && !(h->bucket_loaded && h->rel_w_loaded))
        return bfail(RSB_ERR_STATE, "T5 forward before relative_position_bucket and the relative_attention_bias weight were loaded");
    if (max_seqlen > ATT_MAXS || max_seqlen > h->max_pos)
        return bfail(RSB_ERR_UNSUPPORTED, "sequence longer than %s%ld tokens", "", (long)std::min(ATT_MAXS, h->max_pos));
    const bool roberta = h->padding_idx >= 0;
    if (roberta && h->padding_idx + max_seqlen >= h->max_pos)    // the last token's position is at most padding_idx + S
        return bfail(RSB_ERR_UNSUPPORTED, "RoBERTa positions of a %s%ld-token sequence pass max_position_embeddings",
                     "", (long)max_seqlen);
    size_t off[7];
    const size_t need = bert_ws_layout(h, T, off);
    if (ws_bytes < need) return bfail(RSB_ERR_OOM, "encoder workspace too small (%s need %ld bytes)", "", (long)need);
    cudaStream_t st = (cudaStream_t)stream;
    if (roberta && token_type_ids) {                     // HF raises on a token type outside the table: refuse, not clamp
        std::vector<int32_t> tt(T);
        if (cudaMemcpyAsync(tt.data(), token_type_ids, (size_t)T * sizeof(int32_t), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
            cudaStreamSynchronize(st) != cudaSuccess)
            return bfail(RSB_ERR_CUDA, "copy of token_type_ids failed");
        for (int32_t v : tt)
            if (v < 0 || v >= h->type_vocab)
                return bfail(RSB_ERR_INVALID, "token type %s%ld is outside this RoBERTa handle's type_vocab_size", "", (long)v);
    }
    unsigned char* w = static_cast<unsigned char*>(ws);
    __half* Hs = reinterpret_cast<__half*>(w + off[0]);
    __half* QKV = reinterpret_cast<__half*>(w + off[1]);
    __half* CTX = reinterpret_cast<__half*>(w + off[2]);
    __half* TMP = reinterpret_cast<__half*>(w + off[3]);
    __half* FF = reinterpret_cast<__half*>(w + off[4]);
    int* flags = reinterpret_cast<int*>(w + off[5]);
    h->launches = 0;

    const int rows_per_block = 8;   // 256 threads = 8 warps = 8 rows
    const int ln_grid = (T + rows_per_block - 1) / rows_per_block;
    if (h->t5) {
        embed_gather_kernel<<<ln_grid, 256, 0, st>>>(input_ids, T, h->word, h->vocab, TMP);
        cudaMemsetAsync(flags, 0, (size_t)2 * h->layers * sizeof(int), st);
    } else if (roberta) {
        embed_ln_kernel<true><<<ln_grid, 256, 0, st>>>(input_ids, token_type_ids, cu_seqlens, B, T, h->word, h->pos, h->type,
                                                       h->emb_g, h->emb_b, h->eps, h->vocab, h->max_pos, Hs, h->padding_idx);
    } else {
        embed_ln_kernel<false><<<ln_grid, 256, 0, st>>>(input_ids, token_type_ids, cu_seqlens, B, T, h->word, h->pos, h->type,
                                                        h->emb_g, h->emb_b, h->eps, h->vocab, h->max_pos, Hs, -1);
    }
    h->launches++;
    const int prc = prepare_attention(h, cu_seqlens, B, max_seqlen, st);
    if (prc != RSB_OK) return prc;
    static const bool ln_v1 = getenv("RSB_LN_V1") != nullptr;
    const int ln_rows_grid = std::min(ln_grid, 3 * rsb::device_num_sms());   // 24 warps per SM, ~12 rows per warp at 41k tokens
    auto launch_ln = [&](const __half* x, const __half* g, const __half* b) {
        if (ln_v1) layernorm_kernel<<<ln_grid, 256, 0, st>>>(x, T, g, b, h->eps, Hs);
        else layernorm_rows_kernel<false><<<ln_rows_grid, 256, 0, st>>>(x, T, g, b, h->eps, Hs, nullptr);
    };
    // T5: Hs = rms(X) after the clamp that `flag` (the previous residual add's) calls for
    auto launch_rms = [&](__half* x, const __half* g, const int* flag) {
        layernorm_rows_kernel<true><<<ln_rows_grid, 256, 0, st>>>(x, T, g, nullptr, h->eps, Hs, flag);
    };
    // RSB_BERT_PROFILE=1 (diagnostic): CUDA events between the kernels of the forward, summed per kernel kind over the
    // layers and printed to stderr after each forward -- per-kernel times INSIDE a back-to-back run (ncu's are isolated,
    // cold-cache and at other clocks).  Synchronises the stream; never set in a timed run.  The interval that ends at
    // mark(kind) is counted as `kind`; ln1 / ln2 are the RMS norms before the attention / feed-forward on T5.
    static const bool prof = getenv("RSB_BERT_PROFILE") != nullptr;
    enum { P_QKV, P_ATT, P_AO, P_LN1, P_FFN1, P_FFN2, P_LN2, P_KINDS };
    std::vector<cudaEvent_t> pev;
    std::vector<int> pkind;
    auto mark = [&](int kind) {
        if (!prof) return;
        cudaEvent_t e;
        cudaEventCreate(&e);
        cudaEventRecord(e, st);
        pev.push_back(e);
        pkind.push_back(kind);
    };
    const char* gemm_fail = "tensor map encode failed";
    mark(-1);
    for (int li = 0; li < h->layers; ++li) {
        Layer& l = h->L[li];
        if (h->t5) {
            // pre-norm T5 block on the residual stream X = TMP:  X += o(attn(rms(X))), clamp;  X += wo(relu(wi(rms(X)))), clamp
            // (the clamps are applied by the RMS norm that reads the add's flag)
            launch_rms(TMP, l.ln1_g, li > 0 ? flags + 2 * li - 1 : nullptr);
            mark(P_LN1);
            if (launch_gemm<EPI_BIAS>(Hs, T, l.qkv, QKV, nullptr, st) != RSB_OK) return bfail(RSB_ERR_CUDA, gemm_fail);
            mark(P_QKV);
            launch_attention(h, QKV, cu_seqlens, B, max_seqlen, CTX, st);
            mark(P_ATT);
            if (launch_gemm<EPI_BIAS_RESIDUAL_INF>(CTX, T, l.attn_out, TMP, TMP, st, false, flags + 2 * li) != RSB_OK)
                return bfail(RSB_ERR_CUDA, gemm_fail);
            mark(P_AO);
            launch_rms(TMP, l.ln2_g, flags + 2 * li);
            mark(P_LN2);
            if (launch_gemm<EPI_BIAS_RELU>(Hs, T, l.ffn1, FF, nullptr, st) != RSB_OK) return bfail(RSB_ERR_CUDA, gemm_fail);
            mark(P_FFN1);
            if (launch_gemm<EPI_BIAS_RESIDUAL_INF>(FF, T, l.ffn2, TMP, TMP, st, true, flags + 2 * li + 1) != RSB_OK)
                return bfail(RSB_ERR_CUDA, gemm_fail);
            mark(P_FFN2);
        } else {
            if (launch_gemm<EPI_BIAS>(Hs, T, l.qkv, QKV, nullptr, st) != RSB_OK) return bfail(RSB_ERR_CUDA, gemm_fail);
            mark(P_QKV);
            launch_attention(h, QKV, cu_seqlens, B, max_seqlen, CTX, st);
            mark(P_ATT);
            if (launch_gemm<EPI_BIAS_RESIDUAL>(CTX, T, l.attn_out, TMP, Hs, st) != RSB_OK) return bfail(RSB_ERR_CUDA, gemm_fail);
            mark(P_AO);
            launch_ln(TMP, l.ln1_g, l.ln1_b);
            mark(P_LN1);
            if (launch_gemm<EPI_BIAS_GELU>(Hs, T, l.ffn1, FF, nullptr, st) != RSB_OK) return bfail(RSB_ERR_CUDA, gemm_fail);
            mark(P_FFN1);
            if (launch_gemm<EPI_BIAS_RESIDUAL>(FF, T, l.ffn2, TMP, Hs, st, true) != RSB_OK) return bfail(RSB_ERR_CUDA, gemm_fail);
            mark(P_FFN2);
            launch_ln(TMP, l.ln2_g, l.ln2_b);
            mark(P_LN2);
        }
        h->launches += 6;   // + the attention launch(es), counted in launch_attention
    }
    if (h->t5) {                                         // the last feed-forward's clamp, then final_layer_norm
        launch_rms(TMP, h->final_g, flags + 2 * h->layers - 1);
        h->launches++;
    }
    // sentence-transformers head: Pooling -> Dense (768 x 768 on the tensor-core GEMM, M = B) -> Normalize
    __half* out = static_cast<__half*>(out_f16);
    if (pooling == RSB_POOL_TOKENS) {                    // diagnostic: the final hidden states themselves, [T, 768], no head
        cudaMemcpyAsync(out, Hs, (size_t)T * h->hidden * 2, cudaMemcpyDeviceToDevice, st);
    } else {
        __half* pooled = (pooling & RSB_POOL_DENSE) ? CTX : out;
        pool_kernel<<<B, 256, 0, st>>>(Hs, cu_seqlens, pooling & RSB_POOL_CLS, pooled);
        h->launches++;
    }
    if (pooling & RSB_POOL_DENSE) {
        if (launch_gemm<EPI_BIAS>(CTX, B, h->dense, out, nullptr, st) != RSB_OK) return bfail(RSB_ERR_CUDA, gemm_fail);
        h->launches++;
    }
    if (pooling & RSB_POOL_NORMALIZE) {
        l2normalize_rows_kernel<<<(B + 7) / 8, 256, 0, st>>>(out, B);
        h->launches++;
    }
    if (prof) {
        cudaStreamSynchronize(st);
        float sum[P_KINDS] = {};
        for (size_t i = 0; i + 1 < pev.size(); ++i) {
            float ms = 0.f;
            cudaEventElapsedTime(&ms, pev[i], pev[i + 1]);
            sum[pkind[i + 1]] += ms;
        }
        for (cudaEvent_t e : pev) cudaEventDestroy(e);
        const float L = (float)h->layers * 1e-3f;
        fprintf(stderr, "[rsb_%s profile] T=%d us/layer: qkv %.1f attn %.1f attn_out %.1f ln1 %.1f ffn1 %.1f ffn2 %.1f ln2 %.1f  (sum %.1f)\n",
                h->t5 ? "t5" : "bert", T, sum[P_QKV] / L, sum[P_ATT] / L, sum[P_AO] / L, sum[P_LN1] / L, sum[P_FFN1] / L,
                sum[P_FFN2] / L, sum[P_LN2] / L, (sum[0] + sum[1] + sum[2] + sum[3] + sum[4] + sum[5] + sum[6]) / L);
    }
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return bfail(RSB_ERR_CUDA, "encoder launch failed: %s", cudaGetErrorString(e));
    return RSB_OK;
}

extern "C" int64_t rsb_bert_launches(rsb_bert_t* h) { return h ? h->launches : 0; }

// diagnostic: one attention step of the forward on a caller's QKV, through the forward's own dispatch
extern "C" int rsb_bert_attention(rsb_bert_t* h, const void* qkv, const int32_t* cu_seqlens, int B, int T, int max_seqlen,
                                  void* ctx, rsb_stream_t stream) {
    if (!h || !qkv || !cu_seqlens || !ctx) return bfail(RSB_ERR_INVALID, "null argument");
    if (B <= 0 || T <= 0) return bfail(RSB_ERR_INVALID, "empty batch");
    if (h->t5 && !(h->bucket_loaded && h->rel_w_loaded))
        return bfail(RSB_ERR_STATE, "T5 attention before relative_position_bucket and the relative_attention_bias weight were loaded");
    if (max_seqlen > ATT_MAXS || max_seqlen > h->max_pos)
        return bfail(RSB_ERR_UNSUPPORTED, "sequence longer than %s%ld tokens", "", (long)std::min(ATT_MAXS, h->max_pos));
    cudaStream_t st = (cudaStream_t)stream;
    h->launches = 0;
    const int rc = prepare_attention(h, cu_seqlens, B, max_seqlen, st);
    if (rc != RSB_OK) return rc;
    launch_attention(h, static_cast<const __half*>(qkv), cu_seqlens, B, max_seqlen, static_cast<__half*>(ctx), st);
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return bfail(RSB_ERR_CUDA, "attention launch failed: %s", cudaGetErrorString(e));
    return RSB_OK;
}

// plain GEMM entry (tests / roofline of the tensor-core kernel): C[M,N] = A[M,K] W[N,K]^T + bias, epilogue as above
// (0 bias, 1 GELU, 2 residual, 3 ReLU), OR-ed with RSB_GEMM_REVERSED to visit the row tiles last-to-first as FFN2 does
namespace {

// rsb_gemm_f16's checks and launch for element type T; bf16 has no ReLU epilogue (only the encoder uses it).
template <typename T>
int gemm_entry(const void* A, const void* W, const void* bias, const void* residual, void* C, int M, int N, int K,
               int epilogue, cudaStream_t st) {
    constexpr bool bf16 = std::is_same<T, __nv_bfloat16>::value;
    if (!A || !W || !bias || !C) return bfail(RSB_ERR_INVALID, "null argument");
    if (M <= 0 || N % G_BN || K % G_BK || N <= 0 || K <= 0) return bfail(RSB_ERR_INVALID, "need N %% 128 == 0 and K %% 64 == 0");
    const bool m_rev = (epilogue & RSB_GEMM_REVERSED) != 0;
    epilogue &= ~RSB_GEMM_REVERSED;
    if (epilogue == EPI_BIAS_RESIDUAL && !residual) return bfail(RSB_ERR_INVALID, "residual is NULL");
    Linear lin;
    lin.w = (__half*)W; lin.b = (__half*)bias; lin.N = N; lin.K = K;
    lin.map_ok = make_map(&lin.map, W, N, K, G_BN, bf16);
    if (!lin.map_ok) return bfail(RSB_ERR_CUDA, "tensor map encode failed");
    const T* a = static_cast<const T*>(A);
    T* c = static_cast<T*>(C);
    int rc;
    if (epilogue == EPI_BIAS) rc = launch_gemm<EPI_BIAS, T>(a, M, lin, c, nullptr, st, m_rev);
    else if (epilogue == EPI_BIAS_GELU) rc = launch_gemm<EPI_BIAS_GELU, T>(a, M, lin, c, nullptr, st, m_rev);
    else if (epilogue == EPI_BIAS_RESIDUAL) rc = launch_gemm<EPI_BIAS_RESIDUAL, T>(a, M, lin, c, static_cast<const T*>(residual), st, m_rev);
    else if constexpr (!bf16) {
        if (epilogue == EPI_BIAS_RELU) rc = launch_gemm<EPI_BIAS_RELU>(a, M, lin, c, nullptr, st, m_rev);
        else return bfail(RSB_ERR_INVALID, "unknown epilogue");
    } else {
        return bfail(RSB_ERR_INVALID, "unknown epilogue (bf16: 0 bias, 1 GELU, 2 residual)");
    }
    if (rc != RSB_OK) return bfail(RSB_ERR_CUDA, "tensor map encode failed");
    cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return bfail(RSB_ERR_CUDA, "gemm launch failed: %s", cudaGetErrorString(e));
    return RSB_OK;
}

}  // namespace

extern "C" int rsb_gemm_f16(const void* A, const void* W, const void* bias, const void* residual, void* C, int M, int N,
                            int K, int epilogue, rsb_stream_t stream) {
    return gemm_entry<__half>(A, W, bias, residual, C, M, N, K, epilogue, (cudaStream_t)stream);
}

int rsb::gemm_bf16(const void* A, const void* W, const void* bias, const void* residual, void* C, int M, int N, int K,
                   int epilogue, cudaStream_t stream) {
    return gemm_entry<__nv_bfloat16>(A, W, bias, residual, C, M, N, K, epilogue, stream);
}
