// rsb_common.cuh -- device helpers shared by all kernels: order-preserving score keys, the shared-memory
// candidate buffer with threshold filtering, and a block-wide bitonic sort.
#ifndef RSB_COMMON_CUH_
#define RSB_COMMON_CUH_

#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace rsb {

typedef unsigned long long u64;

// ---- stored rows: elements c .. c+3 of a row (c % 4 == 0) as fp32 ------------------------------------------
// fp32 rows: one 16-byte load; fp16 rows: one 8-byte load of 4 halves (exact conversion).  The kernels that score
// rows are templated on the row type and run the same fmaf sequence on these values, so an fp16 row and an fp32
// row holding the same (fp16-representable) values give bit-identical scores.
__device__ __forceinline__ float4 load_row4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float4 load_row4(const __half* p) {
    const uint2 u = __ldg(reinterpret_cast<const uint2*>(p));
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
}

// SQ8 decode (faiss ScalarQuantizer QT_8bit, non-uniform): x = vmin + ((c + 0.5f) / 255.f) * vdiff for the code c in
// byte `byte` of w, every operation a separately rounded fp32 op.  c + 0.5 is exact from the bits of 2^23 + c; the
// quotient comes from a reciprocal multiply and one fma correction, which gives the correctly rounded (c + 0.5f) / 255.f
// for each of the 256 codes (a plain reciprocal multiply differs for 191 of them).  __fmul_rn / __fadd_rn keep nvcc
// from contracting the decode.  Used by the SQ8 re-rank store and the IVF-SQ8 list scan.
__device__ __forceinline__ float sq8_decode(unsigned w, unsigned byte, float vmin, float vdiff) {
    constexpr float inv = 1.f / 255.f;
    const float a = __fadd_rn(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7440u | byte)), -8388607.5f);
    const float t = __fmul_rn(a, inv);
    const float u = __fmaf_rn(__fmaf_rn(-t, 255.f, a), inv, t);
    return __fadd_rn(vmin, __fmul_rn(u, vdiff));
}

// ---- order-preserving float <-> uint mapping (larger float => larger uint) -------------------------------
__device__ __forceinline__ unsigned ord_f32(float f) {
    unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float unord_f32(unsigned u) {
    return __uint_as_float((u & 0x80000000u) ? (u ^ 0x80000000u) : ~u);
}
// 64-bit sort key: score in the high word, (0xFFFFFFFF - slot) in the low word, so that a DESCENDING sort
// yields score-descending order with ties broken by ascending slot.
__device__ __forceinline__ u64 make_key(unsigned ord, unsigned slot) {
    return (static_cast<u64>(ord) << 32) | static_cast<u64>(0xFFFFFFFFu - slot);
}
__device__ __forceinline__ unsigned key_ord(u64 k) { return static_cast<unsigned>(k >> 32); }
__device__ __forceinline__ unsigned key_slot(u64 k) { return 0xFFFFFFFFu - static_cast<unsigned>(k); }

__host__ __device__ __forceinline__ int next_pow2(int x) {
    int p = 1;
    while (p < x) p <<= 1;
    return p;
}

// ---- candidate buffer ------------------------------------------------------------------------------------
// keys[cap] in shared memory + a shared counter.  Warps append candidates that beat the running threshold;
// the owner guarantees (by calling block_maybe_compact often enough) that it can never overflow.
// Must be called by all 32 lanes of a warp (uses full-mask ballot/shfl).
__device__ __forceinline__ void warp_append(u64* keys, int* count, bool pass, u64 key) {
    const unsigned mask = __ballot_sync(0xffffffffu, pass);
    if (mask) {
        const int lane = threadIdx.x & 31;
        const int leader = __ffs(mask) - 1;
        int base = 0;
        if (lane == leader) base = atomicAdd(count, __popc(mask));
        base = __shfl_sync(0xffffffffu, base, leader);
        if (pass) keys[base + __popc(mask & ((1u << lane) - 1u))] = key;
    }
}

// ---- block-wide bitonic sort, DESCENDING -------------------------------------------------------------------
// Register variant: thread t owns elements [t*E, (t+1)*E).  Compare-exchange partners at distance < E live in the
// same thread, at distance < 32*E in the same warp (one shuffle), and only the few stages with a partner in
// another warp go through shared memory -- 6 barrier-separated stages instead of 55 for 1024 keys on 256 threads.
template <int E>
__device__ __forceinline__ u64 bitonic_pick(u64 mine, u64 other, int i, int size, int stride) {
    const bool desc = (i & size) == 0, lower = (i & stride) == 0;
    const bool take_max = desc == lower;
    return ((mine < other) == take_max) ? other : mine;
}

template <int E>
__device__ __forceinline__ void block_sort_desc_regs(u64* keys, int P) {
    const int t = threadIdx.x;
    const bool owner = t * E < P;          // P <= E * blockDim.x; threads past P carry dummies
    u64 v[E];
    __syncthreads();
#pragma unroll
    for (int e = 0; e < E; ++e) v[e] = owner ? keys[t * E + e] : 0ull;
    for (int size = 2; size <= P; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            if (stride >= 32 * E) {
                __syncthreads();           // earlier partner reads are done
                if (owner) {
#pragma unroll
                    for (int e = 0; e < E; ++e) keys[t * E + e] = v[e];
                }
                __syncthreads();
                if (owner) {
#pragma unroll
                    for (int e = 0; e < E; ++e) {
                        const int i = t * E + e;
                        v[e] = bitonic_pick<E>(v[e], keys[i ^ stride], i, size, stride);
                    }
                }
            } else if (stride >= E) {
                const int lane_mask = stride / E;
#pragma unroll
                for (int e = 0; e < E; ++e) {
                    const u64 other = __shfl_xor_sync(0xffffffffu, v[e], lane_mask);
                    v[e] = bitonic_pick<E>(v[e], other, t * E + e, size, stride);
                }
            } else {
#pragma unroll
                for (int s = E / 2; s >= 1; s >>= 1) {     // compile-time distances: static register indices
                    if (stride == s) {
#pragma unroll
                        for (int e = 0; e < E; ++e) {
                            if ((e & s) == 0) {
                                const bool desc = ((t * E + e) & size) == 0;
                                const u64 a = v[e], b = v[e | s];
                                if ((a < b) == desc) { v[e] = b; v[e | s] = a; }
                            }
                        }
                    }
                }
            }
        }
    }
    __syncthreads();
    if (owner) {
#pragma unroll
        for (int e = 0; e < E; ++e) keys[t * E + e] = v[e];
    }
    __syncthreads();
}

// Block-wide bitonic sort of keys[0..P) (P a power of two), DESCENDING.  All threads of the block call it.
__device__ __forceinline__ void block_sort_desc(u64* keys, int P) {
    const int tid = threadIdx.x, nt = blockDim.x;
    // The register variant is used for P <= blockDim (one key per thread); for 2..8 keys per thread its shuffles run
    // on the same LSU pipe the look-ups saturate and it executes ~1.7x the instructions, so larger sorts stay on the
    // shared-memory network unless RSB_SORT_REGS_ALL is defined.
#ifndef RSB_SORT_CLASSIC
    if ((nt & (nt - 1)) == 0 && nt >= 32) {                // block-uniform dispatch
        if (P <= nt) { block_sort_desc_regs<1>(keys, P); return; }
#ifdef RSB_SORT_REGS_ALL
        if (P == 2 * nt) { block_sort_desc_regs<2>(keys, P); return; }
        if (P == 4 * nt) { block_sort_desc_regs<4>(keys, P); return; }
        if (P == 8 * nt) { block_sort_desc_regs<8>(keys, P); return; }
#endif
    }
#endif
    for (int size = 2; size <= P; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            __syncthreads();
            for (int i = tid; i < (P >> 1); i += nt) {
                // index of the lower element of the i-th compare-exchange pair for this stride
                const int lo = ((i & ~(stride - 1)) << 1) | (i & (stride - 1));
                const int hi = lo | stride;
                const bool desc = ((lo & size) == 0);
                const u64 a = keys[lo], b = keys[hi];
                if ((a < b) == desc) { keys[lo] = b; keys[hi] = a; }
            }
        }
    }
    __syncthreads();
}

// Sort the current candidates and keep the best k.  Returns the new threshold (ordered uint): the k-th best
// score if at least k candidates exist, else `tau`.  All threads call it; on return *count <= k and
// keys[0..*count) is sorted descending.  Contains barriers on entry and exit.
__device__ __forceinline__ unsigned block_compact(u64* keys, int* count, int k, int cap, unsigned tau) {
    __syncthreads();
    const int n = *count;
    int P = next_pow2(n < 2 ? 2 : n);
    if (P > cap) P = cap;
    for (int i = n + threadIdx.x; i < P; i += blockDim.x) keys[i] = 0ull;
    block_sort_desc(keys, P);  // starts and ends with a barrier
    unsigned t = tau;
    if (n >= k) {
        const unsigned kth = key_ord(keys[k - 1]);
        t = kth > tau ? kth : tau;
    }
    __syncthreads();
    if (threadIdx.x == 0 && n > k) *count = k;
    __syncthreads();
    return t;
}

// Called at a block-uniform point: compacts iff fewer than `need_free` slots remain.  ONE barrier: every thread
// votes with the counter value it sees on arrival.  The counter only grows between compactions and a warp's
// appends (atomics whose return value it consumed) are complete before it arrives, so the last thread to arrive
// sees the final value and the OR of the votes is the decision on the final value -- identical in every thread.
__device__ __forceinline__ unsigned block_maybe_compact(u64* keys, int* count, int k, int cap, int need_free,
                                                        unsigned tau) {
    const int over = __syncthreads_or(*reinterpret_cast<volatile int*>(count) > cap - need_free);
    if (over) tau = block_compact(keys, count, k, cap, tau);
    return tau;
}

// capacity of the candidate buffer for a given k and per-interval slack (power of two, >= k + slack)
__host__ __device__ __forceinline__ int cand_capacity(int k, int slack) { return next_pow2(k + slack); }

}  // namespace rsb
#endif
