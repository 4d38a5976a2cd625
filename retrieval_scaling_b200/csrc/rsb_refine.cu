// rsb_refine.cu -- exact re-ranking of IVF-PQ candidates against a caller-owned re-rank store (faiss IndexRefine /
// IndexRefineFlat::search, reference call site src/indicies/ivf_pq.py:119-123 `get_knn_scores`).
//
//   refine_rows_kernel<T>  per (query, candidate chunk): gather the candidates' rows of the store (T = fp16 or fp32),
//                          score <q, x_id> in fp32, sort the chunk's keys (score desc, id asc) and either write the
//                          final (D, I) row (one chunk per query) or the chunk's top-k keys for merge_items_flat_kernel.
//
// The kernel is bound by gather bandwidth: every candidate row is read once per query (nq * k' * d * elem_bytes bytes
// per batch) and used for one dot product.  A warp scores RF_ROWS rows at a time and issues all of their 16-byte loads
// before it consumes any of them, so each warp keeps several rows in flight; the query lives in shared memory.
#include "rsb_common.cuh"
#include "rsb_internal.h"

#include <cuda_fp16.h>
#include <float.h>

#include <algorithm>

namespace rsb {

constexpr int RF_THREADS = 256, RF_WARPS = RF_THREADS / 32, RF_ROWS = 4;
constexpr int RF_MIN_CHUNK = 256;     // candidates per CTA below which splitting a query stops paying

// A lane takes 8 consecutive elements per step (one 16-byte load of fp16, two of fp32) and adds them in element
// order, so both store types sum in the same order: equal decoded values give bit-identical scores.
constexpr int RF_E = 8;
template <typename T> struct Loads { static constexpr int n = RF_E * (int)sizeof(T) / 16; };

__device__ __forceinline__ float dot8(const uint4 (&v)[2], const float* qs, float acc, float) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const float4 a = *reinterpret_cast<const float4*>(qs + 4 * j);
        acc = fmaf(__uint_as_float(v[j].x), a.x, acc); acc = fmaf(__uint_as_float(v[j].y), a.y, acc);
        acc = fmaf(__uint_as_float(v[j].z), a.z, acc); acc = fmaf(__uint_as_float(v[j].w), a.w, acc);
    }
    return acc;
}
__device__ __forceinline__ float dot8(const uint4 (&v)[1], const float* qs, float acc, __half) {
    const float4 a = *reinterpret_cast<const float4*>(qs);
    const float4 b = *reinterpret_cast<const float4*>(qs + 4);
    const float2 x0 = __half22float2(*reinterpret_cast<const __half2*>(&v[0].x));
    const float2 x1 = __half22float2(*reinterpret_cast<const __half2*>(&v[0].y));
    const float2 x2 = __half22float2(*reinterpret_cast<const __half2*>(&v[0].z));
    const float2 x3 = __half22float2(*reinterpret_cast<const __half2*>(&v[0].w));
    acc = fmaf(x0.x, a.x, acc); acc = fmaf(x0.y, a.y, acc); acc = fmaf(x1.x, a.z, acc); acc = fmaf(x1.y, a.w, acc);
    acc = fmaf(x2.x, b.x, acc); acc = fmaf(x2.y, b.y, acc); acc = fmaf(x3.x, b.z, acc); acc = fmaf(x3.y, b.w, acc);
    return acc;
}

// grid = (nq, nchunks).  Block (q, c) scores candidates [c * chunk, min(k_base, (c + 1) * chunk)) of query q.
// Candidates with id < 0 (the base search's padding) or id >= ntotal are skipped.
// direct = 1 (nchunks == 1): writes D/I [nq, k_out], padded with (-FLT_MAX, -1).
// direct = 0: writes the chunk's best min(k_item, valid) keys to out_keys[(q * nchunks + c) * k_item ...] and their
// number to out_cnt[q * nchunks + c], for merge_items_flat_kernel.
// Four CTAs per SM (64 registers): without the bound ptxas picks 48 registers for the fp32 form and spills.
template <typename T>
__global__ __launch_bounds__(RF_THREADS, 4)
void refine_rows_kernel(const float* __restrict__ Q, const T* __restrict__ X, int d, int64_t ntotal,
                        const int64_t* __restrict__ cand, int k_base, int chunk, int P, int k_out, int direct,
                        float* __restrict__ D, int64_t* __restrict__ I, u64* __restrict__ out_keys,
                        int* __restrict__ out_cnt) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);                     // [P]
    float* qs = reinterpret_cast<float*>(smem_raw + (size_t)P * 8);   // [d]
    constexpr int NL = Loads<T>::n;                                   // 16-byte loads per lane and step
    const int q = blockIdx.x, c = blockIdx.y, nchunks = gridDim.y;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int j0 = c * chunk;
    const int n = min(chunk, k_base - j0);
    for (int e = tid * 4; e < d; e += RF_THREADS * 4)
        *reinterpret_cast<float4*>(qs + e) = *reinterpret_cast<const float4*>(Q + (size_t)q * d + e);
    for (int i = tid; i < P; i += RF_THREADS) keys[i] = 0ull;
    __syncthreads();
    const int64_t* ids = cand + (size_t)q * k_base + j0;
    for (int r0 = warp * RF_ROWS; r0 < n; r0 += RF_WARPS * RF_ROWS) {
        int64_t id[RF_ROWS];
        bool ok[RF_ROWS];
        const uint4* row[RF_ROWS];
        float acc[RF_ROWS];
#pragma unroll
        for (int r = 0; r < RF_ROWS; ++r) {
            id[r] = r0 + r < n ? ids[r0 + r] : -1;
            ok[r] = id[r] >= 0 && id[r] < ntotal;                     // warp-uniform
            row[r] = reinterpret_cast<const uint4*>(X + (size_t)(ok[r] ? id[r] : 0) * d);
            acc[r] = 0.f;
        }
        for (int e = lane * RF_E; e < d; e += 32 * RF_E) {
            uint4 v[RF_ROWS][NL];
#pragma unroll
            for (int r = 0; r < RF_ROWS; ++r)
#pragma unroll
                for (int j = 0; j < NL; ++j)
                    v[r][j] = ok[r] ? __ldg(row[r] + e / RF_E * NL + j) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
            for (int r = 0; r < RF_ROWS; ++r) acc[r] = dot8(v[r], qs + e, acc[r], T());
        }
#pragma unroll
        for (int r = 0; r < RF_ROWS; ++r) {
            for (int o = 16; o > 0; o >>= 1) acc[r] += __shfl_xor_sync(0xffffffffu, acc[r], o);
            if (lane == 0 && ok[r]) keys[r0 + r] = make_key(ord_f32(acc[r]), (unsigned)id[r]);
        }
    }
    block_sort_desc(keys, P);                                         // valid keys are non-zero: they sort first
    if (direct) {
        for (int i = tid; i < k_out; i += RF_THREADS) {
            const u64 key = i < P ? keys[i] : 0ull;
            D[(size_t)q * k_out + i] = key ? unord_f32(key_ord(key)) : -FLT_MAX;
            I[(size_t)q * k_out + i] = key ? (int64_t)key_slot(key) : -1;
        }
        return;
    }
    const int k_item = min(k_out, chunk);
    const size_t item = (size_t)q * nchunks + c;
    for (int i = tid; i < k_item; i += RF_THREADS) {
        const u64 key = keys[i];
        if (key) out_keys[item * k_item + i] = key;
    }
    if (tid == 0) {                                                   // number of valid keys among the first k_item
        int lo = 0, hi = k_item;
        while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (keys[mid]) lo = mid + 1; else hi = mid;
        }
        out_cnt[item] = lo;
    }
}

RefinePlan refine_plan(int nq, int k_base, int k) {
    RefinePlan p;
    // Enough CTAs to cover every SM a few times: small batches split each query's candidates into chunks of at least
    // RF_MIN_CHUNK rows, whose partial top-k lists are merged by merge_items_flat_kernel.
    const int want = 4 * device_num_sms();
    const int max_chunks = std::max(1, k_base / RF_MIN_CHUNK);
    int nchunks = std::max(1, std::min(max_chunks, (want + std::max(nq, 1) - 1) / std::max(nq, 1)));
    p.chunk = (k_base + nchunks - 1) / nchunks;
    p.nchunks = (k_base + p.chunk - 1) / p.chunk;
    p.P = next_pow2(std::max(p.chunk, 2));
    p.k_item = std::min(k, p.chunk);
    p.ws_bytes = p.nchunks > 1 ? (size_t)nq * p.nchunks * ((size_t)p.k_item * 8 + 4) + 16 : 0;
    return p;
}

int launch_refine_rows(const RefinePlan& p, const float* Q, int nq, const void* X, int elem_bytes, int d,
                       int64_t ntotal, const int64_t* cand, int k_base, int k, float* D, int64_t* I, void* ws,
                       cudaStream_t st) {
    if (nq <= 0) return 0;
    const size_t smem = (size_t)p.P * 8 + (size_t)d * 4;
    if (smem > 200 * 1024) return -1;
    const int direct = p.nchunks == 1;
    u64* keys = direct ? nullptr : static_cast<u64*>(ws);
    int* cnt = direct ? nullptr : reinterpret_cast<int*>(static_cast<unsigned char*>(ws) + (size_t)nq * p.nchunks * p.k_item * 8);
    dim3 grid(nq, p.nchunks);
    if (elem_bytes == 2) {
        static PerDeviceSize configured;
        if (smem > 48 * 1024 && configured.raise(smem))
            cudaFuncSetAttribute(refine_rows_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        refine_rows_kernel<__half><<<grid, RF_THREADS, smem, st>>>(Q, static_cast<const __half*>(X), d, ntotal, cand, k_base,
                                                                   p.chunk, p.P, k, direct, D, I, keys, cnt);
    } else {
        static PerDeviceSize configured;
        if (smem > 48 * 1024 && configured.raise(smem))
            cudaFuncSetAttribute(refine_rows_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        refine_rows_kernel<float><<<grid, RF_THREADS, smem, st>>>(Q, static_cast<const float*>(X), d, ntotal, cand, k_base,
                                                                  p.chunk, p.P, k, direct, D, I, keys, cnt);
    }
    if (!direct) launch_merge_items(keys, cnt, nq, p.nchunks, p.k_item, k, nullptr, 0, D, I, st);
    return 0;
}

}  // namespace rsb
