// rsb_refine.cu -- exact re-ranking of IVF-PQ candidates against a caller-owned re-rank store (faiss IndexRefine /
// IndexRefineFlat::search, reference call site src/indicies/ivf_pq.py:119-123 `get_knn_scores`).
//
//   refine_rows_kernel<T>  per (query, candidate chunk): gather the candidates' rows of the store (T = fp16, fp32 or
//                          uint8 SQ8 codes, decoded per element), score <q, x_id> in fp32, sort the chunk's keys (score desc, id asc) and either write the
//                          final (D, I) row (one chunk per query) or the chunk's top-k keys for merge_items_flat_kernel.
//
// The kernel is bound by gather bandwidth: every candidate row is read once per query (nq * k' * d * elem_bytes bytes
// per batch) and used for one dot product.  A warp scores RF_ROWS rows at a time and issues all of their 16-byte loads
// before it consumes any of them, so each warp keeps several rows in flight; the query lives in shared memory.
//
// Tiered store (rows [0, n_dev) in device memory, rows [n_dev, ntotal) in mapped page-locked host memory), per chunk
// of queries whose worst case fits the staging buffer:
//   tier_keys_kernel -> cub radix sort of (host row, candidate position) -> tier_flag_kernel -> cub inclusive scan
//   -> tier_scatter_kernel   every distinct host row of the chunk gets one staging slot; slot[q, j] per candidate
//   gather_host_rows_kernel<T>   copies the distinct host rows over PCIe into the staging buffer, once each
//   refine_rows_kernel<T, true>  as above, reading host-tier rows from the staging buffer
// The distinct-row count stays on the device (the gather grid covers the worst case), so nothing synchronises the host.
#include "rsb_common.cuh"
#include "rsb_internal.h"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cuda_fp16.h>
#include <float.h>
#include <limits.h>

#include <algorithm>

namespace rsb {

constexpr int RF_THREADS = 256, RF_WARPS = RF_THREADS / 32, RF_ROWS = 4;
constexpr int RF_MIN_CHUNK = 256;     // candidates per CTA below which splitting a query stops paying

// A lane takes 8 consecutive elements per step (one 16-byte load of fp16, two of fp32, one 8-byte load of SQ8 codes)
// and adds them in element order, so every store type sums in the same order: equal decoded values give
// bit-identical scores.
constexpr int RF_E = 8;
template <typename T> struct Loads { using V = uint4; static constexpr int n = RF_E * (int)sizeof(T) / 16; };
template <> struct Loads<uint8_t> { using V = uint2; static constexpr int n = 1; };

// dot8(v, qs, acc, T(), sq): acc += <q[e .. e+8), x[e .. e+8)> by fmaf in element order.  sq (SQ8 only) points at
// vmin[e] in shared memory, with vdiff[e] d floats further on (sq_d).
__device__ __forceinline__ float dot8(const uint4 (&v)[2], const float* qs, float acc, float, const float*, int) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const float4 a = *reinterpret_cast<const float4*>(qs + 4 * j);
        acc = fmaf(__uint_as_float(v[j].x), a.x, acc); acc = fmaf(__uint_as_float(v[j].y), a.y, acc);
        acc = fmaf(__uint_as_float(v[j].z), a.z, acc); acc = fmaf(__uint_as_float(v[j].w), a.w, acc);
    }
    return acc;
}
__device__ __forceinline__ float dot8(const uint4 (&v)[1], const float* qs, float acc, __half, const float*, int) {
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

// SQ8 codes: sq8_decode (rsb_common.cuh) per element, then the same fmaf.
__device__ __forceinline__ float dot8(const uint2 (&v)[1], const float* qs, float acc, uint8_t, const float* sq,
                                      int sq_d) {
#pragma unroll
    for (int j = 0; j < 2; ++j) {
        const unsigned w = j ? v[0].y : v[0].x;
        const float4 a = *reinterpret_cast<const float4*>(qs + 4 * j);
        const float4 lo = *reinterpret_cast<const float4*>(sq + 4 * j);
        const float4 df = *reinterpret_cast<const float4*>(sq + sq_d + 4 * j);
        acc = fmaf(sq8_decode(w, 0, lo.x, df.x), a.x, acc); acc = fmaf(sq8_decode(w, 1, lo.y, df.y), a.y, acc);
        acc = fmaf(sq8_decode(w, 2, lo.z, df.z), a.z, acc); acc = fmaf(sq8_decode(w, 3, lo.w, df.w), a.w, acc);
    }
    return acc;
}

// grid = (nq, nchunks).  Block (q, c) scores candidates [c * chunk, min(k_base, (c + 1) * chunk)) of query q.
// Candidates with id < 0 (the base search's padding) or id >= ntotal are skipped.
// direct = 1 (nchunks == 1): writes D/I [nq, k_out], padded with (-FLT_MAX, -1).
// direct = 0: writes the chunk's best min(k_item, valid) keys to out_keys[(q * nchunks + c) * k_item ...] and their
// number to out_cnt[q * nchunks + c], for merge_items_flat_kernel.
// Four CTAs per SM (64 registers): without the bound ptxas picks 48 registers for the fp32 form and spills.  The SQ8
// form (decode arithmetic, vmin / vdiff operands) spills at 64 registers and runs three CTAs per SM (80 registers).
// TIERED: ids >= n_dev are read from staging + slot[q * k_base + j] * d instead of X + id * d (the key keeps the id);
// the lane mapping and the fmaf order are the same, so a row scores bit-identically from either place.
// T = uint8_t (SQ8 codes): sq [2, d] fp32 (vmin, vdiff) is copied to shared memory after the query, and every element
// is decoded before its fmaf, so the scores are those of an fp32 store holding the decoded rows.
template <typename T, bool TIERED>
__global__ __launch_bounds__(RF_THREADS, sizeof(T) == 1 ? 3 : 4)
void refine_rows_kernel(const float* __restrict__ Q, const T* __restrict__ X, int d, int64_t ntotal,
                        const int64_t* __restrict__ cand, int k_base, int chunk, int P, int k_out, int direct,
                        float* __restrict__ D, int64_t* __restrict__ I, u64* __restrict__ out_keys,
                        int* __restrict__ out_cnt, int64_t n_dev, const T* __restrict__ staging,
                        const int* __restrict__ slot, const float* __restrict__ sq) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);                     // [P]
    float* qs = reinterpret_cast<float*>(smem_raw + (size_t)P * 8);   // [d], then (SQ8) vmin [d], vdiff [d]
    using V = typename Loads<T>::V;
    constexpr int NL = Loads<T>::n;                                   // loads of V per lane and step
    constexpr bool SQ8 = sizeof(T) == 1;
    const int q = blockIdx.x, c = blockIdx.y, nchunks = gridDim.y;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int j0 = c * chunk;
    const int n = min(chunk, k_base - j0);
    for (int e = tid * 4; e < d; e += RF_THREADS * 4)
        *reinterpret_cast<float4*>(qs + e) = *reinterpret_cast<const float4*>(Q + (size_t)q * d + e);
    if (SQ8)
        for (int e = tid * 4; e < 2 * d; e += RF_THREADS * 4)
            *reinterpret_cast<float4*>(qs + d + e) = *reinterpret_cast<const float4*>(sq + e);
    for (int i = tid; i < P; i += RF_THREADS) keys[i] = 0ull;
    __syncthreads();
    const int64_t* ids = cand + (size_t)q * k_base + j0;
    for (int r0 = warp * RF_ROWS; r0 < n; r0 += RF_WARPS * RF_ROWS) {
        int64_t id[RF_ROWS];
        bool ok[RF_ROWS];
        const V* row[RF_ROWS];
        float acc[RF_ROWS];
#pragma unroll
        for (int r = 0; r < RF_ROWS; ++r) {
            id[r] = r0 + r < n ? ids[r0 + r] : -1;
            ok[r] = id[r] >= 0 && id[r] < ntotal;                     // warp-uniform
            const T* src = X + (size_t)(ok[r] ? id[r] : 0) * d;
            if (TIERED && ok[r] && id[r] >= n_dev) src = staging + (size_t)slot[(size_t)q * k_base + j0 + r0 + r] * d;
            row[r] = reinterpret_cast<const V*>(src);
            acc[r] = 0.f;
        }
        for (int e = lane * RF_E; e < d; e += 32 * RF_E) {
            V v[RF_ROWS][NL];
#pragma unroll
            for (int r = 0; r < RF_ROWS; ++r)
#pragma unroll
                for (int j = 0; j < NL; ++j)
                    v[r][j] = ok[r] ? __ldg(row[r] + e / RF_E * NL + j) : V{};
#pragma unroll
            for (int r = 0; r < RF_ROWS; ++r) acc[r] = dot8(v[r], qs + e, acc[r], T(), qs + d + e, d);
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

static size_t refine_smem(const RefinePlan& p, int d, int elem_bytes) {
    return (size_t)p.P * 8 + (size_t)d * 4 * (elem_bytes == 1 ? 3 : 1);
}
bool refine_smem_fits(const RefinePlan& p, int d, int elem_bytes) { return refine_smem(p, d, elem_bytes) <= 200 * 1024; }

// tiered launch: rows id >= s.n_dev are read from staging + slot[q * k_base + j] * d
struct TierArgs {
    const void* staging;
    const int* slot;      // [nq, k_base]
};

template <typename T, bool TIERED>
static void launch_rows(const RefinePlan& p, dim3 grid, size_t smem, const float* Q, const RefineStore& s,
                        const int64_t* cand, int k_base, int k, int direct, float* D, int64_t* I, u64* keys, int* cnt,
                        const TierArgs* tier, cudaStream_t st) {
    static PerDeviceSize configured;
    if (smem > 48 * 1024 && configured.raise(smem))
        cudaFuncSetAttribute(refine_rows_kernel<T, TIERED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    refine_rows_kernel<T, TIERED><<<grid, RF_THREADS, smem, st>>>(
        Q, static_cast<const T*>(s.dev), s.d, s.ntotal, cand, k_base, p.chunk, p.P, k, direct, D, I, keys, cnt,
        s.n_dev, TIERED ? static_cast<const T*>(tier->staging) : nullptr, TIERED ? tier->slot : nullptr, s.sq);
}

template <typename T>
static void launch_rows(const RefinePlan& p, dim3 grid, size_t smem, const float* Q, const RefineStore& s,
                        const int64_t* cand, int k_base, int k, int direct, float* D, int64_t* I, u64* keys, int* cnt,
                        const TierArgs* tier, cudaStream_t st) {
    if (tier) launch_rows<T, true>(p, grid, smem, Q, s, cand, k_base, k, direct, D, I, keys, cnt, tier, st);
    else launch_rows<T, false>(p, grid, smem, Q, s, cand, k_base, k, direct, D, I, keys, cnt, tier, st);
}

// tier: null for the all-device store
static int refine_rows(const RefinePlan& p, const float* Q, int nq, const RefineStore& s, const int64_t* cand,
                       int k_base, int k, float* D, int64_t* I, void* ws, const TierArgs* tier, cudaStream_t st) {
    if (nq <= 0) return 0;
    const size_t smem = refine_smem(p, s.d, s.elem_bytes);
    if (!refine_smem_fits(p, s.d, s.elem_bytes)) return -1;
    const int direct = p.nchunks == 1;
    u64* keys = direct ? nullptr : static_cast<u64*>(ws);
    int* cnt = direct ? nullptr : reinterpret_cast<int*>(static_cast<unsigned char*>(ws) + (size_t)nq * p.nchunks * p.k_item * 8);
    dim3 grid(nq, p.nchunks);
    if (s.elem_bytes == 1)
        launch_rows<uint8_t>(p, grid, smem, Q, s, cand, k_base, k, direct, D, I, keys, cnt, tier, st);
    else if (s.elem_bytes == 2)
        launch_rows<__half>(p, grid, smem, Q, s, cand, k_base, k, direct, D, I, keys, cnt, tier, st);
    else
        launch_rows<float>(p, grid, smem, Q, s, cand, k_base, k, direct, D, I, keys, cnt, tier, st);
    if (!direct) launch_merge_items(keys, cnt, nq, p.nchunks, p.k_item, k, nullptr, 0, D, I, st);
    return 0;
}

int launch_refine_rows(const RefinePlan& p, const float* Q, int nq, const RefineStore& s, const int64_t* cand,
                       int k_base, int k, float* D, int64_t* I, void* ws, cudaStream_t st) {
    return refine_rows(p, Q, nq, s, cand, k_base, k, D, I, ws, nullptr, st);
}

// ---- tiered store: de-duplication of host-tier candidates, staged gather ------------------------------------------
constexpr int TK_THREADS = 256;
constexpr int GH_THREADS = 256, GH_U = 8;     // gather: 8 independent 16-byte loads per thread, all issued before any store

// key = host row (id - n_dev) for a host-tier candidate, n_host (sorts last) for anything else; value = position.
__global__ void tier_keys_kernel(const int64_t* __restrict__ cand, int L, int64_t n_dev, int64_t ntotal, unsigned n_host,
                                 unsigned* __restrict__ keys, int* __restrict__ vals, int* __restrict__ slot) {
    const int i = blockIdx.x * TK_THREADS + threadIdx.x;
    if (i >= L) return;
    const int64_t id = cand[i];
    keys[i] = id >= n_dev && id < ntotal ? (unsigned)(id - n_dev) : n_host;
    vals[i] = i;
    slot[i] = -1;
}

// flag[i] = 1 on the first element of each run of equal host rows (sorted keys)
__global__ void tier_flag_kernel(const unsigned* __restrict__ keys, int L, unsigned n_host, int* __restrict__ flag) {
    const int i = blockIdx.x * TK_THREADS + threadIdx.x;
    if (i >= L) return;
    const unsigned key = keys[i];
    flag[i] = key < n_host && (i == 0 || keys[i - 1] != key);
}

// inc = inclusive scan of flag: the run of element i owns staging slot inc[i] - 1
__global__ void tier_scatter_kernel(const unsigned* __restrict__ keys, const int* __restrict__ vals,
                                    const int* __restrict__ flag, const int* __restrict__ inc, int L, unsigned n_host,
                                    int* __restrict__ slot, unsigned* __restrict__ uniq, int* __restrict__ count,
                                    long long* __restrict__ host_rows) {
    const int i = blockIdx.x * TK_THREADS + threadIdx.x;
    if (i >= L) return;
    const unsigned key = keys[i];
    if (key < n_host) {
        slot[vals[i]] = inc[i] - 1;
        if (flag[i]) uniq[inc[i] - 1] = key;
    }
    if (i == L - 1) {
        *count = inc[i];
        if (host_rows) *host_rows += inc[i];
    }
}

// staging[s] = host[uniq[s]] for s < *count.  The grid covers the worst case (every candidate distinct); blocks past
// the device-side count return at once.  host is the device alias of the mapped host tier (row 0 = store row n_dev).
template <typename T>
__global__ __launch_bounds__(GH_THREADS)
void gather_host_rows_kernel(const uint4* __restrict__ host, const unsigned* __restrict__ uniq,
                             const int* __restrict__ count, int d, uint4* __restrict__ staging) {
    const int row16 = d * (int)sizeof(T) / 16;
    const size_t total = (size_t)*count * row16;
    const size_t b0 = (size_t)blockIdx.x * GH_THREADS * GH_U + threadIdx.x;
    if (b0 - threadIdx.x >= total) return;
    uint4 v[GH_U];
#pragma unroll
    for (int u = 0; u < GH_U; ++u) {
        const size_t e = b0 + (size_t)u * GH_THREADS;
        if (e < total) {
            const size_t r = e / row16;
            v[u] = host[(size_t)uniq[r] * row16 + (e - r * row16)];
        }
    }
#pragma unroll
    for (int u = 0; u < GH_U; ++u) {
        const size_t e = b0 + (size_t)u * GH_THREADS;
        if (e < total) staging[e] = v[u];
    }
}

static size_t al(size_t x) { return (x + 255) / 256 * 256; }

TieredPlan tiered_plan(int nq, int k_base, int k, int d, int elem_bytes, size_t staging_bytes) {
    TieredPlan p{};
    nq = std::max(nq, 1);
    const size_t per_q = (size_t)k_base * d * elem_bytes;
    if (per_q == 0 || staging_bytes < per_q) return p;
    size_t qc = std::min<size_t>(staging_bytes / per_q, (size_t)nq);
    qc = std::min<size_t>(qc, (size_t)(INT_MAX / k_base));
    p.qc = (int)qc;
    const int last = nq % p.qc ? nq % p.qc : p.qc;
    const int L = p.qc * k_base;
    size_t sort_bytes = 0, scan_bytes = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const unsigned*)nullptr, (unsigned*)nullptr,
                                        (const int*)nullptr, (int*)nullptr, L, 0, 32) != cudaSuccess ||
        cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, (const int*)nullptr, (int*)nullptr, L) != cudaSuccess) {
        cudaGetLastError();
        p.qc = 0;
        return p;
    }
    p.cub_bytes = std::max(sort_bytes, scan_bytes);
    p.ref_bytes = std::max(refine_plan(p.qc, k_base, k).ws_bytes, refine_plan(last, k_base, k).ws_bytes);
    p.smem_ok = refine_smem_fits(refine_plan(p.qc, k_base, k), d, elem_bytes) &&
                refine_smem_fits(refine_plan(last, k_base, k), d, elem_bytes);
    const size_t a4 = al((size_t)L * 4);
    p.off_keys = 0;                      // tier keys, then the run flags
    p.off_keys2 = p.off_keys + a4;       // sorted keys
    p.off_vals = p.off_keys2 + a4;       // positions, then the inclusive scan
    p.off_vals2 = p.off_vals + a4;       // sorted positions
    p.off_slot = p.off_vals2 + a4;
    p.off_uniq = p.off_slot + a4;
    p.off_count = p.off_uniq + a4;
    p.off_cub = p.off_count + 256;
    p.off_ref = p.off_cub + al(p.cub_bytes);
    p.off_stage = p.off_ref + al(p.ref_bytes);
    p.total = p.off_stage + al(qc * per_q);
    return p;
}

struct TierProfile {
    bool on = false;
    cudaEvent_t ev[4] = {};
    double ms[3] = {0, 0, 0};
};
static TierProfile g_tier_prof;

int tiered_profile(int enable, double* ms3) {
    TierProfile& t = g_tier_prof;
    if (ms3)
        for (int i = 0; i < 3; ++i) ms3[i] = t.ms[i];
    for (double& m : t.ms) m = 0;
    if (enable && !t.on) {
        for (auto& e : t.ev)
            if (cudaEventCreate(&e) != cudaSuccess) return -1;
    } else if (!enable && t.on) {
        for (auto& e : t.ev) cudaEventDestroy(e);
    }
    t.on = enable != 0;
    return 0;
}

cudaError_t launch_refine_tiered(const TieredPlan& p, const float* Q, int nq, const RefineStore& s, const int64_t* cand,
                                 int k_base, int k, float* D, int64_t* I, void* ws, long long* host_rows,
                                 cudaStream_t st) {
    const int64_t n_dev = s.n_dev, ntotal = s.ntotal;
    const int d = s.d;
    unsigned char* w = static_cast<unsigned char*>(ws);
    unsigned* keys = reinterpret_cast<unsigned*>(w + p.off_keys);
    unsigned* keys2 = reinterpret_cast<unsigned*>(w + p.off_keys2);
    int* flag = reinterpret_cast<int*>(w + p.off_keys);
    int* vals = reinterpret_cast<int*>(w + p.off_vals);
    int* inc = reinterpret_cast<int*>(w + p.off_vals);
    int* vals2 = reinterpret_cast<int*>(w + p.off_vals2);
    int* slot = reinterpret_cast<int*>(w + p.off_slot);
    unsigned* uniq = reinterpret_cast<unsigned*>(w + p.off_uniq);
    int* count = reinterpret_cast<int*>(w + p.off_count);
    void* cub_tmp = w + p.off_cub;
    const unsigned n_host = (unsigned)(ntotal - n_dev);
    int bits = 1;
    while (bits < 32 && ((uint64_t)1 << bits) <= n_host) ++bits;     // n_host itself (the "not host" key) must fit
    uint4* staging = reinterpret_cast<uint4*>(w + p.off_stage);
    TierArgs tier;
    tier.staging = staging;
    tier.slot = slot;
    TierProfile& prof = g_tier_prof;
    const size_t row_bytes = (size_t)d * s.elem_bytes;
    const uint4* host = static_cast<const uint4*>(s.host);
    for (int q0 = 0; q0 < nq; q0 += p.qc) {
        const int nc = std::min(p.qc, nq - q0);
        const int L = nc * k_base;
        const int tb = (L + TK_THREADS - 1) / TK_THREADS;
        const int64_t* cq = cand + (size_t)q0 * k_base;
        if (prof.on) cudaEventRecord(prof.ev[0], st);
        tier_keys_kernel<<<tb, TK_THREADS, 0, st>>>(cq, L, n_dev, ntotal, n_host, keys, vals, slot);
        size_t tmp = p.cub_bytes;
        cudaError_t e = cub::DeviceRadixSort::SortPairs(cub_tmp, tmp, keys, keys2, vals, vals2, L, 0, bits, st);
        if (e != cudaSuccess) return e;
        tier_flag_kernel<<<tb, TK_THREADS, 0, st>>>(keys2, L, n_host, flag);
        tmp = p.cub_bytes;
        e = cub::DeviceScan::InclusiveSum(cub_tmp, tmp, flag, inc, L, st);
        if (e != cudaSuccess) return e;
        tier_scatter_kernel<<<tb, TK_THREADS, 0, st>>>(keys2, vals2, flag, inc, L, n_host, slot, uniq, count, host_rows);
        if (prof.on) cudaEventRecord(prof.ev[1], st);
        const size_t words = (size_t)L * row_bytes / 16;
        const unsigned gb = (unsigned)((words + GH_THREADS * GH_U - 1) / (GH_THREADS * GH_U));
        if (s.elem_bytes == 1)
            gather_host_rows_kernel<uint8_t><<<gb, GH_THREADS, 0, st>>>(host, uniq, count, d, staging);
        else if (s.elem_bytes == 2)
            gather_host_rows_kernel<__half><<<gb, GH_THREADS, 0, st>>>(host, uniq, count, d, staging);
        else
            gather_host_rows_kernel<float><<<gb, GH_THREADS, 0, st>>>(host, uniq, count, d, staging);
        if (prof.on) cudaEventRecord(prof.ev[2], st);
        if (refine_rows(refine_plan(nc, k_base, k), Q + (size_t)q0 * d, nc, s, cq, k_base, k, D + (size_t)q0 * k,
                        I + (size_t)q0 * k, w + p.off_ref, &tier, st) != 0)
            return cudaErrorInvalidConfiguration;       // not reached: the caller checked p.smem_ok
        if (prof.on) {                                  // profiling only: waits for the chunk to read its events
            cudaEventRecord(prof.ev[3], st);
            e = cudaEventSynchronize(prof.ev[3]);
            if (e != cudaSuccess) return e;
            for (int i = 0; i < 3; ++i) {
                float ms = 0.f;
                cudaEventElapsedTime(&ms, prof.ev[i], prof.ev[i + 1]);
                prof.ms[i] += ms;
            }
        }
        e = cudaPeekAtLastError();
        if (e != cudaSuccess) return e;
    }
    return cudaSuccess;
}

// ---- SQ8 store: training (per-dimension min / max) and encoding (faiss ScalarQuantizer QT_8bit, RS_minmax) ---------
constexpr int SQ_THREADS = 256, SQ_SLABS = 1024;

__device__ __forceinline__ float to_f32(float x) { return x; }
__device__ __forceinline__ float to_f32(__half x) { return __half2float(x); }

// while training, sq holds order-preserving keys: ord(min) in [0, d), ord(max) in [d, 2d)
__global__ void sq8_init_kernel(unsigned* __restrict__ sq, int d) {
    const int j = blockIdx.x * SQ_THREADS + threadIdx.x;
    if (j < d) { sq[j] = 0xFFFFFFFFu; sq[d + j] = 0u; }
}

// block (column tile, slab): rows slab, slab + gridDim.y, ... of columns [tile * SQ_THREADS, ...)
template <typename T>
__global__ __launch_bounds__(SQ_THREADS)
void sq8_train_kernel(const T* __restrict__ x, int64_t n, int d, unsigned* __restrict__ sq) {
    const int j = blockIdx.x * SQ_THREADS + threadIdx.x;
    if (j >= d) return;
    float lo = INFINITY, hi = -INFINITY;
    for (int64_t r = blockIdx.y; r < n; r += gridDim.y) {
        const float v = to_f32(x[(size_t)r * d + j]);
        lo = fminf(lo, v);
        hi = fmaxf(hi, v);
    }
    atomicMin(sq + j, ord_f32(lo));
    atomicMax(sq + d + j, ord_f32(hi));
}

// keys -> vmin [d], vdiff = vmax - vmin [d] (fp32)
__global__ void sq8_finish_kernel(float* __restrict__ sq, int d) {
    const int j = blockIdx.x * SQ_THREADS + threadIdx.x;
    if (j >= d) return;
    unsigned* u = reinterpret_cast<unsigned*>(sq);
    const float vmin = unord_f32(u[j]), vmax = unord_f32(u[d + j]);
    sq[j] = vmin;
    sq[d + j] = __fsub_rn(vmax, vmin);
}

// code = (int)(255.f * clamp((x - vmin) / vdiff, 0, 1)), 0 where vdiff == 0; separately rounded fp32 ops.
// list != null (IVF-SQ8 by residual): x is first replaced by the fp32 residual x - centroids[list[row]].
template <typename T>
__global__ __launch_bounds__(SQ_THREADS)
void sq8_encode_kernel(const T* __restrict__ x, size_t total, int d, const float* __restrict__ sq,
                       uint8_t* __restrict__ codes, const int32_t* __restrict__ list,
                       const float* __restrict__ centroids) {
    for (size_t i = (size_t)blockIdx.x * SQ_THREADS + threadIdx.x; i < total; i += (size_t)gridDim.x * SQ_THREADS) {
        const int j = (int)(i % d);
        const float vmin = sq[j], vdiff = sq[d + j];
        float v = to_f32(x[i]);
        if (list) v = __fsub_rn(v, centroids[(size_t)list[i / d] * d + j]);
        float xi = vdiff != 0.f ? __fdiv_rn(__fsub_rn(v, vmin), vdiff) : 0.f;
        xi = xi < 0.f ? 0.f : (xi > 1.f ? 1.f : xi);
        codes[i] = (uint8_t)(int)__fmul_rn(255.f, xi);
    }
}

cudaError_t launch_sq8_train(const void* x, int x_f16, int64_t n, int d, float* sq, cudaStream_t st) {
    unsigned* u = reinterpret_cast<unsigned*>(sq);
    const unsigned tiles = (unsigned)((d + SQ_THREADS - 1) / SQ_THREADS);
    sq8_init_kernel<<<tiles, SQ_THREADS, 0, st>>>(u, d);
    const dim3 grid(tiles, (unsigned)std::min<int64_t>(n, SQ_SLABS));
    if (x_f16) sq8_train_kernel<__half><<<grid, SQ_THREADS, 0, st>>>(static_cast<const __half*>(x), n, d, u);
    else sq8_train_kernel<float><<<grid, SQ_THREADS, 0, st>>>(static_cast<const float*>(x), n, d, u);
    sq8_finish_kernel<<<tiles, SQ_THREADS, 0, st>>>(sq, d);
    return cudaPeekAtLastError();
}

cudaError_t launch_sq8_encode(const void* x, int x_f16, int64_t n, int d, const float* sq, uint8_t* codes,
                              cudaStream_t st, const int32_t* list, const float* centroids) {
    const size_t total = (size_t)n * d;
    const unsigned blocks = (unsigned)std::min<size_t>((total + SQ_THREADS - 1) / SQ_THREADS, 132 * 64);
    if (x_f16)
        sq8_encode_kernel<__half><<<blocks, SQ_THREADS, 0, st>>>(static_cast<const __half*>(x), total, d, sq, codes, list,
                                                                 centroids);
    else
        sq8_encode_kernel<float><<<blocks, SQ_THREADS, 0, st>>>(static_cast<const float*>(x), total, d, sq, codes, list,
                                                                centroids);
    return cudaPeekAtLastError();
}

}  // namespace rsb
