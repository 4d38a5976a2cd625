// rsb_dense.cu -- exact fp32 inner-product scoring (faiss IndexFlatIP semantics; reference call sites
// src/indicies/flat.py:139 and the IVF coarse quantizer inside ivf_flat.py:225 / ivf_pq.py:230) and the top-k
// machinery shared by every index type.
//
//   sgemm_nt_kernel      S[nq, n] = Q[nq, d] . X[n, d]^T   fp32 FMA tiles on the CUDA cores (used when d % 32 != 0,
//                        or when RSB_OPT_COARSE_TENSOR = 0; the default scorers are the wgmma GEMMs of rsb_tf32.cu --
//                        fp16 hi/lo for the coarse quantizer, 3xTF32 for fp32 Flat rows -- followed by
//                        refine_exact_kernel below)
//   select_rows_kernel   per (row, column-split): thread-maxima prefilter + threshold-filtered candidate buffer
//                        -> top-k keys
//   merge_items_kernel   per query: merge the per-item key lists -> D (f32), I (i64)
//   refine_exact_kernel  exact fp32 re-score of tensor-core candidates -> top-k (fp32-exact ids and scores)
//   merge_shards_kernel / merge_shards_peers_kernel   rsb_merge_topk[_peers] (src/search.py:357-367 semantics)
#include "rsb_common.cuh"
#include "rsb_internal.h"

#include <float.h>
#include <stdlib.h>

namespace rsb {

// =============================================================================================================
// SGEMM  C[M,N] = A[M,K] * B[N,K]^T, all row-major with K contiguous.  128x128x16 tiles, 256 threads, each
// thread an 8x8 micro-tile split as 2x2 blocks of 4x4 (rows ty*4+{0..3} and 64+ty*4+{0..3}; same for
// columns) so that the float4 shared-memory reads of a warp are contiguous (bank-conflict free).
// =============================================================================================================
constexpr int BM = 128, BN = 128, BK = 16, PAD = 4;

__global__ __launch_bounds__(256, 2)
void sgemm_nt_kernel(const float* __restrict__ A, int M, const float* __restrict__ B, int N, int K,
                     float* __restrict__ C, int ldc) {
    __shared__ __align__(16) float As[2][BK][BM + PAD];
    __shared__ __align__(16) float Bs[2][BK][BN + PAD];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;

    // global->shared staging: each thread moves 2 float4 of A and 2 of B per k-tile
    const int lrow = tid >> 2;          // 0..63 (+64 for the second)
    const int lk = (tid & 3) * 4;       // 0,4,8,12
    float4 ra[2], rb[2];

    auto gload = [&](int k0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = lrow + h * 64;
            const int k = k0 + lk;
            ra[h] = make_float4(0.f, 0.f, 0.f, 0.f);
            rb[h] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (m0 + row < M && k < K) ra[h] = *reinterpret_cast<const float4*>(A + (size_t)(m0 + row) * K + k);
            if (n0 + row < N && k < K) rb[h] = __ldg(reinterpret_cast<const float4*>(B + (size_t)(n0 + row) * K + k));
        }
    };
    auto sstore = [&](int buf) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int row = lrow + h * 64;
            As[buf][lk + 0][row] = ra[h].x; As[buf][lk + 1][row] = ra[h].y;
            As[buf][lk + 2][row] = ra[h].z; As[buf][lk + 3][row] = ra[h].w;
            Bs[buf][lk + 0][row] = rb[h].x; Bs[buf][lk + 1][row] = rb[h].y;
            Bs[buf][lk + 2][row] = rb[h].z; Bs[buf][lk + 3][row] = rb[h].w;
        }
    };

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    const int nk = (K + BK - 1) / BK;
    gload(0);
    sstore(0);
    __syncthreads();
    for (int kt = 0; kt < nk; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nk) gload((kt + 1) * BK);
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][64 + ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][64 + tx * 4]);
            const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (kt + 1 < nk) {
            sstore(buf ^ 1);
            __syncthreads();
        }
    }

#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int row = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
        if (row >= M) continue;
#pragma unroll
        for (int jh = 0; jh < 2; ++jh) {
            const int col = n0 + jh * 64 + tx * 4;
            float* dst = C + (size_t)row * ldc + col;
            if (col + 3 < N) {
                *reinterpret_cast<float4*>(dst) = make_float4(acc[i][jh * 4 + 0], acc[i][jh * 4 + 1],
                                                              acc[i][jh * 4 + 2], acc[i][jh * 4 + 3]);
            } else {
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (col + j < N) dst[j] = acc[i][jh * 4 + j];
            }
        }
    }
}

void launch_sgemm_nt(const float* A, int M, const float* B, int N, int K, float* C, int ldc, cudaStream_t st) {
    if (M <= 0 || N <= 0) return;
    dim3 grid((N + BN - 1) / BN, (M + BM - 1) / BM);
    sgemm_nt_kernel<<<grid, 256, 0, st>>>(A, M, B, N, K, C, ldc);
}

// =============================================================================================================
// Row-wise top-k select over a score matrix.  grid = (nsplit, nrows); block (s, row) scans columns
// [s*cols_per_split, ...) of `row`, keeps candidates above the running threshold in a shared-memory buffer and
// compacts (bitonic sort, keep k) whenever fewer than 1024 slots remain.  Emits sorted keys.
// =============================================================================================================
constexpr int SEL_THREADS = 256;
constexpr int SEL_SLACK = SEL_THREADS * 4;  // candidates one sweep can add
constexpr int SEL_ROUNDS = 16;              // float4 per thread held in registers per tile
constexpr int SEL_TILE = SEL_SLACK * SEL_ROUNDS;

__global__ __launch_bounds__(SEL_THREADS, 2)
void select_rows_kernel(const float* __restrict__ S, int ncols, int ld, unsigned col_base, int k, int cap,
                        int cols_per_split, u64* __restrict__ out_keys, int* __restrict__ out_cnt,
                        int items_per_row, int item_base) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);
    __shared__ int s_count, s_survivors;
    const int row = blockIdx.y, split = blockIdx.x;
    const int c0 = split * cols_per_split;
    const int c1 = min(ncols, c0 + cols_per_split);
    if (threadIdx.x == 0) s_count = 0;
    __syncthreads();
    unsigned tau = 0u;
    const float* srow = S + (size_t)row * ld;
    // Tiles of SEL_TILE columns are held in registers (16 float4 per thread).  Prefilter: every thread's maximum
    // is an element of the tile, so the k-th largest of the 256 thread maxima is a lower bound of the tile's
    // (hence the row's) k-th best score; only elements at or above it can matter.
    u64* mx = keys + cap;   // 256-entry scratch behind the candidate buffer
    for (int tile = c0; tile < c1; tile += SEL_TILE) {
        float4 v[SEL_ROUNDS];
        // All sixteen 128-bit loads are issued before anything consumes them: with load and use interleaved the
        // in-order issue leaves ONE load in flight per warp.
        // No guards on the loads: c, c0 and ld are multiples of 4 and a row owns ld >= c1 floats, so a float4 at
        // min(c, ld - 4) is always inside the row; lanes past c1 read don't-care values that every use below
        // masks with (c + j < c1).
#pragma unroll
        for (int r = 0; r < SEL_ROUNDS; ++r) {
            const int c = tile + r * SEL_SLACK + threadIdx.x * 4;
            v[r] = __ldg(reinterpret_cast<const float4*>(srow + min(c, ld - 4)));
        }
        unsigned tmax = 0u;
#pragma unroll
        for (int r = 0; r < SEL_ROUNDS; ++r) {
            const int c = tile + r * SEL_SLACK + threadIdx.x * 4;
            if (c < c1) tmax = max(tmax, ord_f32(v[r].x));
            if (c + 1 < c1) tmax = max(tmax, ord_f32(v[r].y));
            if (c + 2 < c1) tmax = max(tmax, ord_f32(v[r].z));
            if (c + 3 < c1) tmax = max(tmax, ord_f32(v[r].w));
        }
        if (k <= SEL_THREADS) {
            __syncthreads();
            mx[threadIdx.x] = static_cast<u64>(tmax) << 32;   // 0 for threads without a valid element
            block_sort_desc(mx, SEL_THREADS);
            const unsigned t0 = key_ord(mx[k - 1]);
            if (t0 > 0u && t0 - 1u > tau) tau = t0 - 1u;      // strict '>' filter below keeps elements == t0
            __syncthreads();
        }
        // How many elements of this tile survive the threshold?  If they all fit in the free part of the candidate
        // buffer (the common case after the prefilter) append them without any intermediate capacity check.
        int mine = 0;
#pragma unroll
        for (int r = 0; r < SEL_ROUNDS; ++r) {
            const int c = tile + r * SEL_SLACK + threadIdx.x * 4;
            mine += (c < c1 && ord_f32(v[r].x) > tau) + (c + 1 < c1 && ord_f32(v[r].y) > tau) +
                    (c + 2 < c1 && ord_f32(v[r].z) > tau) + (c + 3 < c1 && ord_f32(v[r].w) > tau);
        }
        for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
        __syncthreads();                                   // s_survivors free for reuse; s_count stable
        const int held = s_count;                          // read before any warp can start appending again
        if (threadIdx.x == 0) s_survivors = 0;
        __syncthreads();
        if ((threadIdx.x & 31) == 0 && mine) atomicAdd(&s_survivors, mine);
        __syncthreads();
        const bool fits = held + s_survivors <= cap;       // block-uniform
        if (fits) {
#pragma unroll
            for (int r = 0; r < SEL_ROUNDS; ++r) {
                const int c = tile + r * SEL_SLACK + threadIdx.x * 4;
                const float e[4] = {v[r].x, v[r].y, v[r].z, v[r].w};
                unsigned pass = 0u;
#pragma unroll
                for (int j = 0; j < 4; ++j) pass |= ((c + j < c1) && (ord_f32(e[j]) > tau)) ? (1u << j) : 0u;
                // after the prefilter survivors are rare: one vote per round skips the appends for most warps; the
                // append loop stays rolled (it is cold, and sixteen unrolled copies of it bloat the kernel)
                if (__any_sync(0xffffffffu, pass != 0u)) {
#pragma unroll 1
                    for (int j = 0; j < 4; ++j) {
                        const float ej = j == 0 ? e[0] : (j == 1 ? e[1] : (j == 2 ? e[2] : e[3]));
                        warp_append(keys, &s_count, (pass >> j) & 1u, make_key(ord_f32(ej), col_base + (unsigned)(c + j)));
                    }
                }
            }
        } else {
            // Rare (no prefilter because k > 256, or massive ties): sweep the tile again from memory, 1024 columns
            // at a time with a capacity check after each.  Kept as a rolled loop: unrolling it would inline the
            // compaction sixteen times and blow the instruction cache for the common path.
#pragma unroll 1
            for (int r = 0; r < SEL_ROUNDS; ++r) {
                const int c = tile + r * SEL_SLACK + threadIdx.x * 4;
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const bool in = c + j < c1;
                    const unsigned o = in ? ord_f32(srow[c + j]) : 0u;
                    warp_append(keys, &s_count, in && o > tau, make_key(o, col_base + (unsigned)(c + j)));
                }
                tau = block_maybe_compact(keys, &s_count, k, cap, SEL_SLACK, tau);
            }
        }
        tau = block_maybe_compact(keys, &s_count, k, cap, SEL_SLACK, tau);
    }
    block_compact(keys, &s_count, k, cap, tau);
    const int n = min(s_count, k);
    const size_t item = (size_t)row * items_per_row + item_base + split;
    for (int i = threadIdx.x; i < n; i += blockDim.x) out_keys[item * k + i] = keys[i];
    if (threadIdx.x == 0) out_cnt[item] = n;
}

void launch_select_rows(const float* S, int nrows, int ncols, int ld, unsigned col_base, int k, int nsplit,
                        u64* out_keys, int* out_cnt, int items_per_row, int item_base, cudaStream_t st) {
    if (nrows <= 0) return;
    const int cap = cand_capacity(k, SEL_SLACK);
    int cps = (ncols + nsplit - 1) / nsplit;
    cps = (cps + 3) & ~3;
    const size_t smem = (size_t)cap * sizeof(u64) + SEL_THREADS * sizeof(u64);
    static PerDeviceSize configured;
    if (smem > 48 * 1024 && configured.raise(smem))
        cudaFuncSetAttribute(select_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    dim3 grid(nsplit, nrows);
    select_rows_kernel<<<grid, SEL_THREADS, smem, st>>>(S, ncols, ld, col_base, k, cap, cps, out_keys, out_cnt,
                                                       items_per_row, item_base);
}

// =============================================================================================================
// Back end of the fused scorer (rsb_tf32.cu: gemm_ip_tc_kernel<F16, true>).  One block per row: top-kc of the row's
// candidate keys (8 per 128-column half tile) with the thread-maxima prefilter, then the exactness check:
// a dropped element is <= the largest "9th best of a half tile" X of the row, so the result is the row's true
// top-kc iff the kc-th best candidate is strictly greater than X (or nothing was dropped: X == 0).  Rows that fail
// are flagged and re-done exhaustively by exact_rows_kernel.
// =============================================================================================================
__global__ __launch_bounds__(256)
void select_cands_kernel(const u64* __restrict__ cand, int ncand, const unsigned* __restrict__ xbound, int nx, int kc,
                         int cap, u64* __restrict__ out_keys, int* __restrict__ out_cnt, int items_per_row, int item_idx,
                         unsigned char* __restrict__ flags) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);          // [cap], cap >= ncand: can never overflow
    u64* mx = keys + cap;                                  // [256]
    __shared__ int s_count;
    __shared__ unsigned s_x;
    const int row = blockIdx.x;
    const u64* src = cand + (size_t)row * ncand;
    if (threadIdx.x == 0) { s_count = 0; s_x = 0u; }
    u64 tmax = 0ull;
    for (int i = threadIdx.x; i < ncand; i += 256) {
        const u64 key = src[i];
        tmax = key > tmax ? key : tmax;
    }
    unsigned x = 0u;
    for (int i = threadIdx.x; i < nx; i += 256) x = max(x, xbound[(size_t)row * nx + i]);
    for (int o = 16; o > 0; o >>= 1) x = max(x, __shfl_xor_sync(0xffffffffu, x, o));
    mx[threadIdx.x] = tmax;
    __syncthreads();
    if ((threadIdx.x & 31) == 0 && x) atomicMax(&s_x, x);
    block_sort_desc(mx, 256);
    // every thread maximum is a distinct candidate: the kc-th largest of them bounds the row's kc-th best from below
    unsigned tau = 0u;
    if (kc <= 256) {
        const unsigned t0 = key_ord(mx[kc - 1]);
        if (t0 > 1u) tau = t0 - 1u;
    }
    __syncthreads();
    for (int i0 = 0; i0 < ncand; i0 += 256) {              // block-uniform trip count (warp_append needs full warps)
        const int i = i0 + threadIdx.x;
        const u64 key = i < ncand ? src[i] : 0ull;
        warp_append(keys, &s_count, key != 0ull && key_ord(key) > tau, key);
    }
    block_compact(keys, &s_count, kc, cap, tau);           // sorted descending, at most kc left
    const int n = min(s_count, kc);
    const size_t item = (size_t)row * items_per_row + item_idx;
    for (int i = threadIdx.x; i < n; i += 256) out_keys[item * kc + i] = keys[i];
    if (threadIdx.x == 0) {
        out_cnt[item] = n;
        const unsigned X = s_x;
        flags[row] = (X != 0u && (n < kc || key_ord(keys[kc - 1]) <= X)) ? 1 : 0;
    }
}

int launch_select_cands(const u64* cand, int nrows, int ncand, const unsigned* xbound, int nx, int kc, u64* out_keys,
                        int* out_cnt, int items_per_row, int item, unsigned char* flags, cudaStream_t st) {
    if (nrows <= 0) return 0;
    const int cap = next_pow2(max(ncand, 2));
    const size_t smem = (size_t)cap * sizeof(u64) + 256 * sizeof(u64);
    if (smem > 200 * 1024) return -1;
    static PerDeviceSize configured;
    if (smem > 48 * 1024 && configured.raise(smem))
        cudaFuncSetAttribute(select_cands_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    select_cands_kernel<<<nrows, 256, smem, st>>>(cand, ncand, xbound, nx, kc, cap, out_keys, out_cnt, items_per_row,
                                                  item, flags);
    return 0;
}

// Exhaustive fp32 re-do of the flagged rows: one block per row (unflagged rows exit at once), a warp scores one column
// per step (128-bit coalesced loads, query in shared memory), threshold-filtered candidate buffer as in the list scans.
// T = __half: fp16 database rows (Flat with fp16 storage), 8-byte loads, the same lane mapping and fmaf order.
constexpr int XR_THREADS = 256, XR_WARPS = XR_THREADS / 32, XR_CHECK = 16, XR_SLACK = XR_CHECK * XR_WARPS;

template <typename T>
__global__ __launch_bounds__(XR_THREADS)
void exact_rows_kernel(const float* __restrict__ Q, const T* __restrict__ X, int ncols, int d, unsigned col_base,
                       const unsigned char* __restrict__ flags, int kc, int cap, u64* __restrict__ out_keys,
                       int* __restrict__ out_cnt, int items_per_row, int item_idx) {
    const int row = blockIdx.x;
    if (!flags[row]) return;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* qs = reinterpret_cast<float*>(smem_raw);
    u64* keys = reinterpret_cast<u64*>(smem_raw + (((size_t)d * 4 + 15) & ~(size_t)15));
    __shared__ int s_count;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int c = threadIdx.x * 4; c < d; c += XR_THREADS * 4)
        *reinterpret_cast<float4*>(qs + c) = *reinterpret_cast<const float4*>(Q + (size_t)row * d + c);
    if (threadIdx.x == 0) s_count = 0;
    __syncthreads();
    unsigned tau = 0u;
    const int n_iter = (ncols + XR_WARPS - 1) / XR_WARPS;
    for (int it = 0; it < n_iter; ++it) {
        const int col = it * XR_WARPS + warp;
        const bool ok = col < ncols;
        const T* p = X + (size_t)(ok ? col : 0) * d;
        float acc = 0.f;
        for (int c = lane * 4; c < d; c += 128) {
            const float4 xv = load_row4(p + c);
            const float4 qv = *reinterpret_cast<const float4*>(qs + c);
            acc = fmaf(xv.x, qv.x, acc); acc = fmaf(xv.y, qv.y, acc); acc = fmaf(xv.z, qv.z, acc); acc = fmaf(xv.w, qv.w, acc);
        }
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        const unsigned o32 = ord_f32(acc);
        warp_append(keys, &s_count, lane == 0 && ok && o32 > tau, make_key(o32, col_base + (unsigned)col));
        if ((it + 1) % XR_CHECK == 0) tau = block_maybe_compact(keys, &s_count, kc, cap, XR_SLACK, tau);
    }
    block_compact(keys, &s_count, kc, cap, tau);
    const int n = min(s_count, kc);
    const size_t item = (size_t)row * items_per_row + item_idx;
    for (int i = threadIdx.x; i < n; i += XR_THREADS) out_keys[item * kc + i] = keys[i];
    if (threadIdx.x == 0) out_cnt[item] = n;
}

template <typename T>
static void launch_exact_rows_t(const float* Q, int nrows, const T* X, int ncols, int d, unsigned col_base,
                                const unsigned char* flags, int kc, u64* out_keys, int* out_cnt, int items_per_row,
                                int item, cudaStream_t st) {
    const int cap = cand_capacity(kc, XR_SLACK);
    const size_t smem = (((size_t)d * 4 + 15) & ~(size_t)15) + (size_t)cap * 8;
    static PerDeviceSize configured;
    if (smem > 48 * 1024 && configured.raise(smem))
        cudaFuncSetAttribute(exact_rows_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    exact_rows_kernel<T><<<nrows, XR_THREADS, smem, st>>>(Q, X, ncols, d, col_base, flags, kc, cap, out_keys, out_cnt,
                                                         items_per_row, item);
}

void launch_exact_rows(const float* Q, int nrows, const void* X, int elem_bytes, int ncols, int d, unsigned col_base,
                       const unsigned char* flags, int kc, u64* out_keys, int* out_cnt, int items_per_row, int item,
                       cudaStream_t st) {
    if (nrows <= 0 || ncols <= 0) return;
    if (elem_bytes == 2)
        launch_exact_rows_t(Q, nrows, static_cast<const __half*>(X), ncols, d, col_base, flags, kc, out_keys, out_cnt,
                            items_per_row, item, st);
    else
        launch_exact_rows_t(Q, nrows, static_cast<const float*>(X), ncols, d, col_base, flags, kc, out_keys, out_cnt,
                            items_per_row, item, st);
}

// =============================================================================================================
// Merge the sorted per-item key lists of one query into the final (D, I) row.  One block per query.
// slot -> id:  ids == nullptr ? slot + id_offset : ids[slot].
// =============================================================================================================
constexpr int MRG_THREADS = 256;

__global__ __launch_bounds__(MRG_THREADS)
void merge_items_kernel(const u64* __restrict__ keys_in, const int* __restrict__ cnt_in, int nitems, int k_item,
                        int k_out, int cap, const int64_t* __restrict__ ids, int64_t id_offset,
                        float* __restrict__ D, int64_t* __restrict__ I) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);
    __shared__ int s_count;
    const int q = blockIdx.x;
    if (threadIdx.x == 0) s_count = 0;
    __syncthreads();
    unsigned tau = 0u;
    // invariant at the top of every iteration: s_count <= cap - k_item (room for one whole item)
    for (int it = 0; it < nitems; ++it) {
        const size_t item = (size_t)q * nitems + it;
        const int n = cnt_in[item];
        const int nround = (n + 31) & ~31;
        for (int i = threadIdx.x; i < nround; i += blockDim.x) {
            u64 key = 0ull;
            bool pass = false;
            if (i < n) {
                key = keys_in[item * k_item + i];
                pass = key_ord(key) > tau;
            }
            warp_append(keys, &s_count, pass, key);
        }
        tau = block_maybe_compact(keys, &s_count, k_out, cap, k_item, tau);
    }
    block_compact(keys, &s_count, k_out, cap, tau);
    const int n = min(s_count, k_out);
    for (int i = threadIdx.x; i < k_out; i += blockDim.x) {
        float d = -FLT_MAX;
        int64_t id = -1;
        if (i < n) {
            const u64 key = keys[i];
            d = unord_f32(key_ord(key));
            const unsigned slot = key_slot(key);
            id = ids ? ids[slot] : (int64_t)slot + id_offset;
        }
        D[(size_t)q * k_out + i] = d;
        I[(size_t)q * k_out + i] = id;
    }
}

// Default form.  Same result as merge_items_kernel, but the per-item loop -- one dependent
// count load, one key load and one barrier per item, 32 times per query: latency-bound -- is replaced by a prefix sum
// over the item counts and rounds over the flattened candidate range (cap - k_out candidates per round, usually two
// rounds), each thread locating its item by a binary search in shared memory.  On a list-partitioned multi-GPU shard
// most of a query's items are empty, which this form skips for free.
__global__ __launch_bounds__(MRG_THREADS)
void merge_items_flat_kernel(const u64* __restrict__ keys_in, const int* __restrict__ cnt_in, int nitems, int k_item,
                             int k_out, int cap, const int64_t* __restrict__ ids, int64_t id_offset,
                             float* __restrict__ D, int64_t* __restrict__ I) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);
    int* s_off = reinterpret_cast<int*>(keys + cap);              // [nitems + 1] exclusive prefix of the counts
    __shared__ int s_count;
    const int q = blockIdx.x, lane = threadIdx.x & 31;
    if (threadIdx.x < 32) {
        int carry = 0;
        for (int base = 0; base < nitems; base += 32) {
            const int i = base + lane;
            const int c = i < nitems ? cnt_in[(size_t)q * nitems + i] : 0;
            int x = c;
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, x, o);
                if (lane >= o) x += y;
            }
            if (i < nitems) s_off[i] = carry + x - c;
            carry += __shfl_sync(0xffffffffu, x, 31);
        }
        if (lane == 0) { s_off[nitems] = carry; s_count = 0; }
    }
    __syncthreads();
    const int total = s_off[nitems];
    const int chunk = cap - k_out;                                // free slots right after a compaction
    unsigned tau = 0u;
    for (int base = 0; base < total; base += chunk) {
        const int end = min(total, base + chunk);
        for (int i0 = base; i0 < end; i0 += blockDim.x) {         // block-uniform trip count
            const int i = i0 + threadIdx.x;
            u64 key = 0ull;
            bool pass = false;
            if (i < end) {
                int lo = 0, hi = nitems;                          // largest item with s_off[item] <= i
                while (hi - lo > 1) {
                    const int mid = (lo + hi) >> 1;
                    if (s_off[mid] <= i) lo = mid; else hi = mid;
                }
                key = keys_in[((size_t)q * nitems + lo) * k_item + (i - s_off[lo])];
                pass = key_ord(key) > tau;
            }
            warp_append(keys, &s_count, pass, key);
        }
        if (end < total) tau = block_compact(keys, &s_count, k_out, cap, tau);   // back to <= k_out candidates
    }
    block_compact(keys, &s_count, k_out, cap, tau);
    const int n = min(s_count, k_out);
    for (int i = threadIdx.x; i < k_out; i += blockDim.x) {
        float d = -FLT_MAX;
        int64_t id = -1;
        if (i < n) {
            const u64 key = keys[i];
            d = unord_f32(key_ord(key));
            const unsigned slot = key_slot(key);
            id = ids ? ids[slot] : (int64_t)slot + id_offset;
        }
        D[(size_t)q * k_out + i] = d;
        I[(size_t)q * k_out + i] = id;
    }
}

int merge_items_cap(int k_item, int k_out) { return next_pow2(k_out + 2 * k_item); }

void launch_merge_items(const u64* keys, const int* cnt, int nq, int nitems, int k_item, int k_out,
                        const int64_t* ids, int64_t id_offset, float* D, int64_t* I, cudaStream_t st) {
    if (nq <= 0) return;
    const int cap = merge_items_cap(k_item, k_out);
    const size_t smem_f = (size_t)cap * sizeof(u64) + ((size_t)nitems + 1) * sizeof(int);
    if (smem_f <= 200 * 1024) {
        static PerDeviceSize configured_f;
        if (smem_f > 48 * 1024 && configured_f.raise(smem_f))
            cudaFuncSetAttribute(merge_items_flat_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_f);
        merge_items_flat_kernel<<<nq, MRG_THREADS, smem_f, st>>>(keys, cnt, nitems, k_item, k_out, cap, ids, id_offset, D, I);
        return;
    }
    // very many items per query (item offsets do not fit in shared memory): item-by-item form
    const size_t smem = (size_t)cap * sizeof(u64);
    static PerDeviceSize configured;
    if (smem > 48 * 1024 && configured.raise(smem))
        cudaFuncSetAttribute(merge_items_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    merge_items_kernel<<<nq, MRG_THREADS, smem, st>>>(keys, cnt, nitems, k_item, k_out, cap, ids, id_offset, D, I);
}

// =============================================================================================================
// Shard merge (reference src/search.py:357-367): concat per-shard top-k, stable sort by score desc, keep k_out.
// Ties: lower shard first, then lower rank inside the shard  == key low word = 0xFFFFFFFF - (shard*k + rank).
// =============================================================================================================
__global__ __launch_bounds__(MRG_THREADS)
void merge_shards_kernel(const float* __restrict__ D_all, const int64_t* __restrict__ I_all, int nshards, int nq,
                         int k, int k_out, int P, float* __restrict__ D, int64_t* __restrict__ I) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);
    const int q = blockIdx.x;
    const int total = nshards * k;
    for (int i = threadIdx.x; i < P; i += blockDim.x) {
        u64 key = 0ull;
        if (i < total) {
            const int s = i / k, r = i % k;
            const size_t src = ((size_t)s * nq + q) * k + r;
            if (I_all[src] >= 0) key = make_key(ord_f32(D_all[src]), (unsigned)i);
        }
        keys[i] = key;
    }
    block_sort_desc(keys, P);
    for (int i = threadIdx.x; i < k_out; i += blockDim.x) {
        float d = -FLT_MAX;
        int64_t id = -1;
        if (i < P && keys[i] != 0ull) {
            const unsigned pos = key_slot(keys[i]);
            const int s = pos / k, r = pos % k;
            const size_t src = ((size_t)s * nq + q) * k + r;
            d = D_all[src];
            id = I_all[src];
        }
        D[(size_t)q * k_out + i] = d;
        I[(size_t)q * k_out + i] = id;
    }
}

// =============================================================================================================
// Exact fp32 re-score of tensor-core (3xTF32) candidates: for each query, recompute <q, x[id]> with FFMA for the
// k_in candidate rows, sort (score desc, id asc) and keep k_out.  Makes the coarse quantizer's output independent
// of the tensor-core accumulation order (ids/scores as from the CUDA-core path).  T = __half: fp16 rows, same lane
// mapping and fmaf order (scores bit-equal to those of fp32 rows holding the same values).
// =============================================================================================================
template <typename T>
__global__ __launch_bounds__(256)
void refine_exact_kernel(const float* __restrict__ Q, const T* __restrict__ X, int d, const int64_t* __restrict__ I_in,
                         int k_in, int k_out, int P, float* __restrict__ D, int64_t* __restrict__ I,
                         const int64_t* __restrict__ id_map) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);
    float* qs = reinterpret_cast<float*>(smem_raw + (size_t)P * 8);
    const int q = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int c = tid * 4; c < d; c += 256 * 4)
        *reinterpret_cast<float4*>(qs + c) = *reinterpret_cast<const float4*>(Q + (size_t)q * d + c);
    for (int i = k_in + tid; i < P; i += 256) keys[i] = 0ull;
    __syncthreads();
    for (int j = warp; j < k_in; j += 8) {
        const int64_t id = I_in[(size_t)q * k_in + j];
        float acc = 0.f;
        if (id >= 0) {
            const T* x = X + (size_t)id * d;
            for (int c = lane * 4; c < d; c += 128) {
                const float4 xv = load_row4(x + c);
                const float4 qv = *reinterpret_cast<const float4*>(qs + c);
                acc = fmaf(xv.x, qv.x, acc); acc = fmaf(xv.y, qv.y, acc);
                acc = fmaf(xv.z, qv.z, acc); acc = fmaf(xv.w, qv.w, acc);
            }
        }
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) keys[j] = id >= 0 ? make_key(ord_f32(acc), (unsigned)id) : 0ull;
    }
    block_sort_desc(keys, P);
    for (int i = tid; i < k_out; i += 256) {
        float dd = -FLT_MAX;
        int64_t id = -1;
        if (i < P && keys[i] != 0ull) {
            dd = unord_f32(key_ord(keys[i]));
            id = (int64_t)key_slot(keys[i]);
            if (id_map) id = id_map[id];           // row position -> user id (Flat indexes with custom ids)
        }
        D[(size_t)q * k_out + i] = dd;
        I[(size_t)q * k_out + i] = id;
    }
}

template <typename T>
static void launch_refine_exact_t(const float* Q, int nq, const T* X, int d, const int64_t* I_in, int k_in, int k_out,
                                  int P, size_t smem, float* D, int64_t* I, const int64_t* id_map, cudaStream_t st) {
    static PerDeviceSize configured;
    if (smem > 48 * 1024 && configured.raise(smem))
        cudaFuncSetAttribute(refine_exact_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    refine_exact_kernel<T><<<nq, 256, smem, st>>>(Q, X, d, I_in, k_in, k_out, P, D, I, id_map);
}

int launch_refine_exact(const float* Q, int nq, const void* X, int elem_bytes, int d, const int64_t* I_in, int k_in,
                        int k_out, float* D, int64_t* I, const int64_t* id_map, cudaStream_t st) {
    if (nq <= 0) return 0;
    const int P = next_pow2(max(2, k_in));
    const size_t smem = (size_t)P * 8 + (size_t)d * 4;
    if (smem > 200 * 1024) return -1;
    if (elem_bytes == 2)
        launch_refine_exact_t(Q, nq, static_cast<const __half*>(X), d, I_in, k_in, k_out, P, smem, D, I, id_map, st);
    else
        launch_refine_exact_t(Q, nq, static_cast<const float*>(X), d, I_in, k_in, k_out, P, smem, D, I, id_map, st);
    return 0;
}

int launch_merge_shards(const float* D_all, const int64_t* I_all, int nshards, int nq, int k, int k_out, float* D,
                        int64_t* I, cudaStream_t st) {
    if (nq <= 0) return 0;
    const int P = next_pow2(max(2, nshards * k));
    const size_t smem = (size_t)P * sizeof(u64);
    if (smem > 200 * 1024) return -1;
    static PerDeviceSize configured;
    if (smem > 48 * 1024 && configured.raise(smem))
        cudaFuncSetAttribute(merge_shards_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    merge_shards_kernel<<<nq, MRG_THREADS, smem, st>>>(D_all, I_all, nshards, nq, k, k_out, P, D, I);
    return 0;
}

// =============================================================================================================
// Fused gather + merge: same semantics as merge_shards_kernel, but shard s's (scores, ids) are read IN PLACE from
// D_ptrs[s] / I_ptrs[s] -- peer-mapped buffers of the other GPUs (symmetric memory): the loads below are P2P loads
// over NVLink / NVSwitch, so the all-gather never materialises (no NCCL launch, no staging copy).  The caller
// provides the cross-GPU barrier that orders every rank's search before these reads.
// =============================================================================================================
// load shard s's row q (P2P loads for remote shards), build keys, sort; then winner i -> (score, id)
__device__ __forceinline__ void peers_load_sort(const float* const* __restrict__ D_ptrs,
                                                const int64_t* const* __restrict__ I_ptrs, int nshards, int q, int k,
                                                int P, u64* keys) {
    const int total = nshards * k;
    for (int i = threadIdx.x; i < P; i += blockDim.x) {
        u64 key = 0ull;
        if (i < total) {
            const int s = i / k, r = i % k;
            const size_t src = (size_t)q * k + r;
            const int64_t id = I_ptrs[s][src];                       // peer load
            if (id >= 0) key = make_key(ord_f32(D_ptrs[s][src]), (unsigned)i);
        }
        keys[i] = key;
    }
    block_sort_desc(keys, P);
}
__device__ __forceinline__ void peers_winner(const float* const* __restrict__ D_ptrs,
                                             const int64_t* const* __restrict__ I_ptrs, int q, int k, int P,
                                             const u64* keys, int i, float* d, int64_t* id) {
    *d = -FLT_MAX;
    *id = -1;
    if (i < P && keys[i] != 0ull) {
        const unsigned pos = key_slot(keys[i]);
        const int s = pos / k, r = pos % k;
        const size_t src = (size_t)q * k + r;
        *d = D_ptrs[s][src];
        *id = I_ptrs[s][src];
    }
}

__global__ __launch_bounds__(MRG_THREADS)
void merge_shards_peers_kernel(const float* const* __restrict__ D_ptrs, const int64_t* const* __restrict__ I_ptrs,
                               int nshards, int nq, int k, int k_out, int P, float* __restrict__ D,
                               int64_t* __restrict__ I) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);
    const int q = blockIdx.x;
    peers_load_sort(D_ptrs, I_ptrs, nshards, q, k, P, keys);
    for (int i = threadIdx.x; i < k_out; i += blockDim.x) {
        float d;
        int64_t id;
        peers_winner(D_ptrs, I_ptrs, q, k, P, keys, i, &d, &id);
        D[(size_t)q * k_out + i] = d;
        I[(size_t)q * k_out + i] = id;
    }
}

// Query-sliced variant: this GPU merges only queries [q0, q0 + gridDim.x) -- 1/G of the peer traffic and of the
// sorting -- and stores each merged row into EVERY GPU's result buffer (P2P stores), so that after the caller's
// second barrier all GPUs hold the full (nq, k_out) result.  Gather (loads) and broadcast (stores) both ride on
// this one kernel; no NCCL call, no staging buffer.
__global__ __launch_bounds__(MRG_THREADS)
void merge_shards_peers_scatter_kernel(const float* const* __restrict__ D_ptrs,
                                       const int64_t* const* __restrict__ I_ptrs, int nshards, int q0, int k,
                                       int k_out, int P, float* const* __restrict__ D_outs,
                                       int64_t* const* __restrict__ I_outs, int nout) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u64* keys = reinterpret_cast<u64*>(smem_raw);
    const int q = q0 + blockIdx.x;
    peers_load_sort(D_ptrs, I_ptrs, nshards, q, k, P, keys);
    for (int i = threadIdx.x; i < k_out; i += blockDim.x) {
        float d;
        int64_t id;
        peers_winner(D_ptrs, I_ptrs, q, k, P, keys, i, &d, &id);
        const size_t dst = (size_t)q * k_out + i;
        for (int o = 0; o < nout; ++o) {
            D_outs[o][dst] = d;                                      // peer store
            I_outs[o][dst] = id;
        }
    }
}

static int peers_smem_config(const void* fn, int nshards, int k, int* P_out, size_t* smem_out) {
    const int P = next_pow2(max(2, nshards * k));
    const size_t smem = (size_t)P * sizeof(u64);
    if (smem > 200 * 1024) return -1;
    if (smem > 48 * 1024) cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    *P_out = P;
    *smem_out = smem;
    return 0;
}

int launch_merge_shards_peers(const float* const* D_ptrs, const int64_t* const* I_ptrs, int nshards, int nq, int k,
                              int k_out, float* D, int64_t* I, cudaStream_t st) {
    if (nq <= 0) return 0;
    int P;
    size_t smem;
    if (peers_smem_config((const void*)merge_shards_peers_kernel, nshards, k, &P, &smem)) return -1;
    merge_shards_peers_kernel<<<nq, MRG_THREADS, smem, st>>>(D_ptrs, I_ptrs, nshards, nq, k, k_out, P, D, I);
    return 0;
}

int launch_merge_shards_peers_scatter(const float* const* D_ptrs, const int64_t* const* I_ptrs, int nshards, int q0,
                                      int nq_slice, int k, int k_out, float* const* D_outs, int64_t* const* I_outs,
                                      int nout, cudaStream_t st) {
    if (nq_slice <= 0) return 0;
    int P;
    size_t smem;
    if (peers_smem_config((const void*)merge_shards_peers_scatter_kernel, nshards, k, &P, &smem)) return -1;
    merge_shards_peers_scatter_kernel<<<nq_slice, MRG_THREADS, smem, st>>>(D_ptrs, I_ptrs, nshards, q0, k, k_out, P,
                                                                          D_outs, I_outs, nout);
    return 0;
}

}  // namespace rsb
