// rsb_ivf.cu -- inverted-file kernels: the (query, list) work list, the IVF-Flat list scan, and the IVF-PQ path
// (look-up-table build, ADC list scan with conflict-free shared-memory look-ups, residual encoding, interleaved
// code layout).  Replaces faiss IndexIVFFlat.search / IndexIVFPQ.search / .add as called from the reference's
// src/indicies/ivf_flat.py:180,225 and src/indicies/ivf_pq.py:185,230.
#include "rsb_common.cuh"
#include "rsb_internal.h"
#include "rsb_layout.h"
#include "rsb_tc.cuh"

#include <cub/device/device_radix_sort.cuh>

#include <float.h>
#include <stdlib.h>
#include <algorithm>
#include <type_traits>

namespace rsb {

// =============================================================================================================
// (query, list) work list.  A counting sort of the valid pairs into 2*nlist bins: first every query's LEAD pair
// (probe rank 0, its best-scoring list) ordered by list, then all other pairs ordered by list.  Ordering by list
// makes concurrent blocks share a list in L2; scanning the lead lists first gives every query a tight top-k
// threshold before the bulk of its lists is scanned, so those are filtered almost completely.
// =============================================================================================================
size_t pair_work_bytes(int nq, int nprobe, int nlist) {
    size_t b = 0;
    b += ((size_t)(2 * nlist + 1) * 4 + 255) & ~(size_t)255;   // hist
    b += ((size_t)2 * nlist * 4 + 255) & ~(size_t)255;         // cursor
    b += ((size_t)2 * nlist * 4 + 255) & ~(size_t)255;         // icursor
    b += ((size_t)nq * nprobe * 4 + 255) & ~(size_t)255;       // order
    b += ((size_t)nq * nprobe * 8 + 255) & ~(size_t)255;       // items
    b += 256;                                                  // n_items, item_counter, scan_bytes, n_pairs
    return b;
}

PairWork carve_pair_work(void* base, int nq, int nprobe, int nlist) {
    unsigned char* p = static_cast<unsigned char*>(base);
    PairWork w;
    w.hist = reinterpret_cast<int*>(p);      p += ((size_t)(2 * nlist + 1) * 4 + 255) & ~(size_t)255;
    w.cursor = reinterpret_cast<int*>(p);    p += ((size_t)2 * nlist * 4 + 255) & ~(size_t)255;
    w.icursor = reinterpret_cast<int*>(p);   p += ((size_t)2 * nlist * 4 + 255) & ~(size_t)255;
    w.order = reinterpret_cast<int*>(p);     p += ((size_t)nq * nprobe * 4 + 255) & ~(size_t)255;
    w.items = reinterpret_cast<int2*>(p);    p += ((size_t)nq * nprobe * 8 + 255) & ~(size_t)255;
    w.n_items = reinterpret_cast<int*>(p);
    w.item_counter = reinterpret_cast<int*>(p + 16);
    w.scan_bytes = reinterpret_cast<u64*>(p + 32);
    w.n_pairs = reinterpret_cast<int*>(p + 48);
    return w;
}

// Bin of a valid pair.  The LEAD pair of a query is its first (best-ranked) pair whose list is non-empty HERE -- on
// a list-partitioned shard most of a query's lists live on other GPUs, so "probe rank 0" would miss it.  Within
// each half the bins follow list_rank (longest lists first) so that the persistent blocks finish on short items.
// lead_mode 1 (thresholds shared between GPUs): only the query's GLOBALLY best list (probe rank 0) is a lead pair, on the
// GPU that holds it -- that GPU publishes the bound to all peers, and the other GPUs no longer start a cold top-k
// selection of their own for the query (they did on 7 of 8 GPUs, for every query, at the start of every scan).
__device__ __forceinline__ int pair_bin(const int64_t* __restrict__ coarse_ids, const int* __restrict__ list_len,
                                        const int* __restrict__ list_rank, int p, int nprobe, int nlist, int list,
                                        int lead_mode) {
    bool lead = true;
    if (lead_mode == 1) {
        lead = (p % nprobe) == 0;
    } else {
        for (int e = p - p % nprobe; e < p; ++e) {
            const int64_t l = coarse_ids[e];
            if (l >= 0 && l < nlist && list_len[l] > 0) { lead = false; break; }
        }
    }
    const int pos = list_rank ? list_rank[list] : list;
    return lead ? pos : nlist + pos;
}

__global__ void pair_hist_kernel(const int64_t* __restrict__ coarse_ids, int npairs, int nprobe, int nlist,
                                 const int* __restrict__ list_len, const int* __restrict__ list_rank, int* hist,
                                 u64* scan_elems, int lead_mode) {
    u64 local = 0;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < npairs; p += gridDim.x * blockDim.x) {
        const int64_t l = coarse_ids[p];
        if (l >= 0 && l < nlist) {
            const int len = list_len[l];
            if (len > 0) {
                atomicAdd(&hist[pair_bin(coarse_ids, list_len, list_rank, p, nprobe, nlist, (int)l, lead_mode)], 1);
                local += (u64)len;
            }
        }
    }
    // warp reduce then one atomic per warp
    for (int o = 16; o > 0; o >>= 1) local += __shfl_xor_sync(0xffffffffu, local, o);
    if ((threadIdx.x & 31) == 0 && local) atomicAdd(scan_elems, local);
}

// single-block exclusive scan: cursor[l] = sum_{i<l} c(i); *total = sum, where c(i) = hist[i] for i < half and
// ceil(hist[i] / 2) (the number of paired items of a bin) from `half` on
__global__ void pair_scan_kernel(const int* __restrict__ hist, int nlist, int* cursor, int* total, int* total2,
                                 int half) {
    __shared__ int warp_sums[32];
    __shared__ int carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int base = 0; base < nlist; base += blockDim.x) {
        const int i = base + threadIdx.x;
        const int v = i < nlist ? (i < half ? hist[i] : (hist[i] + 1) >> 1) : 0;
        int x = v;
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) warp_sums[warp] = x;
        __syncthreads();
        if (warp == 0) {
            int s = lane < nw ? warp_sums[lane] : 0;
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, s, o);
                if (lane >= o) s += y;
            }
            warp_sums[lane] = s;  // inclusive
        }
        __syncthreads();
        const int carry = carry_s;
        const int wprefix = warp ? warp_sums[warp - 1] : 0;
        if (i < nlist) cursor[i] = carry + wprefix + x - v;
        __syncthreads();
        if (threadIdx.x == 0) carry_s = carry + warp_sums[nw - 1];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        *total = carry_s;
        if (total2) *total2 = carry_s;
    }
}

__global__ void pair_scatter_kernel(const int64_t* __restrict__ coarse_ids, int npairs, int nprobe, int nlist,
                                    const int* __restrict__ list_len, const int* __restrict__ list_rank, int* cursor,
                                    int* order, int lead_mode) {
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < npairs; p += gridDim.x * blockDim.x) {
        const int64_t l = coarse_ids[p];
        if (l >= 0 && l < nlist && list_len[l] > 0)
            order[atomicAdd(&cursor[pair_bin(coarse_ids, list_len, list_rank, p, nprobe, nlist, (int)l, lead_mode)], 1)] = p;
    }
}

// Paired items: the c pairs of a non-lead bin (one list, c different queries) become ceil(c / 2) items of two pairs
// (the last one single when c is odd); lead pairs stay single items.  Bin order -- and so the lead-first, by-list
// order of the work list -- is kept.  After the scatter, cursor[b] is the END of bin b in `order`.
__global__ void pair_items_kernel(const int* __restrict__ hist, const int* __restrict__ cursor,
                                  const int* __restrict__ icursor, const int* __restrict__ order, int nlist,
                                  int2* __restrict__ items) {
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b < 2 * nlist; b += gridDim.x * blockDim.x) {
        const int c = hist[b];
        const int* src = order + (cursor[b] - c);
        int2* dst = items + icursor[b];
        if (b < nlist) {
            for (int i = 0; i < c; ++i) dst[i] = make_int2(src[i], -1);
        } else {
            for (int i = 0; 2 * i < c; ++i) dst[i] = make_int2(src[2 * i], 2 * i + 1 < c ? src[2 * i + 1] : -1);
        }
    }
}

void launch_pair_setup(const int64_t* coarse_ids, int nq, int nprobe, int nlist, const int* list_len,
                       const int* list_rank, PairWork w, cudaStream_t st, int lead_mode, bool paired) {
    const int npairs = nq * nprobe;
    cudaMemsetAsync(w.hist, 0, (size_t)(2 * nlist + 1) * 4, st);
    cudaMemsetAsync(w.n_items, 0, 256, st);  // n_items, item_counter, scan_bytes, n_pairs
    if (npairs == 0) return;
    const int blocks = min(1024, (npairs + 255) / 256);
    pair_hist_kernel<<<blocks, 256, 0, st>>>(coarse_ids, npairs, nprobe, nlist, list_len, list_rank, w.hist,
                                             w.scan_bytes, lead_mode);
    pair_scan_kernel<<<1, 1024, 0, st>>>(w.hist, 2 * nlist, w.cursor, w.n_pairs, paired ? nullptr : w.n_items,
                                         2 * nlist);
    pair_scatter_kernel<<<blocks, 256, 0, st>>>(coarse_ids, npairs, nprobe, nlist, list_len, list_rank, w.cursor,
                                                w.order, lead_mode);
    if (paired) {
        pair_scan_kernel<<<1, 1024, 0, st>>>(w.hist, 2 * nlist, w.icursor, w.n_items, nullptr, nlist);
        pair_items_kernel<<<(2 * nlist + 255) / 256, 256, 0, st>>>(w.hist, w.cursor, w.icursor, w.order, nlist,
                                                                   w.items);
    }
}

// Raise the running threshold of query q to v: locally with atomicMax and, when the thresholds are shared between
// GPUs, on every peer with a relaxed system-scope max-reduction (no return value: the NVLink round trip is never
// waited for).  Called by one thread.  Peers are only written when the local value actually went up.
__device__ __forceinline__ void raise_tau(const ScanArgs& a, int q, unsigned v) {
    const unsigned old = atomicMax(a.tau + q, v);
    if (a.n_peers > 0 && old < v) {
        for (int p = 0; p < a.n_peers; ++p) {
            unsigned* dst = a.tau_peers[p];
            if (dst == a.tau) continue;                                  // this GPU's own array
            asm volatile("red.relaxed.sys.global.max.u32 [%0], %1;" ::"l"(dst + q), "r"(v) : "memory");
        }
    }
}

// =============================================================================================================
// IVF-Flat list scan.  One block per (query, list) item (persistent blocks, dynamic scheduler).  A warp scores
// two stored vectors per step: 128-bit coalesced loads of the vectors, the query staged in shared memory,
// fp32 FMA, a 5-shuffle transposing reduction; scores above the running threshold go to the block's candidate
// buffer.  HBM/L2-bandwidth bound: 4*d bytes per scored vector (fp32 rows) or 2*d (fp16 rows: lane l loads the
// 4 halves of elements 4l + 128j .. +3 with one 8-byte load and runs the fp32 kernel's fmaf sequence on them, so
// scores are bit-identical to those of fp32 rows holding the same values), or d bytes (SQ8 codes, T = uint8_t: lane l
// loads the 4 codes of elements 4l + 128j .. +3 with one 4-byte load, decodes each with sq8_decode from vmin / vdiff
// staged in shared memory after the query, and runs the same fmaf sequence, so scores are bit-identical to those of
// fp32 rows holding the decoded values; by_residual adds the list's coarse score once, after the reduction).
// The rows of list l start at row list_data[l] of `vecs`; the candidate slot (the id lookup) stays a.list_off[l] + v.
// The all-device search passes list_data = a.list_off; a tiered index scans a staging buffer of host lists with their
// staging offsets (launch_ivf_piece_tables).
// =============================================================================================================
constexpr int FS_THREADS = 256;
constexpr int FS_WARPS = FS_THREADS / 32;
constexpr int FS_CHECK = 16;                             // iterations between capacity checks
constexpr int FS_SLACK = FS_CHECK * FS_WARPS * 2;        // candidates appended between checks (256)

// floats of shared memory before the candidate keys: the query [d], then (SQ8) vmin [d] and vdiff [d]
template <typename T> constexpr int fs_smem_rows() { return sizeof(T) == 1 ? 3 : 1; }

template <typename T>
__device__ __forceinline__ void ivfflat_scan_body(ScanArgs a, const float* __restrict__ queries,
                                                  const T* __restrict__ vecs, int d, int cap,
                                                  const int64_t* __restrict__ list_data,
                                                  const float* __restrict__ sq, int by_residual) {
    constexpr bool SQ8 = sizeof(T) == 1;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* qs = reinterpret_cast<float*>(smem_raw);
    u64* keys = reinterpret_cast<u64*>(smem_raw + (((size_t)d * 4 * fs_smem_rows<T>() + 15) & ~(size_t)15));
    __shared__ int s_count, s_item;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n_items = *a.n_items;
    if constexpr (SQ8) {
        for (int c = tid * 4; c < 2 * d; c += FS_THREADS * 4)
            *reinterpret_cast<float4*>(qs + d + c) = *reinterpret_cast<const float4*>(sq + c);
    }
    int cur_q = -1;
    for (;;) {
        __syncthreads();
        if (tid == 0) { s_item = atomicAdd(a.item_counter, 1); s_count = 0; }
        __syncthreads();
        const int item = s_item;
        if (item >= n_items) break;
        const int pair = a.order[item];
        const int q = pair / a.nprobe;
        const int list = (int)a.coarse_ids[pair];
        if (q != cur_q) {
            for (int c = tid * 4; c < d; c += FS_THREADS * 4)
                *reinterpret_cast<float4*>(qs + c) = *reinterpret_cast<const float4*>(queries + (size_t)q * d + c);
            cur_q = q;
        }
        unsigned tau = *reinterpret_cast<volatile unsigned*>(a.tau + q);
        __syncthreads();
        const int len = a.list_len[list];
        const int64_t base = a.list_off[list];
        const int64_t dbase = list_data[list];
        [[maybe_unused]] const float coarse = SQ8 && by_residual ? a.coarse_scores[pair] : 0.f;
        const int n_iter = (len + 2 * FS_WARPS - 1) / (2 * FS_WARPS);
        for (int it = 0; it < n_iter; ++it) {
            const int v0 = (it * FS_WARPS + warp) * 2, v1 = v0 + 1;
            const bool ok0 = v0 < len, ok1 = v1 < len;
            const T* p0 = vecs + (size_t)(dbase + (ok0 ? v0 : 0)) * d;
            const T* p1 = vecs + (size_t)(dbase + (ok1 ? v1 : 0)) * d;
            float a0 = 0.f, a1 = 0.f;
#pragma unroll 6
            for (int c = lane * 4; c < d; c += 128) {
                float4 x0, x1;
                if constexpr (SQ8) {
                    const unsigned w0 = __ldg(reinterpret_cast<const unsigned*>(p0 + c));
                    const unsigned w1 = __ldg(reinterpret_cast<const unsigned*>(p1 + c));
                    const float4 lo = *reinterpret_cast<const float4*>(qs + d + c);
                    const float4 df = *reinterpret_cast<const float4*>(qs + 2 * d + c);
                    x0 = make_float4(sq8_decode(w0, 0, lo.x, df.x), sq8_decode(w0, 1, lo.y, df.y),
                                     sq8_decode(w0, 2, lo.z, df.z), sq8_decode(w0, 3, lo.w, df.w));
                    x1 = make_float4(sq8_decode(w1, 0, lo.x, df.x), sq8_decode(w1, 1, lo.y, df.y),
                                     sq8_decode(w1, 2, lo.z, df.z), sq8_decode(w1, 3, lo.w, df.w));
                } else {
                    x0 = load_row4(p0 + c);
                    x1 = load_row4(p1 + c);
                }
                const float4 qv = *reinterpret_cast<const float4*>(qs + c);
                a0 = fmaf(x0.x, qv.x, a0); a0 = fmaf(x0.y, qv.y, a0); a0 = fmaf(x0.z, qv.z, a0); a0 = fmaf(x0.w, qv.w, a0);
                a1 = fmaf(x1.x, qv.x, a1); a1 = fmaf(x1.y, qv.y, a1); a1 = fmaf(x1.z, qv.z, a1); a1 = fmaf(x1.w, qv.w, a1);
            }
            // transposing reduction: lanes 0-15 end with the total of v0, lanes 16-31 with that of v1
            float keep = (lane & 16) ? a1 : a0;
            const float send = (lane & 16) ? a0 : a1;
            keep += __shfl_xor_sync(0xffffffffu, send, 16);
            keep += __shfl_xor_sync(0xffffffffu, keep, 8);
            keep += __shfl_xor_sync(0xffffffffu, keep, 4);
            keep += __shfl_xor_sync(0xffffffffu, keep, 2);
            keep += __shfl_xor_sync(0xffffffffu, keep, 1);
            if constexpr (SQ8) {
                if (by_residual) keep = __fadd_rn(coarse, keep);     // faiss: coarse_dis + <q, decoded residual>
            }
            const unsigned o = ord_f32(keep);
            const bool mine = (lane == 0 && ok0) || (lane == 16 && ok1);
            const unsigned slot = (unsigned)(base + ((lane & 16) ? v1 : v0));
            warp_append(keys, &s_count, mine && o > tau, make_key(o, slot));
            if ((it + 1) % FS_CHECK == 0) {
                tau = block_maybe_compact(keys, &s_count, a.k, cap, FS_SLACK, tau);
                const unsigned g = *reinterpret_cast<volatile unsigned*>(a.tau + q);
                tau = g > tau ? g : tau;
            }
        }
        tau = block_compact(keys, &s_count, a.k, cap, tau);
        const int n = min(s_count, a.k);
        for (int i = tid; i < n; i += FS_THREADS) a.out_keys[(size_t)pair * a.k + i] = keys[i];
        if (tid == 0) {
            a.out_cnt[pair] = n;
            if (n >= a.k) raise_tau(a, q, key_ord(keys[a.k - 1]));
        }
    }
}

template <typename T>
__global__ __launch_bounds__(FS_THREADS)
void ivfflat_scan_kernel(ScanArgs a, const float* __restrict__ queries, const T* __restrict__ vecs, int d, int cap,
                         const int64_t* __restrict__ list_data) {
    ivfflat_scan_body<T>(a, queries, vecs, d, cap, list_data, nullptr, 0);
}

// SQ8 codes: sq [2, d] = (vmin, vdiff); by_residual != 0 adds a.coarse_scores[pair] to every score of the pair
__global__ __launch_bounds__(FS_THREADS)
void ivfflat_scan_sq8_kernel(ScanArgs a, const float* __restrict__ queries, const uint8_t* __restrict__ vecs, int d,
                             int cap, const int64_t* __restrict__ list_data, const float* __restrict__ sq, int by_residual) {
    ivfflat_scan_body<uint8_t>(a, queries, vecs, d, cap, list_data, sq, by_residual);
}

static int num_sms() { return device_num_sms(); }

template <typename T, typename... Extra>
static void launch_ivfflat_scan_t(void (*kernel)(ScanArgs, const float*, const T*, int, int, const int64_t*, Extra...),
                                  const ScanArgs& a, const float* queries, const T* vecs, int d, int npairs,
                                  const int64_t* list_data, cudaStream_t st, Extra... extra) {
    const int cap = cand_capacity(a.k, FS_SLACK);
    const size_t smem = (((size_t)d * 4 * fs_smem_rows<T>() + 15) & ~(size_t)15) + (size_t)cap * 8;
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    int occ = 1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, FS_THREADS, smem);
    if (occ < 1) occ = 1;
    const int grid = min(npairs, num_sms() * occ);
    kernel<<<grid, FS_THREADS, smem, st>>>(a, queries, vecs, d, cap, list_data, extra...);
}

void launch_ivfflat_scan(const ScanArgs& a, const float* queries, const void* vecs, const int64_t* list_data,
                         int elem_bytes, int d, int nq, cudaStream_t st, const float* sq, bool by_residual) {
    const int npairs = nq * a.nprobe;
    if (npairs == 0) return;
    if (elem_bytes == 1)
        launch_ivfflat_scan_t(ivfflat_scan_sq8_kernel, a, queries, static_cast<const uint8_t*>(vecs), d, npairs,
                              list_data, st, sq, by_residual ? 1 : 0);
    else if (elem_bytes == 2)
        launch_ivfflat_scan_t(ivfflat_scan_kernel<__half>, a, queries, static_cast<const __half*>(vecs), d, npairs,
                              list_data, st);
    else launch_ivfflat_scan_t(ivfflat_scan_kernel<float>, a, queries, static_cast<const float*>(vecs), d, npairs,
                               list_data, st);
}

// ---- tiered IVF-Flat (rsb_reserve_lists) -------------------------------------------------------------------
// flags[l] = 1 for every list l >= l_dev that a valid pair of the batch probes (flags zeroed by the caller)
__global__ void ivf_probed_flags_kernel(const int64_t* __restrict__ coarse_ids, int npairs, int nlist, int l_dev,
                                        const int* __restrict__ list_len, unsigned char* __restrict__ flags) {
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < npairs; p += gridDim.x * blockDim.x) {
        const int64_t l = coarse_ids[p];
        if (l >= l_dev && l < nlist && list_len[l] > 0) flags[l] = 1;
    }
}
void launch_ivf_probed_flags(const int64_t* coarse_ids, int npairs, int nlist, int l_dev, const int* list_len,
                             unsigned char* flags, cudaStream_t st) {
    cudaMemsetAsync(flags, 0, (size_t)nlist, st);
    if (npairs <= 0) return;
    ivf_probed_flags_kernel<<<std::min(1024, (npairs + 255) / 256), 256, 0, st>>>(coarse_ids, npairs, nlist, l_dev,
                                                                                  list_len, flags);
}

// piece `chunk` of the host lists: list_len masked to the lists copied into that chunk, their staging row offsets
__global__ void ivf_piece_tables_kernel(const int* __restrict__ list_len, const int64_t* __restrict__ stage_off,
                                        const int* __restrict__ chunk_of, int nlist, int chunk, int* __restrict__ len_out,
                                        int64_t* __restrict__ data_out) {
    for (int l = blockIdx.x * blockDim.x + threadIdx.x; l < nlist; l += gridDim.x * blockDim.x) {
        const bool in = chunk_of[l] == chunk;
        len_out[l] = in ? list_len[l] : 0;
        data_out[l] = in ? stage_off[l] : 0;
    }
}
void launch_ivf_piece_tables(const int* list_len, const int64_t* stage_off, const int* chunk_of, int nlist, int chunk,
                             int* len_out, int64_t* data_out, cudaStream_t st) {
    ivf_piece_tables_kernel<<<(nlist + 255) / 256, 256, 0, st>>>(list_len, stage_off, chunk_of, nlist, chunk, len_out,
                                                                  data_out);
}

// Build of a reserved index: the i-th row of the batch in list order (sorted_src[i], list sorted_list[i]) goes to slot
// dst_base[l] + (i - batch_start[l]).  Its id goes to ids_slots[slot]; its row to dev_rows[slot] when the slot is in the
// device tier (l < l_dev), else to host_stage[i - host_begin] (the batch's host-tier rows, in list order, for the
// copies to the host tier).  row_bytes % 16 == 0.
__global__ void ivf_place_rows_kernel(const int32_t* __restrict__ sorted_list, const int64_t* __restrict__ sorted_src,
                                      int64_t n, const int64_t* __restrict__ batch_start,
                                      const int64_t* __restrict__ dst_base, int l_dev, int64_t host_begin,
                                      const uint4* __restrict__ src_rows, const int64_t* __restrict__ src_ids,
                                      int row_words, uint4* __restrict__ dev_rows, uint4* __restrict__ host_stage,
                                      int64_t* __restrict__ ids_slots) {
    const int64_t total = n * row_words;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = e / row_words;
        const int w = (int)(e - i * row_words);
        const int l = sorted_list[i];
        const int64_t src = sorted_src[i];
        const int64_t slot = dst_base[l] + (i - batch_start[l]);
        if (w == 0) ids_slots[slot] = src_ids[src];
        const uint4 v = src_rows[src * row_words + w];
        if (l < l_dev) dev_rows[slot * row_words + w] = v;
        else host_stage[(i - host_begin) * row_words + w] = v;
    }
}
void launch_ivf_place_rows(const int32_t* sorted_list, const int64_t* sorted_src, int64_t n, const int64_t* batch_start,
                           const int64_t* dst_base, int l_dev, int64_t host_begin, const void* src_rows,
                           const int64_t* src_ids, int row_bytes, void* dev_rows, void* host_stage, int64_t* ids_slots,
                           cudaStream_t st) {
    if (n <= 0) return;
    const int w = row_bytes / 16;
    const int64_t total = n * w;
    ivf_place_rows_kernel<<<(int)std::min<int64_t>(8192, (total + 255) / 256), 256, 0, st>>>(
        sorted_list, sorted_src, n, batch_start, dst_base, l_dev, host_begin, static_cast<const uint4*>(src_rows),
        src_ids, w, static_cast<uint4*>(dev_rows), static_cast<uint4*>(host_stage), ids_slots);
}

// =============================================================================================================
// PQ look-up tables.  lut[q][j*64 + pos] = < q_m , cb[m][j] >  for pos = m + M*c, c < 64/M  (replicated rows so
// that every warp lane owns a distinct shared-memory bank in the scan kernel, see rsb_layout.h).
// cbT is the codebook transposed to [256][d]:  cbT[j][m*dsub + t] = cb[m][j][t]  (coalesced reads here).
// =============================================================================================================
__global__ void codebook_transpose_kernel(const float* __restrict__ cb, int M, int dsub, float* __restrict__ cbT) {
    const int d = M * dsub;
    const int total = 256 * d;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const int j = i / d, c = i % d;
        const int m = c / dsub, t = c % dsub;
        cbT[i] = cb[((size_t)m * 256 + j) * dsub + t];
    }
}
void launch_codebook_transpose(const float* cb, int M, int dsub, float* cbT, cudaStream_t st) {
    codebook_transpose_kernel<<<256, 256, 0, st>>>(cb, M, dsub, cbT);
}

// LUT_QB = queries per block: every block streams the whole codebook (L2 reads) and uses each entry for LUT_QB
// queries, so larger values cut the L2 traffic; the launcher picks the value whose grid fills whole waves.
template <int LUT_QB>
__global__ __launch_bounds__(256, 2)
void pq_lut_kernel(const float* __restrict__ queries, int nq, int d, int M, const float* __restrict__ cbT,
                   float* __restrict__ lut) {
    extern __shared__ __align__(16) float qs_lut[];   // [LUT_QB][d]
    const int q0 = blockIdx.x * LUT_QB;
    const int nqb = min(LUT_QB, nq - q0);
    const int dsub = d / M;
    for (int c = threadIdx.x; c < LUT_QB * d; c += blockDim.x) {
        const int qq = c / d;
        qs_lut[c] = qq < nqb ? queries[(size_t)(q0 + qq) * d + (c - qq * d)] : 0.f;
    }
    __syncthreads();
    const int reps = kLutRowWords / M;
    if (dsub == 12 && (256 % M) == 0) {
        // fast path (M = 64, d = 768): 256 % M == 0 makes every thread's sub-quantizer m = tid % M loop-invariant,
        // so its LUT_QB query slices (12 floats each) live in registers; the loop then only streams the
        // transposed codebook (coalesced 48-byte reads) and writes coalesced table rows.
        const int m = threadIdx.x % M;
        float x[LUT_QB][12];
#pragma unroll
        for (int qq = 0; qq < LUT_QB; ++qq)
#pragma unroll
            for (int t = 0; t < 12; ++t) x[qq][t] = qs_lut[qq * d + m * 12 + t];
        for (int j = threadIdx.x / M; j < 256; j += blockDim.x / M) {
            const float4* c4 = reinterpret_cast<const float4*>(cbT + (size_t)j * d + m * 12);
            const float4 c0 = __ldg(c4), c1 = __ldg(c4 + 1), c2 = __ldg(c4 + 2);
            const float cv[12] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w, c2.x, c2.y, c2.z, c2.w};
#pragma unroll
            for (int qq = 0; qq < LUT_QB; ++qq) {
                float s = 0.f;
#pragma unroll
                for (int t = 0; t < 12; ++t) s = fmaf(x[qq][t], cv[t], s);
                if (qq < nqb) {
                    float* out = lut + (size_t)(q0 + qq) * kLutWords + j * kLutRowWords + m;
                    for (int r = 0; r < reps; ++r) out[M * r] = s;
                }
            }
        }
        return;
    }
    for (int idx = threadIdx.x; idx < 256 * M; idx += blockDim.x) {
        const int j = idx / M, m = idx % M;
        const float* c = cbT + (size_t)j * d + m * dsub;
        float s[LUT_QB];
#pragma unroll
        for (int qq = 0; qq < LUT_QB; ++qq) s[qq] = 0.f;
        if ((dsub & 3) == 0) {
            for (int t = 0; t < dsub; t += 4) {
                const float4 cv = __ldg(reinterpret_cast<const float4*>(c + t));
#pragma unroll
                for (int qq = 0; qq < LUT_QB; ++qq) {
                    const float* x = qs_lut + qq * d + m * dsub + t;
                    s[qq] = fmaf(x[0], cv.x, s[qq]); s[qq] = fmaf(x[1], cv.y, s[qq]);
                    s[qq] = fmaf(x[2], cv.z, s[qq]); s[qq] = fmaf(x[3], cv.w, s[qq]);
                }
            }
        } else {
            for (int t = 0; t < dsub; ++t) {
                const float cv = __ldg(c + t);
#pragma unroll
                for (int qq = 0; qq < LUT_QB; ++qq) s[qq] = fmaf(qs_lut[qq * d + m * dsub + t], cv, s[qq]);
            }
        }
#pragma unroll
        for (int qq = 0; qq < LUT_QB; ++qq) {
            if (qq < nqb) {
                float* out = lut + (size_t)(q0 + qq) * kLutWords;
                for (int r = 0; r < reps; ++r) out[j * kLutRowWords + m + M * r] = s[qq];
            }
        }
    }
}

// M = 64, dsub = 12 (the BASELINE configuration): codebook-stationary variant.  A block owns 8 code values j for all
// 64 sub-quantizers: every thread keeps the two 12-float codebook entries (j, m), (j+4, m) in registers for its
// whole life and streams queries through shared memory (16 at a time, 48 KB), so the inner loop is 3 conflict-free
// LDS.128 + 24 FMA + 2 coalesced stores per query with no global-memory latency in it.  The query-stationary kernel
// above is latency-bound on the codebook loads; this one is bound by the 64 KB/query table write.
constexpr int L64_QS = 16;

// JT = code values per thread (rows j0 + 4*i of the transposed codebook): 4 instead of 2 halves the shared-memory reads
// of the query sub-vectors per table entry (the kernel's binding pipe) at 48 codebook registers per thread.
template <int JT>
__global__ __launch_bounds__(256, JT == 2 ? 4 : 3)
void pq_lut64_kernel(const float* __restrict__ queries, int nq, int qn, const float* __restrict__ cbT,
                     float* __restrict__ lut) {
    extern __shared__ __align__(16) float qs64[];                  // [L64_QS][768]
    const int m = threadIdx.x & 63, jl = threadIdx.x >> 6;
    const int j0 = blockIdx.x * (4 * JT) + jl;
    float c[JT][12];
#pragma unroll
    for (int i = 0; i < JT; ++i) {
        const float4* p = reinterpret_cast<const float4*>(cbT + (size_t)(j0 + 4 * i) * 768 + m * 12);
#pragma unroll
        for (int v = 0; v < 3; ++v) {
            const float4 a = __ldg(p + v);
            c[i][4 * v] = a.x; c[i][4 * v + 1] = a.y; c[i][4 * v + 2] = a.z; c[i][4 * v + 3] = a.w;
        }
    }
    const int qbeg = blockIdx.y * qn, qend = min(nq, qbeg + qn);
    for (int qb = qbeg; qb < qend; qb += L64_QS) {
        const int nb = min(L64_QS, qend - qb);
        __syncthreads();
        const float4* src = reinterpret_cast<const float4*>(queries + (size_t)qb * 768);   // nb rows are contiguous
        for (int i = threadIdx.x; i < nb * 192; i += 256) reinterpret_cast<float4*>(qs64)[i] = src[i];
        __syncthreads();
#pragma unroll 4
        for (int qq = 0; qq < nb; ++qq) {
            const float4* x4 = reinterpret_cast<const float4*>(qs64 + qq * 768 + m * 12);
            const float4 xa = x4[0], xb = x4[1], xc = x4[2];
            const float x[12] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w, xc.x, xc.y, xc.z, xc.w};
            float* out = lut + (size_t)(qb + qq) * kLutWords + m;
#pragma unroll
            for (int i = 0; i < JT; ++i) {
                float sacc = 0.f;
#pragma unroll
                for (int t = 0; t < 12; ++t) sacc = fmaf(x[t], c[i][t], sacc);   // same summation order as pq_lut_kernel
                out[(j0 + 4 * i) * kLutRowWords] = sacc;
            }
        }
    }
}

template <int JT>
static void launch_pq_lut64_t(const float* queries, int nq, const float* codebook_t, float* lut, cudaStream_t st) {
    const size_t smem = (size_t)L64_QS * 768 * 4;
    static PerDeviceSize configured;
    if (configured.raise(smem))
        cudaFuncSetAttribute(pq_lut64_kernel<JT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    // queries per block: ~256, adjusted so that the grid is a whole number of waves of the resident blocks per SM
    const int jblocks = 256 / (4 * JT);
    const long slots = (JT == 2 ? 4L : 3L) * num_sms();
    const long waves = std::max(1L, (nq * (long)jblocks + slots * 128) / (slots * 256));
    long qn = (nq * (long)jblocks + slots * waves - 1) / (slots * waves);
    qn = std::max<long>(L64_QS, (qn + L64_QS - 1) / L64_QS * L64_QS);
    dim3 grid(jblocks, (unsigned)((nq + qn - 1) / qn));
    pq_lut64_kernel<JT><<<grid, 256, smem, st>>>(queries, nq, (int)qn, codebook_t, lut);
}
static void launch_pq_lut64(const float* queries, int nq, const float* codebook_t, float* lut, cudaStream_t st) {
    static const bool jt2 = getenv("RSB_LUT_JT2") != nullptr;      // A/B switch: round-1 form (2 code values per thread)
    if (jt2) launch_pq_lut64_t<2>(queries, nq, codebook_t, lut, st);
    else launch_pq_lut64_t<4>(queries, nq, codebook_t, lut, st);
}

template <int QB>
static void launch_pq_lut_q(const float* queries, int nq, int d, int M, const float* codebook_t, float* lut,
                            cudaStream_t st) {
    const size_t smem = (size_t)QB * d * 4;
    static PerDeviceSize configured;
    if (smem > 48 * 1024 && configured.raise(smem))
        cudaFuncSetAttribute(pq_lut_kernel<QB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    pq_lut_kernel<QB><<<(nq + QB - 1) / QB, 256, smem, st>>>(queries, nq, d, M, codebook_t, lut);
}
static void launch_pq_lut_t(int qb, const float* queries, int nq, int d, int M, const float* codebook_t, float* lut,
                            cudaStream_t st) {
    switch (qb) {
        case 5: launch_pq_lut_q<5>(queries, nq, d, M, codebook_t, lut, st); break;
        case 6: launch_pq_lut_q<6>(queries, nq, d, M, codebook_t, lut, st); break;
        case 7: launch_pq_lut_q<7>(queries, nq, d, M, codebook_t, lut, st); break;
        case 8: launch_pq_lut_q<8>(queries, nq, d, M, codebook_t, lut, st); break;
        default: launch_pq_lut_q<4>(queries, nq, d, M, codebook_t, lut, st); break;
    }
}

void launch_pq_lut(const float* queries, int nq, int d, int M, const float* codebook_t, float* lut,
                   cudaStream_t st) {
    if (nq <= 0) return;
    static const bool lut_v1 = getenv("RSB_LUT_V1") != nullptr;   // experiment switch: query-stationary kernel
    if (M == 64 && d == 768 && !lut_v1) {
        launch_pq_lut64(queries, nq, codebook_t, lut, st);
        return;
    }
    // per-block time ~ (codebook stream, fixed) + (per-query FMAs and stores); modelled 4 : 1 per query.  Choose the
    // queries-per-block that minimises waves x per-block time on 2 resident blocks per SM.
    const int slots = 2 * num_sms();
    int best = 4;
    long best_cost = -1;
    for (int qb = 4; qb <= 8; ++qb) {
        if ((size_t)qb * d * 4 > 200 * 1024) break;
        const long blocks = (nq + qb - 1) / qb;
        const long cost = ((blocks + slots - 1) / slots) * (4 + qb);
        if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = qb; }
    }
    launch_pq_lut_t(best, queries, nq, d, M, codebook_t, lut, st);
}

// 10-bit quantisation of a query's fp32 table for the paired scan (one block per query, in the table's
// [code value j][64 words] layout; word w holds sub-quantizer w % M).  Q = rint((T - lo_m) / delta) with
// delta = max_m (max_j T - lo_m) / 1023, so a sum of M <= 64 entries fits in 16 bits.  The residual
// T - (lo_m + delta * Q) is measured in fp64 rather than assumed to be delta / 2: the fp32 quotient may round
// across a half-way point.
__global__ __launch_bounds__(256)
void pq_lut_quant_kernel(const float* __restrict__ lut, int M, unsigned short* __restrict__ qlut,
                         PQQuant* __restrict__ quant) {
    __shared__ float s_lo[4][64], s_hi[4][64], s_abs[4][64];
    __shared__ double s_res[4][64];
    const int q = blockIdx.x, w = threadIdx.x & 63, jr = threadIdx.x >> 6;
    const float* t = lut + (size_t)q * kLutWords;
    float lo = FLT_MAX, hi = -FLT_MAX, am = 0.f;
    for (int j = jr; j < 256; j += 4) {
        const float x = t[j * kLutRowWords + w];
        lo = fminf(lo, x); hi = fmaxf(hi, x); am = fmaxf(am, fabsf(x));
    }
    s_lo[jr][w] = lo; s_hi[jr][w] = hi; s_abs[jr][w] = am;
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) { lo = fminf(lo, s_lo[i][w]); hi = fmaxf(hi, s_hi[i][w]); am = fmaxf(am, s_abs[i][w]); }
    float range = 0.f;
    for (int m = 0; m < M; ++m) {
        float l = s_lo[0][m], h = s_hi[0][m];
#pragma unroll
        for (int i = 1; i < 4; ++i) { l = fminf(l, s_lo[i][m]); h = fmaxf(h, s_hi[i][m]); }
        range = fmaxf(range, h - l);
    }
    const float delta = range > 0.f ? range / 1023.f : 1.f;
    double res = 0.0;
    for (int j = jr; j < 256; j += 4) {
        const float x = t[j * kLutRowWords + w];
        const float qv = fminf(fmaxf(rintf((x - lo) / delta), 0.f), 1023.f);
        qlut[(size_t)q * kLutWords + j * kLutRowWords + w] = (unsigned short)qv;
        res = fmax(res, fabs((double)x - ((double)lo + (double)delta * (double)qv)));
    }
    __syncthreads();                                   // every thread has read s_lo / s_hi / s_abs
    if (jr == 0) { s_lo[0][w] = lo; s_abs[0][w] = am; }
    s_res[jr][w] = res;
    __syncthreads();
    if (threadIdx.x == 0) {
        PQQuant r{0.0, (double)delta, 0.0, 0.0};
        for (int m = 0; m < M; ++m) {
            r.base += (double)s_lo[0][m];
            r.err += fmax(fmax(s_res[0][m], s_res[1][m]), fmax(s_res[2][m], s_res[3][m]));
            r.amax += (double)s_abs[0][m];
        }
        quant[q] = r;
    }
}

void launch_pq_lut_quant(const float* lut, int nq, int M, unsigned short* qlut, PQQuant* quant, cudaStream_t st) {
    if (nq <= 0) return;
    pq_lut_quant_kernel<<<nq, 256, 0, st>>>(lut, M, qlut, quant);
}

// =============================================================================================================
// 4-bit sub-quantizers (faiss nbits = 4).  Codes are packed two per byte, LSB first (faiss PQEncoderGeneric): byte b
// of a code is c[2b] | c[2b+1] << 4.  Grouping the M sub-quantizers in pairs gives one 256-entry table per code byte,
//        T'[b][j] = T[2b][j & 15] + T[2b+1][j >> 4]          (one fp32 rounding per entry)
// and score = dis0 + sum_b T'[b][byte_b]: an 8-bit table over M_b = M / 2 "byte sub-quantizers".  A 4-bit index is
// therefore stored, interleaved, quantised (pq_lut_quant_kernel) and scanned exactly like an 8-bit index of M_b
// sub-quantizers; only the table build below and the encoder are specific to it.
// =============================================================================================================
// One block per query.  Phase 1: the M x 16 sub-products <q_m, cb[m][c]> (sequential fmaf over dsub, the order of the
// 8-bit table kernels), kept in shared memory split by parity of m -- E[c][b] = T[2b][c], O[c][b] = T[2b+1][c] -- so
// that in phase 2 consecutive lanes (consecutive b) read consecutive banks.  Phase 2 writes T' straight into the
// scan's table layout: IL = the interleaved [j][64 words] rows (word w holds byte sub-quantizer w % M_b, replicated
// when M_b < 64), else the generic [b][256] table.
template <bool IL>
__global__ __launch_bounds__(256)
void pq_lut4_kernel(const float* __restrict__ queries, int d, int M, const float* __restrict__ codebook,
                    float* __restrict__ lut) {
    extern __shared__ __align__(16) float s_lut4[];          // query [d] | E [16][M/2] | O [16][M/2]
    const int q = blockIdx.x, dsub = d / M, Mb = M >> 1;
    float* qs = s_lut4;
    float* E = s_lut4 + d;
    float* O = E + 16 * Mb;
    for (int c = threadIdx.x; c < d; c += blockDim.x) qs[c] = queries[(size_t)q * d + c];
    __syncthreads();
    for (int i = threadIdx.x; i < M * 16; i += blockDim.x) {
        const int m = i >> 4, c = i & 15;
        const float* cb = codebook + (size_t)i * dsub;          // cb[m][c] of [M, 16, dsub]
        const float* x = qs + m * dsub;
        float s = 0.f;
        for (int t = 0; t < dsub; ++t) s = fmaf(x[t], __ldg(cb + t), s);
        ((m & 1) ? O : E)[c * Mb + (m >> 1)] = s;
    }
    __syncthreads();
    if (IL) {
        float* out = lut + (size_t)q * kLutWords;
        for (int i = threadIdx.x; i < kLutWords; i += blockDim.x) {
            const int j = i / kLutRowWords, b = (i % kLutRowWords) % Mb;
            out[i] = E[(j & 15) * Mb + b] + O[(j >> 4) * Mb + b];
        }
    } else {
        float* out = lut + (size_t)q * Mb * 256;
        for (int i = threadIdx.x; i < Mb * 256; i += blockDim.x) {
            const int b = i >> 8, j = i & 255;
            out[i] = E[(j & 15) * Mb + b] + O[(j >> 4) * Mb + b];
        }
    }
}

void launch_pq_lut4(const float* queries, int nq, int d, int M, const float* codebook, float* lut, cudaStream_t st) {
    if (nq <= 0) return;
    const size_t smem = ((size_t)d + 16 * (size_t)M) * 4;
    if (pq_interleaved_layout(M / 2)) {
        static PerDeviceSize configured;
        if (smem > 48 * 1024 && configured.raise(smem))
            cudaFuncSetAttribute(pq_lut4_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        pq_lut4_kernel<true><<<nq, 256, smem, st>>>(queries, d, M, codebook, lut);
    } else {
        static PerDeviceSize configured;
        if (smem > 48 * 1024 && configured.raise(smem))
            cudaFuncSetAttribute(pq_lut4_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        pq_lut4_kernel<false><<<nq, 256, smem, st>>>(queries, d, M, codebook, lut);
    }
}

// =============================================================================================================
// IVF-PQ ADC list scan -- the hot kernel.  score(code) = dis0 + sum_m T[m][code[m]].
//
// One block (256 threads, 8 warps) per item; persistent blocks pull items (sorted by list, so
// concurrent blocks share a list in L2) from an atomic counter.  The query's 64 KB fp32 table sits in shared
// memory laid out [code value j][64 words]; K = M/16 lanes cooperate on one vector and every look-up address is
// produced by ONE PRMT:  addr = (code_byte << 8) | lane_word_offset  (rsb_layout.h proves the 32 lanes of a warp
// always fall in 32 different banks).  Codes arrive as one fully-coalesced 128-bit load per lane per pass from
// the interleaved block layout, software-prefetched one block ahead.  A (K-1)-shuffle transposing reduction
// leaves lane l with the score of block-local vector l; scores above the running threshold are appended to the
// block's candidate buffer (warp-aggregated shared atomics), which is compacted by a bitonic sort only when it
// fills.  The per-query threshold is shared between blocks through global memory (atomicMax) so later lists of
// a query are filtered by what earlier lists already found.
//
// PAIRED items (two queries probing the same list, see pair_items_kernel) score both queries with one look-up: the
// block packs the two queries' 10-bit quantised tables (pq_lut_quant_kernel) into one 64 KB table of u32 words,
// query a in the low 16 bits and query b in the high 16, and accumulates with integer adds -- a sum of M <= 64
// entries is at most 64 * 1023 < 2^16, so the lanes never carry into each other.  For the integer sum S of a vector:
//     s <= dis0 + base + delta * S + err + gamma * (|dis0| + amax)
// where s is the fp32 score the single-item path computes, err bounds the table's quantisation residuals and the
// gamma term bounds the fp32 rounding of the ~66-term sum (gamma = 70 * 2^-24).  A vector whose S >= S_min, the
// smallest S that could reach the running threshold, is appended as a pending entry; pending entries are re-scored
// exactly by the whole block (pq_resolve / pq_slot_score, from the fp32 table in global memory, in pq_block_score's
// summation order) before any compaction and before the item's candidates are emitted, and kept iff the exact score
// passes today's test: the candidate sets, and so the results, are those of the single-item path.
// =============================================================================================================
constexpr int PQ_THREADS = 256;
constexpr int PQ_WARPS = PQ_THREADS / 32;
#ifndef RSB_PQ_CHECK
#define RSB_PQ_CHECK 2
#endif
constexpr int PQ_CHECK = RSB_PQ_CHECK;                       // code blocks per warp between capacity checks (2 or 3)
static_assert(PQ_CHECK == 2 || PQ_CHECK == 3, "the scan loop is written for 2 or 3 blocks per check");
constexpr int PQ_SLACK = PQ_CHECK * PQ_WARPS * 32;           // 512 / 768 candidates between checks
// Paired items check capacity after every code block per warp: the two candidate buffers then need
// cand_capacity(k, 256) entries each, which for k <= 256 fit in the single-item buffer's cand_capacity(k, 512) entries,
// so paired and single items share one block shape (3 blocks of 256 threads per SM) and shared-memory footprint.
constexpr int PQ_PAIR_SLACK = PQ_WARPS * 32;                 // 256 candidates per buffer between checks
// Shared-window address at which this kernel's dynamic shared memory is expected to start (the kernel declares
// no static shared memory; sm_90+ reserve the first 1 KB of the window).  When the runtime address matches, the
// table base is folded into the LDS immediate ("FAST" path: PRMT -> LDS [R + 0x400] -> FADD); otherwise the
// generic path (one extra add per look-up) is taken.  Which path ran is reported through ScanArgs::dbg_flag.
constexpr unsigned PQ_LUT_SADDR = 1024;

__device__ __forceinline__ unsigned smem_addr_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

// T = float: the fp32 table; T = unsigned: the packed 2 x 16-bit table of a paired item (same word layout)
template <bool FAST, typename T>
__device__ __forceinline__ T lut_at(const unsigned char* lutb, unsigned codes, unsigned off, unsigned sel) {
    // result byte0 = off (lane word offset, < 256), byte1 = selected code byte, bytes 2,3 = 0
    const unsigned a = __byte_perm(codes, off, sel);
    if (FAST) {
        T v;
        if constexpr (std::is_same<T, float>::value)
            asm volatile("ld.shared.f32 %0, [%1+%2];" : "=f"(v) : "r"(a), "n"(PQ_LUT_SADDR));
        else
            asm volatile("ld.shared.u32 %0, [%1+%2];" : "=r"(v) : "r"(a), "n"(PQ_LUT_SADDR));
        return v;
    }
    return *reinterpret_cast<const T*>(lutb + a);
}

// 16 look-ups of one pass; `at(codes, off, sel)` returns the table entry (shared-memory table, or the fp32 table in
// global memory for the exact re-score of a paired item)
template <typename T, typename At>
__device__ __forceinline__ T pq_pass(At at, const uint4 c, const unsigned (&off)[16]) {
    T s0, s1;
    s0 = at(c.x, off[0], 0x5504);
    s1 = at(c.x, off[1], 0x5514);
    s0 += at(c.x, off[2], 0x5524);
    s1 += at(c.x, off[3], 0x5534);
    s0 += at(c.y, off[4], 0x5504);
    s1 += at(c.y, off[5], 0x5514);
    s0 += at(c.y, off[6], 0x5524);
    s1 += at(c.y, off[7], 0x5534);
    s0 += at(c.z, off[8], 0x5504);
    s1 += at(c.z, off[9], 0x5514);
    s0 += at(c.z, off[10], 0x5524);
    s1 += at(c.z, off[11], 0x5534);
    s0 += at(c.w, off[12], 0x5504);
    s1 += at(c.w, off[13], 0x5514);
    s0 += at(c.w, off[14], 0x5524);
    s1 += at(c.w, off[15], 0x5534);
    return s0 + s1;
}

// score of block-local vector `lane` from the K code chunks of one 32-vector block (T = unsigned: the two packed
// 16-bit sums of a paired item)
template <int K, bool FAST, typename T = float>
__device__ __forceinline__ T pq_block_score(const unsigned char* lutb, const uint4 (&c)[K],
                                            const unsigned (&off)[16], int r) {
    const auto at = [lutb](unsigned w, unsigned o, unsigned sel) { return lut_at<FAST, T>(lutb, w, o, sel); };
    T p[K];
#pragma unroll
    for (int t = 0; t < K; ++t) p[t] = pq_pass<T>(at, c[t], off);
    if (K == 4) {
        // lane rank r holds partials of the group's vectors t = 0..3; route vector t to lane rank t
        T k0 = (r & 2) ? p[2] : p[0];
        T k1 = (r & 2) ? p[K - 1] : p[1];
        const T s0 = (r & 2) ? p[0] : p[2];
        const T s1 = (r & 2) ? p[1] : p[K - 1];
        k0 += __shfl_xor_sync(0xffffffffu, s0, 2);
        k1 += __shfl_xor_sync(0xffffffffu, s1, 2);
        const T keep = (r & 1) ? k1 : k0;
        const T send = (r & 1) ? k0 : k1;
        return keep + __shfl_xor_sync(0xffffffffu, send, 1);
    } else if (K == 2) {
        const T keep = r ? p[K - 1] : p[0];
        const T send = r ? p[0] : p[K - 1];
        return keep + __shfl_xor_sync(0xffffffffu, send, 1);
    }
    return p[0];
}

// Exact fp32 score (without dis0) of the vector at `slot`, computed by one thread from the fp32 table in global
// memory.  Equal bit for bit to pq_block_score<K, FAST, float>: block-local vector v = g*K + t is lane (g, t)'s
// vector, and lane (g, r) holds its pass-t chunk, read here from the interleaved layout (rsb_layout.h) with lane
// (g, r)'s look-up offsets.  Each pass runs pq_pass (same entries, same order), giving partials p_0 .. p_{K-1}
// (index = lane rank).  The shuffle tree of pq_block_score leaves lane t with, for K = 4,
// (p_t + p_{t^2}) + (p_{t^1} + p_{t^3}): step one adds the partner at distance 2 to the kept partial, step two the
// partner at distance 1.  fp32 addition is commutative, so for every t that is (p_0 + p_2) + (p_1 + p_3); K = 2
// gives p_0 + p_1, K = 1 p_0.  The passes run one at a time (16 table loads in flight), so the re-score fits in the
// scan loop's register allocation.
template <int K>
__device__ __forceinline__ float pq_slot_score(const float* __restrict__ lutq, const uint4* __restrict__ codes4,
                                               unsigned slot) {
    const unsigned char* tb = reinterpret_cast<const unsigned char*>(lutq);
    const auto at = [tb](unsigned w, unsigned o, unsigned sel) {
        return __ldg(reinterpret_cast<const float*>(tb + __byte_perm(w, o, sel)));
    };
    const int v = (int)(slot & 31u), g = v / K, t = v % K;
    const uint4* chunk = codes4 + (size_t)(slot >> 5) * (K * 32) + t * 32 + g * K;   // + r: lane (g, r)'s chunk
    float even = 0.f, odd = 0.f;                                     // p_0 (+ p_2), p_1 (+ p_3)
#pragma unroll 1
    for (int r = 0; r < K; ++r) {
        unsigned off[16];
#pragma unroll
        for (int s = 0; s < 16; ++s) off[s] = 4u * (unsigned)pq_pos(16 * K, K, g, r, s);
        const float p = pq_pass<float>(at, __ldg(chunk + r), off);
        if (r & 1) odd = r < 2 ? p : odd + p;
        else even = r < 2 ? p : even + p;
    }
    return K == 1 ? even : even + odd;
}

// Predicated 128-bit loads: past the end of the list the registers simply keep their old contents (the scores of
// such blocks are never used), which saves the eight zeroing moves per block a select would cost.
template <int K>
__device__ __forceinline__ void pq_load_block(uint4 (&dst)[K], const uint4* cbase, int b, int nblk, int lane) {
    const uint4* p = cbase + (size_t)b * (K * 32) + lane;
    const int ok = b < nblk;
#pragma unroll
    for (int t = 0; t < K; ++t)
        asm("{\n\t.reg .pred p;\n\tsetp.ne.s32 p, %5, 0;\n\t@p ld.global.nc.v4.u32 {%0, %1, %2, %3}, [%4];\n\t}"
            : "+r"(dst[t].x), "+r"(dst[t].y), "+r"(dst[t].z), "+r"(dst[t].w)
            : "l"(p + t * 32), "r"(ok));
}

// scan one inverted list for one query; returns the updated threshold.  Two code-register sets (A/B) ping-pong so
// that the next block's 128-bit loads are in flight while the current block is scored (no register copies).
template <int K, bool FAST>
__device__ __forceinline__ unsigned pq_scan_list(const unsigned char* lutb, const uint4* cbase, int nblk, int len,
                                                 unsigned slot0, float dis0, const unsigned (&off)[16], int r,
                                                 u64* keys, int* s_count, unsigned tau, int k, int cap,
                                                 const ScanArgs& a, int q, int lane, int warp) {
    unsigned* tau_g = a.tau + q;
    const int n_iter = (nblk + PQ_WARPS - 1) / PQ_WARPS;
    uint4 A[K], B[K];
#pragma unroll
    for (int t = 0; t < K; ++t) A[t] = B[t] = make_uint4(0, 0, 0, 0);
    pq_load_block<K>(A, cbase, warp, nblk, lane);
    pq_load_block<K>(B, cbase, warp + PQ_WARPS, nblk, lane);
    // one step: score the block held in register set X (lane l owns block-local vector l), then refill X with the
    // block two steps ahead (the other set holds the next one)
#define RSB_PQ_STEP(X, b)                                                                                  \
    {                                                                                                      \
        const int b_ = (b);                                                                                \
        if (b_ < nblk) {                                                                                   \
            const float score = dis0 + pq_block_score<K, FAST>(lutb, X, off, r);                           \
            const int vi = b_ * 32 + lane;                                                                 \
            const unsigned o = ord_f32(score);                                                             \
            warp_append(keys, s_count, vi < len && o > tau, make_key(o, slot0 + (unsigned)vi));            \
        }                                                                                                  \
        pq_load_block<K>(X, cbase, b_ + 2 * PQ_WARPS, nblk, lane);                                         \
    }
    // capacity check (one barrier); a compaction that found k candidates tightens the bound for every block
    // working on this query
    // The other blocks' bound for this query is read from global memory at the START of a check interval and merged in
    // at its end, so the load is not consumed right after it is issued.  A bound that is one interval old is still a
    // valid bound.
#define RSB_PQ_CHECKPOINT()                                                                                \
    {                                                                                                      \
        const unsigned tau_new = block_maybe_compact(keys, s_count, k, cap, PQ_SLACK, tau);                \
        if (tau_new > tau && threadIdx.x == 0) raise_tau(a, q, tau_new);                                   \
        tau = gt > tau_new ? gt : tau_new;                                                                 \
    }
    if (PQ_CHECK == 2) {
        for (int it = 0; it < n_iter; it += 2) {
            const int b0 = it * PQ_WARPS + warp;
            const unsigned gt = *reinterpret_cast<const volatile unsigned*>(tau_g);
            RSB_PQ_STEP(A, b0);
            RSB_PQ_STEP(B, b0 + PQ_WARPS);
            RSB_PQ_CHECKPOINT();
        }
    } else {   // three blocks per check: the register sets alternate A B A | B A B
        for (int it = 0; it < n_iter; it += 6) {
            const int b0 = it * PQ_WARPS + warp;
            unsigned gt = *reinterpret_cast<const volatile unsigned*>(tau_g);
            RSB_PQ_STEP(A, b0);
            RSB_PQ_STEP(B, b0 + PQ_WARPS);
            RSB_PQ_STEP(A, b0 + 2 * PQ_WARPS);
            RSB_PQ_CHECKPOINT();
            gt = *reinterpret_cast<const volatile unsigned*>(tau_g);
            RSB_PQ_STEP(B, b0 + 3 * PQ_WARPS);
            RSB_PQ_STEP(A, b0 + 4 * PQ_WARPS);
            RSB_PQ_STEP(B, b0 + 5 * PQ_WARPS);
            RSB_PQ_CHECKPOINT();
        }
    }
#undef RSB_PQ_STEP
#undef RSB_PQ_CHECKPOINT
    return tau;
}

// S_min: the smallest integer sum that can still give an fp32 score above the threshold tau, for
// c0 = dis0 + base + err + gamma * (|dis0| + amax) and inv_delta = 1 / delta (rounded down, less one for the fp64
// evaluation, whose relative error is ~1e-16 on a value < 2^17); 0 = re-score all.
__device__ __forceinline__ int pq_smin(unsigned tau, double c0, double inv_delta) {
    if (tau == 0u) return 0;
    const float t = unord_f32(tau);
    if (!isfinite(t)) return 0;
    const double x = floor(((double)t - c0) * inv_delta) - 1.0;
    return x > 0.0 ? (x < 65536.0 ? (int)x : 65536) : 0;
}

// Shared-memory state of a paired item; h = 0 / 1 for query a / b.
struct PQPairState {
    double thr[2][2];     // {c0, inv_delta} of pq_smin
    int q[2];
    float dis0[2];
    int count[2];         // candidate counts
};

// Resolve the PENDING entries of query h's candidate buffer of a paired item.  The look-up loop appends a vector
// whose integer sum reaches S_min as the key make_key(0, slot): no scored key has ordered score 0, because a scored
// key is appended only when its ordered score exceeds a threshold >= 0.  Here each pending vector is re-scored
// exactly (pq_slot_score) and kept iff its ordered score beats `tau`, a valid bound for the query like the register
// copy the single-item path keeps; scored entries are kept as they are.  All threads call it at a block-uniform
// point; afterwards the buffer holds scored keys only (in no particular order), so a compaction derives its
// threshold from exact scores.  The buffer is rewritten in place, 256 entries per round: a round's survivors land
// below the next round's entries.
template <int K>
__device__ __forceinline__ void pq_resolve(u64* keys, PQPairState* st, int h, const float* __restrict__ lut_g,
                                           const uint4* __restrict__ codes4, unsigned tau, u64* rescored) {
    int* count = &st->count[h];
    __syncthreads();                                                   // every append is done
    const int n = *count;
    __syncthreads();                                                   // every thread has read n
    if (threadIdx.x == 0) *count = 0;
    const float* lutq = lut_g + (size_t)st->q[h] * kLutWords;
    const float dis0 = st->dis0[h];
    for (int i0 = 0; i0 < n; i0 += PQ_THREADS) {
        const int i = i0 + threadIdx.x;
        u64 key = i < n ? keys[i] : 0ull;
        const bool pending = i < n && key_ord(key) == 0u;
        __syncthreads();                                               // this round's entries have been read
        bool keep = i < n;
        if (pending) {
            const unsigned slot = key_slot(key);
            const unsigned o = ord_f32(dis0 + pq_slot_score<K>(lutq, codes4, slot));
            key = make_key(o, slot);
            keep = o > tau;
        }
        if (rescored) {
            const unsigned m = __ballot_sync(0xffffffffu, pending);
            if (m && (threadIdx.x & 31) == 0) atomicAdd(rescored, (u64)__popc(m));
        }
        warp_append(keys, count, keep, key);
    }
    __syncthreads();
}

// scan one inverted list for the two queries of a paired item (packed 2 x 16-bit table in shared memory)
template <int K, bool FAST>
__device__ __forceinline__ void pq_scan_pair(const unsigned char* lutb, const uint4* cbase, int nblk, int len,
                                             unsigned slot0, const unsigned (&off)[16], int r, u64* keys_a,
                                             u64* keys_b, PQPairState* st, const float* __restrict__ lut_g,
                                             const uint4* __restrict__ codes4, int k, int cap2, const ScanArgs& a,
                                             int lane, int warp) {
    const int n_iter = (nblk + PQ_WARPS - 1) / PQ_WARPS;
    const int lim = cap2 - PQ_PAIR_SLACK;
    unsigned tau_a = *reinterpret_cast<const volatile unsigned*>(a.tau + st->q[0]);
    unsigned tau_b = *reinterpret_cast<const volatile unsigned*>(a.tau + st->q[1]);
    int smin_a = pq_smin(tau_a, st->thr[0][0], st->thr[0][1]), smin_b = pq_smin(tau_b, st->thr[1][0], st->thr[1][1]);
    uint4 A[K], B[K];
#pragma unroll
    for (int t = 0; t < K; ++t) A[t] = B[t] = make_uint4(0, 0, 0, 0);
    pq_load_block<K>(A, cbase, warp, nblk, lane);
    pq_load_block<K>(B, cbase, warp + PQ_WARPS, nblk, lane);
    // integer sums of both queries in one look-up; a vector whose sum reaches S_min is appended as pending
#define RSB_PQ_STEP2(X, b)                                                                                 \
    {                                                                                                      \
        const int b_ = (b);                                                                                \
        if (b_ < nblk) {                                                                                   \
            const unsigned sum = pq_block_score<K, FAST, unsigned>(lutb, X, off, r);                       \
            const int vi = b_ * 32 + lane;                                                                 \
            const u64 pend = make_key(0u, slot0 + (unsigned)vi);                                           \
            warp_append(keys_a, &st->count[0], vi < len && (int)(sum & 0xffffu) >= smin_a, pend);          \
            warp_append(keys_b, &st->count[1], vi < len && (int)(sum >> 16) >= smin_b, pend);              \
        }                                                                                                  \
        pq_load_block<K>(X, cbase, b_ + 2 * PQ_WARPS, nblk, lane);                                         \
    }
    // One barrier checks both buffers.  A buffer over its limit has its pending entries resolved, then is compacted;
    // a compaction that found k candidates raises the query's global threshold.  The global thresholds (ga, gb) are
    // read at the START of the code block and merged in here, so their loads are not waited for (a bound one block
    // old is still a valid bound).  S_min is recomputed whenever a threshold moved.  The over-limit branch gives the
    // two code register sets up to the re-score and loads their blocks (next X = bx, Y = by) again afterwards, so the
    // re-score does not add to the loop's register allocation.
#define RSB_PQ_CHECKPOINT2(X, bx, Y, by)                                                                   \
    {                                                                                                      \
        const unsigned ta0 = tau_a, tb0 = tau_b;                                                           \
        tau_a = ga > tau_a ? ga : tau_a;                                                                   \
        tau_b = gb > tau_b ? gb : tau_b;                                                                   \
        if (__syncthreads_or(*reinterpret_cast<volatile int*>(&st->count[0]) > lim ||                      \
                             *reinterpret_cast<volatile int*>(&st->count[1]) > lim)) {                     \
            if (st->count[0] > lim) {                                                                      \
                pq_resolve<K>(keys_a, st, 0, lut_g, codes4, tau_a, a.rescored);                            \
                const unsigned t_ = block_compact(keys_a, &st->count[0], k, cap2, tau_a);                  \
                if (t_ > tau_a && threadIdx.x == 0) raise_tau(a, st->q[0], t_);                            \
                tau_a = t_;                                                                                \
            }                                                                                              \
            if (st->count[1] > lim) {                                                                      \
                pq_resolve<K>(keys_b, st, 1, lut_g, codes4, tau_b, a.rescored);                            \
                const unsigned t_ = block_compact(keys_b, &st->count[1], k, cap2, tau_b);                  \
                if (t_ > tau_b && threadIdx.x == 0) raise_tau(a, st->q[1], t_);                            \
                tau_b = t_;                                                                                \
            }                                                                                              \
            for (int t = 0; t < K; ++t) X[t] = Y[t] = make_uint4(0, 0, 0, 0);                              \
            pq_load_block<K>(X, cbase, bx, nblk, lane);                                                    \
            pq_load_block<K>(Y, cbase, by, nblk, lane);                                                    \
        }                                                                                                  \
        if (tau_a != ta0) smin_a = pq_smin(tau_a, st->thr[0][0], st->thr[0][1]);                           \
        if (tau_b != tb0) smin_b = pq_smin(tau_b, st->thr[1][0], st->thr[1][1]);                           \
    }
    for (int it = 0; it < n_iter; it += 2) {
        const int b0 = it * PQ_WARPS + warp;
        unsigned ga = *reinterpret_cast<const volatile unsigned*>(a.tau + st->q[0]);
        unsigned gb = *reinterpret_cast<const volatile unsigned*>(a.tau + st->q[1]);
        RSB_PQ_STEP2(A, b0);
        RSB_PQ_CHECKPOINT2(B, b0 + PQ_WARPS, A, b0 + 2 * PQ_WARPS);
        ga = *reinterpret_cast<const volatile unsigned*>(a.tau + st->q[0]);
        gb = *reinterpret_cast<const volatile unsigned*>(a.tau + st->q[1]);
        RSB_PQ_STEP2(B, b0 + PQ_WARPS);
        RSB_PQ_CHECKPOINT2(A, b0 + 2 * PQ_WARPS, B, b0 + 3 * PQ_WARPS);
    }
#undef RSB_PQ_STEP2
#undef RSB_PQ_CHECKPOINT2
    pq_resolve<K>(keys_a, st, 0, lut_g, codes4, tau_a, a.rescored);     // emit sees scored keys only
    pq_resolve<K>(keys_b, st, 1, lut_g, codes4, tau_b, a.rescored);
}

// PAIRED = false compiles the single-item path alone, so it keeps its own register allocation (the paired branch needs
// more registers than the single-item loop and would make the single-item loop spill).  It runs every search without
// a paired work list (one query, RSB_PQ_SINGLE_ITEMS) and every paired work list in which no two pairs share a list
// (n_items == n_pairs, e.g. the full sweep): both variants are launched and each returns at once unless it is the one
// the work list needs.
template <int K, bool PAIRED>
__global__ __launch_bounds__(PQ_THREADS, 3)
void ivfpq_scan_kernel(ScanArgs a, const float* __restrict__ lut_g, const uint8_t* __restrict__ codes, int cap,
                       int cap2) {
    constexpr int M = 16 * K;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    unsigned char* lutb = smem_raw;                                    // 64 KB table (fp32, or packed 2 x u16)
    // candidate buffers: one of `cap` entries (single items) or two of `cap2` (paired items), in one region
    u64* keys_a = reinterpret_cast<u64*>(smem_raw + kLutWords * 4);
    u64* keys_b = keys_a + cap2;
    PQPairState* st = reinterpret_cast<PQPairState*>(keys_a + max(cap, 2 * cap2));
    int* s_count = st->count;                                          // [0]: single items and query a
    int* s_ctrl = reinterpret_cast<int*>(st + 1);
    uint64_t* lut_bar = reinterpret_cast<uint64_t*>(s_ctrl);          // 8-byte aligned
    int* s_item = s_ctrl + 2;                                          // two slots (current / next item)
    int* s_work = s_ctrl + 4;                                          // the item's pairs, see below

    if (a.items && PAIRED != (*a.n_items != *a.n_pairs)) return;      // the other variant scans this work list
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane / K, r = lane % K;
    unsigned off[16];
#pragma unroll
    for (int s = 0; s < 16; ++s) off[s] = 4u * (unsigned)pq_pos(M, K, g, r, s);

    const bool fast = smem_addr_u32(smem_raw) == PQ_LUT_SADDR;         // block-uniform
    if (a.dbg_flag && blockIdx.x == 0 && tid == 0) *a.dbg_flag = fast ? 1u : 2u;

    unsigned lut_phase = 0u;
    if (tid == 0) {
        rsbtc::mbar_init(lut_bar, 1);
        rsbtc::fence_barrier_init();
        s_item[0] = atomicAdd(a.item_counter, 1);
    }

    // Emit a pair's candidates.  They only need sorting (and trimming to k) when more than k survived; the
    // per-query merge kernel treats every item as an unordered set.
    const auto emit = [&](int pair, int q, u64* keys, int* count, int capacity, unsigned tau) {
        int n = *count;
        bool sorted = false;
        if (n > a.k) {                                                 // block-uniform
            block_compact(keys, count, a.k, capacity, tau);
            n = a.k;
            sorted = true;
        }
        for (int i = tid; i < n; i += PQ_THREADS) a.out_keys[(size_t)pair * a.k + i] = keys[i];
        if (tid == 0) {
            a.out_cnt[pair] = n;
            if (sorted) raise_tau(a, q, key_ord(keys[a.k - 1]));
        }
    };

    const int n_items = *a.n_items;
    int cur_q = -1, par = 0;
    for (;;) {
        __syncthreads();                                           // (B) previous item done; s_item[par] visible
        const int item = s_item[par];
        if (item >= n_items) break;
        // thread 0 reserves the block's NEXT item now and publishes it at the end of this one, so the atomic's
        // round trip is hidden behind the scan
        int next_item = 0;
        if (tid == 0) {
            next_item = atomicAdd(a.item_counter, 1);
            const int2 it = PAIRED ? a.items[item] : make_int2(a.order[item], -1);
            // A paired item whose queries do not both have a bound yet (thresholds that come from another GPU) is
            // scanned as two single items: without a bound every vector would need the exact re-score.
            bool pair = it.y >= 0;
            if (pair) {
                const unsigned ta = *reinterpret_cast<volatile unsigned*>(a.tau + it.x / a.nprobe);
                const unsigned tb = *reinterpret_cast<volatile unsigned*>(a.tau + it.y / a.nprobe);
                pair = ta != 0u && tb != 0u;
            }
            s_work[0] = it.x;                                      // single item, or query a of a paired item
            s_work[1] = pair ? it.y : -1;                          // query b of a paired item
            s_work[2] = pair ? -1 : it.y;                          // second single item of a split pair
        }
        __syncthreads();
        const int w0 = s_work[0], w1 = s_work[1], w2 = s_work[2];
        const int list = (int)a.coarse_ids[w0];
        const int len = a.list_len[list];
        const int64_t slot0 = a.list_off[list];                       // multiple of 32
        const int nblk = (len + 31) >> 5;
        const uint4* cbase = reinterpret_cast<const uint4*>(codes + (size_t)slot0 * M);  // K*32 uint4 per block

        if (PAIRED && w1 >= 0) {
            // ---- paired item: pack the two quantised tables (query a low half, query b high half)
            const int qa = w0 / a.nprobe, qb = w1 / a.nprobe;
            const uint4* ta = reinterpret_cast<const uint4*>(a.qlut + (size_t)qa * kLutWords);
            const uint4* tb = reinterpret_cast<const uint4*>(a.qlut + (size_t)qb * kLutWords);
            uint4* dst = reinterpret_cast<uint4*>(lutb);
#pragma unroll 2
            for (int i = tid; i < kLutWords / 8; i += PQ_THREADS) {
                const uint4 x = __ldg(ta + i), y = __ldg(tb + i);
                dst[2 * i] = make_uint4(__byte_perm(x.x, y.x, 0x5410), __byte_perm(x.x, y.x, 0x7632),
                                        __byte_perm(x.y, y.y, 0x5410), __byte_perm(x.y, y.y, 0x7632));
                dst[2 * i + 1] = make_uint4(__byte_perm(x.z, y.z, 0x5410), __byte_perm(x.z, y.z, 0x7632),
                                            __byte_perm(x.w, y.w, 0x5410), __byte_perm(x.w, y.w, 0x7632));
            }
            cur_q = -1;
            if (tid < 2) {
                constexpr double gamma = 70.0 / 16777216.0;
                const int pair = tid ? w1 : w0, q = tid ? qb : qa;
                const float dis0 = a.coarse_scores[pair];
                const PQQuant qq = a.quant[q];
                st->thr[tid][0] = (double)dis0 + qq.base + qq.err + gamma * (fabs((double)dis0) + qq.amax);
                st->thr[tid][1] = 1.0 / qq.delta;
                st->q[tid] = q;
                st->dis0[tid] = dis0;
                st->count[tid] = 0;
            }
            __syncthreads();
            const uint4* codes4 = reinterpret_cast<const uint4*>(codes);
            if (fast)
                pq_scan_pair<K, true>(lutb, cbase, nblk, len, (unsigned)slot0, off, r, keys_a, keys_b, st, lut_g,
                                      codes4, a.k, cap2, a, lane, warp);
            else
                pq_scan_pair<K, false>(lutb, cbase, nblk, len, (unsigned)slot0, off, r, keys_a, keys_b, st, lut_g,
                                       codes4, a.k, cap2, a, lane, warp);
            __syncthreads();
            emit(w0, qa, keys_a, &st->count[0], cap2, 0u);
            emit(w1, qb, keys_b, &st->count[1], cap2, 0u);
        } else {
            // ---- single item(s): the query's fp32 table
            for (int h = 0; h < 2; ++h) {
                const int pair = h ? w2 : w0;
                if (pair < 0) break;                                   // block-uniform
                if (h) __syncthreads();                                // the first item's emit is done
                const int q = pair / a.nprobe;
                const float dis0 = a.coarse_scores[pair];
                if (tid == 0) s_count[0] = 0;
                if (q != cur_q) {                                      // block-uniform
                    // 64 KB table: one bulk copy by the TMA engine (global -> shared, no register staging, no trip
                    // through the LSU data pipe that the look-ups saturate), completion signalled on an mbarrier.
                    // All generic-proxy accesses of the previous table finished before the last barrier; the proxy
                    // fence orders them before the async-proxy writes.
                    if (tid == 0) {
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                        rsbtc::mbar_expect_tx(lut_bar, kLutWords * 4);
                        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                     ::"r"(smem_addr_u32(smem_raw)),
                                       "l"(reinterpret_cast<unsigned long long>(lut_g + (size_t)q * kLutWords)),
                                       "r"(kLutWords * 4), "r"(smem_addr_u32(lut_bar))
                                     : "memory");
                    }
                    rsbtc::mbar_wait(lut_bar, lut_phase);
                    lut_phase ^= 1u;
                    cur_q = q;
                }
                unsigned tau = *reinterpret_cast<volatile unsigned*>(a.tau + q);
                __syncthreads();
                if (fast)
                    tau = pq_scan_list<K, true>(lutb, cbase, nblk, len, (unsigned)slot0, dis0, off, r, keys_a, s_count,
                                                tau, a.k, cap, a, q, lane, warp);
                else
                    tau = pq_scan_list<K, false>(lutb, cbase, nblk, len, (unsigned)slot0, dis0, off, r, keys_a,
                                                 s_count, tau, a.k, cap, a, q, lane, warp);
                __syncthreads();
                emit(pair, q, keys_a, s_count, cap, tau);
            }
        }
        if (tid == 0) s_item[par ^ 1] = next_item;
        par ^= 1;
    }
}

__device__ __forceinline__ int find_segment(const int64_t* seg_starts, int nseg, int64_t row);

// =============================================================================================================
// Generic-M path (any number of sub-quantizers M with M % 4 == 0, M <= 128, nbits = 8; e.g. the 24 / 48 / 96 that
// faiss -- and therefore the reference's `n_subquantizers` key, src/indicies/ivf_pq.py:146-152 -- accepts on d = 768).
// The conflict-free interleaved layout above exists for M = 16, 32, 64 only; here codes stay in natural [slot][M]
// order, the table is [m][256] and one thread scores one vector with a sequential sum over m (the oracle's order).
// Functionally complete, not tuned: look-ups hit random banks (2-3 way conflicts) and every thread reads its own row.
// =============================================================================================================
__global__ __launch_bounds__(256)
void pq_lut_generic_kernel(const float* __restrict__ queries, int d, int M, const float* __restrict__ codebook,
                           float* __restrict__ lut) {
    extern __shared__ __align__(16) float qs_g[];                      // [d]
    const int q = blockIdx.x, j = threadIdx.x, dsub = d / M;
    for (int c = threadIdx.x; c < d; c += blockDim.x) qs_g[c] = queries[(size_t)q * d + c];
    __syncthreads();
    float* out = lut + (size_t)q * M * 256;
    for (int m = 0; m < M; ++m) {
        const float* cb = codebook + ((size_t)m * 256 + j) * dsub;
        float sacc = 0.f;
        for (int t = 0; t < dsub; ++t) sacc = fmaf(qs_g[m * dsub + t], __ldg(cb + t), sacc);
        out[m * 256 + j] = sacc;
    }
}
void launch_pq_lut_generic(const float* queries, int nq, int d, int M, const float* codebook, float* lut, cudaStream_t st) {
    if (nq <= 0) return;
    pq_lut_generic_kernel<<<nq, 256, (size_t)d * 4, st>>>(queries, d, M, codebook, lut);
}

constexpr int GS_THREADS = 256, GS_CHECK = 2, GS_SLACK = GS_CHECK * GS_THREADS;

__global__ __launch_bounds__(GS_THREADS)
void ivfpq_scan_generic_kernel(ScanArgs a, const float* __restrict__ lut_g, const uint8_t* __restrict__ codes, int M,
                               int cap) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* lut = reinterpret_cast<float*>(smem_raw);                    // [M][256]
    u64* keys = reinterpret_cast<u64*>(smem_raw + (size_t)M * 1024);
    __shared__ int s_count, s_item;
    const int tid = threadIdx.x;
    const int n_items = *a.n_items;
    int cur_q = -1;
    for (;;) {
        __syncthreads();
        if (tid == 0) { s_item = atomicAdd(a.item_counter, 1); s_count = 0; }
        __syncthreads();
        const int item = s_item;
        if (item >= n_items) break;
        const int pair = a.order[item];
        const int q = pair / a.nprobe;
        const int list = (int)a.coarse_ids[pair];
        const float dis0 = a.coarse_scores[pair];
        if (q != cur_q) {                                               // block-uniform
            const float4* src = reinterpret_cast<const float4*>(lut_g + (size_t)q * M * 256);
            for (int i = tid; i < M * 64; i += GS_THREADS) reinterpret_cast<float4*>(lut)[i] = src[i];
            cur_q = q;
        }
        unsigned tau = *reinterpret_cast<volatile unsigned*>(a.tau + q);
        __syncthreads();
        const int len = a.list_len[list];
        const int64_t slot0 = a.list_off[list];
        const int n_iter = (len + GS_THREADS - 1) / GS_THREADS;
        for (int it = 0; it < n_iter; ++it) {
            const int v = it * GS_THREADS + tid;
            const bool ok = v < len;
            float sc = 0.f;
            if (ok) {
                const uint32_t* c = reinterpret_cast<const uint32_t*>(codes + (size_t)(slot0 + v) * M);
                for (int w = 0; w < M / 4; ++w) {
                    const uint32_t u = __ldg(c + w);
                    const float* t = lut + (size_t)w * 1024;
                    sc += t[u & 255u];
                    sc += t[256 + ((u >> 8) & 255u)];
                    sc += t[512 + ((u >> 16) & 255u)];
                    sc += t[768 + (u >> 24)];
                }
            }
            const unsigned o = ord_f32(dis0 + sc);
            warp_append(keys, &s_count, ok && o > tau, make_key(o, (unsigned)(slot0 + v)));
            if ((it + 1) % GS_CHECK == 0) {
                const unsigned tau_new = block_maybe_compact(keys, &s_count, a.k, cap, GS_SLACK, tau);
                if (tau_new > tau && tid == 0) raise_tau(a, q, tau_new);
                const unsigned gt = *reinterpret_cast<const volatile unsigned*>(a.tau + q);
                tau = gt > tau_new ? gt : tau_new;
            }
        }
        tau = block_compact(keys, &s_count, a.k, cap, tau);
        const int n = min(s_count, a.k);
        for (int i = tid; i < n; i += GS_THREADS) a.out_keys[(size_t)pair * a.k + i] = keys[i];
        if (tid == 0) {
            a.out_cnt[pair] = n;
            if (n >= a.k) raise_tau(a, q, key_ord(keys[a.k - 1]));
        }
    }
}

static int launch_ivfpq_scan_generic(const ScanArgs& a, const float* lut, const uint8_t* codes, int M, int npairs,
                                     cudaStream_t st) {
    const int cap = cand_capacity(a.k, GS_SLACK);
    const size_t smem = (size_t)M * 1024 + (size_t)cap * 8;
    if (smem > 200 * 1024) return -1;
    cudaFuncSetAttribute(ivfpq_scan_generic_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    int occ = 1;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, ivfpq_scan_generic_kernel, GS_THREADS, smem);
    if (occ < 1) occ = 1;
    const int grid = min(npairs, num_sms() * occ);
    ivfpq_scan_generic_kernel<<<grid, GS_THREADS, smem, st>>>(a, lut, codes, M, cap);
    return 0;
}

// natural-order codes of the padded slot space -> compact CSR order (export of a generic-M index)
__global__ void compact_slots_rows_kernel(const uint8_t* __restrict__ src_slots, const int64_t* __restrict__ list_nat_off,
                                          const int64_t* __restrict__ list_slot_off, int nlist, int row_words,
                                          uint32_t* __restrict__ dst_nat) {
    const int64_t n = list_nat_off[nlist];
    const int64_t total = n * row_words;
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < total; w += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = w / row_words;
        const int c = (int)(w % row_words);
        const int l = find_segment(list_nat_off, nlist, i);
        const int64_t slot = list_slot_off[l] + (i - list_nat_off[l]);
        dst_nat[w] = reinterpret_cast<const uint32_t*>(src_slots)[slot * row_words + c];
    }
}
void launch_compact_slots_rows(const uint8_t* src_slots, const int64_t* list_nat_off, const int64_t* list_slot_off, int nlist,
                               int row_bytes, uint8_t* dst_nat, cudaStream_t st) {
    compact_slots_rows_kernel<<<4096, 256, 0, st>>>(src_slots, list_nat_off, list_slot_off, nlist, row_bytes / 4,
                                                    reinterpret_cast<uint32_t*>(dst_nat));
}

template <int K>
static void launch_ivfpq_scan_t(const ScanArgs& a, const float* lut, const uint8_t* codes, int npairs,
                                cudaStream_t st) {
    const int cap = cand_capacity(a.k, PQ_SLACK);
    const auto launch = [&](auto kernel, int cap2) {
        // table + candidate buffer region + PQPairState, LUT mbarrier, item slots, the item's pairs
        const size_t smem = (size_t)kLutWords * 4 + (size_t)std::max(cap, 2 * cap2) * 8 + sizeof(PQPairState) + 32;
        cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        int occ = 1;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, PQ_THREADS, smem);
        if (occ < 1) occ = 1;
        const int grid = min(npairs, num_sms() * occ);
        kernel<<<grid, PQ_THREADS, smem, st>>>(a, lut, codes, cap, cap2);
    };
    if (a.items) launch(ivfpq_scan_kernel<K, true>, cand_capacity(a.k, PQ_PAIR_SLACK));
    launch(ivfpq_scan_kernel<K, false>, 0);
}


__global__ void smem_base_probe_kernel(unsigned* out) {
    extern __shared__ __align__(16) unsigned char probe_smem[];
    if (threadIdx.x == 0) *out = smem_addr_u32(probe_smem);
}
unsigned probe_dynamic_smem_base(cudaStream_t st) {
    unsigned* d = nullptr;
    unsigned h = 0;
    if (cudaMalloc(&d, 4) != cudaSuccess) return 0;
    smem_base_probe_kernel<<<1, 32, 1024, st>>>(d);
    cudaMemcpyAsync(&h, d, 4, cudaMemcpyDeviceToHost, st);
    cudaStreamSynchronize(st);
    cudaFree(d);
    return h;
}

int launch_ivfpq_scan(const ScanArgs& a, const float* lut, const uint8_t* codes, int M, int nq, cudaStream_t st) {
    const int npairs = nq * a.nprobe;
    if (!a.tau_external) cudaMemsetAsync(a.tau, 0, (size_t)nq * 4, st);
    cudaMemsetAsync(a.out_cnt, 0, (size_t)npairs * 4, st);
    if (npairs == 0) return 0;
    switch (M) {
        case 16: launch_ivfpq_scan_t<1>(a, lut, codes, npairs, st); return 0;
        case 32: launch_ivfpq_scan_t<2>(a, lut, codes, npairs, st); return 0;
        case 64: launch_ivfpq_scan_t<4>(a, lut, codes, npairs, st); return 0;
        default: return launch_ivfpq_scan_generic(a, lut, codes, M, npairs, st);
    }
}

// =============================================================================================================
// Residual PQ encoding (faiss IndexIVFPQ.add -> ProductQuantizer::compute_code on x - centroid[list]).
// grid (row tiles of 128, M); the sub-quantizer's 256 x dsub codebook is staged in shared memory and read by
// broadcast; each thread owns one row and keeps its residual sub-vector in registers.
// =============================================================================================================
template <int DSUB>
__global__ __launch_bounds__(128)
void pq_encode_kernel(const float* __restrict__ x, int64_t n, int d, const int32_t* __restrict__ list,
                      const float* __restrict__ centroids, const float* __restrict__ codebook, int M,
                      uint8_t* __restrict__ codes) {
    extern __shared__ __align__(16) float cb_s[];
    const int m = blockIdx.y;
    const float* cb = codebook + (size_t)m * 256 * DSUB;
    for (int i = threadIdx.x; i < 256 * DSUB; i += blockDim.x) cb_s[i] = cb[i];
    __syncthreads();
    const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n) return;
    float rr[DSUB];
    if (list) {
        const int l = list[row];
#pragma unroll
        for (int t = 0; t < DSUB; ++t)
            rr[t] = x[(size_t)row * d + m * DSUB + t] - __ldg(centroids + (size_t)l * d + m * DSUB + t);
    } else {                                   // rows are already residuals (PQ training: k-means assignment step)
#pragma unroll
        for (int t = 0; t < DSUB; ++t) rr[t] = x[(size_t)row * d + m * DSUB + t];
    }
    float best = FLT_MAX;
    int bj = 0;
    for (int j = 0; j < 256; ++j) {
        float dist = 0.f;
#pragma unroll
        for (int t = 0; t < DSUB; ++t) {
            const float df = rr[t] - cb_s[j * DSUB + t];
            dist = fmaf(df, df, dist);
        }
        if (dist < best) { best = dist; bj = j; }
    }
    codes[(size_t)row * M + m] = (uint8_t)bj;
}

// generic dsub (any value): residual re-read from global each time (slow path, rarely used)
__global__ __launch_bounds__(128)
void pq_encode_generic_kernel(const float* __restrict__ x, int64_t n, int d, const int32_t* __restrict__ list,
                              const float* __restrict__ centroids, const float* __restrict__ codebook, int M,
                              int dsub, uint8_t* __restrict__ codes) {
    const int m = blockIdx.y;
    const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n) return;
    const float* xr = x + (size_t)row * d + m * dsub;
    const float* cr = list ? centroids + (size_t)list[row] * d + m * dsub : nullptr;
    const float* cb = codebook + (size_t)m * 256 * dsub;
    float best = FLT_MAX;
    int bj = 0;
    for (int j = 0; j < 256; ++j) {
        float dist = 0.f;
        for (int t = 0; t < dsub; ++t) {
            const float df = (xr[t] - (cr ? cr[t] : 0.f)) - __ldg(cb + j * dsub + t);
            dist = fmaf(df, df, dist);
        }
        if (dist < best) { best = dist; bj = j; }
    }
    codes[(size_t)row * M + m] = (uint8_t)bj;
}

template <int DSUB>
static void launch_pq_encode_t(const float* x, int64_t n, int d, const int32_t* list, const float* centroids,
                               const float* codebook, int M, uint8_t* codes, cudaStream_t st) {
    const size_t smem = (size_t)256 * DSUB * 4;
    if (smem > 48 * 1024)
        cudaFuncSetAttribute(pq_encode_kernel<DSUB>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    dim3 grid((unsigned)((n + 127) / 128), M);
    pq_encode_kernel<DSUB><<<grid, 128, smem, st>>>(x, n, d, list, centroids, codebook, M, codes);
}

void launch_pq_encode(const float* x, int64_t n, int d, const int32_t* list, const float* centroids,
                      const float* codebook, int M, uint8_t* codes, cudaStream_t st) {
    if (n <= 0) return;
    const int dsub = d / M;
    switch (dsub) {
        case 4: launch_pq_encode_t<4>(x, n, d, list, centroids, codebook, M, codes, st); break;
        case 8: launch_pq_encode_t<8>(x, n, d, list, centroids, codebook, M, codes, st); break;
        case 12: launch_pq_encode_t<12>(x, n, d, list, centroids, codebook, M, codes, st); break;
        case 16: launch_pq_encode_t<16>(x, n, d, list, centroids, codebook, M, codes, st); break;
        case 24: launch_pq_encode_t<24>(x, n, d, list, centroids, codebook, M, codes, st); break;
        case 32: launch_pq_encode_t<32>(x, n, d, list, centroids, codebook, M, codes, st); break;
        case 48: launch_pq_encode_t<48>(x, n, d, list, centroids, codebook, M, codes, st); break;
        default: {
            dim3 grid((unsigned)((n + 127) / 128), M);
            pq_encode_generic_kernel<<<grid, 128, 0, st>>>(x, n, d, list, centroids, codebook, M, dsub, codes);
        }
    }
}

// 4-bit residual encoding: nearest of the 16 entries of each sub-quantizer (L2, the arithmetic and the first-minimum
// tie rule of pq_encode_kernel).  grid (row tiles of 128, M / 2 when packed, else M); a block stages the 16 x dsub
// codebooks of the sub-quantizers it encodes.  packed: codes [n, M/2], byte b = c[2b] | c[2b+1] << 4 (faiss order);
// unpacked (PQ training's assignment step): codes [n, M], one code per byte.
__global__ __launch_bounds__(128)
void pq_encode4_kernel(const float* __restrict__ x, int64_t n, int d, const int32_t* __restrict__ list,
                       const float* __restrict__ centroids, const float* __restrict__ codebook, int M, int packed,
                       uint8_t* __restrict__ codes) {
    extern __shared__ __align__(16) float cb4_s[];           // [per][16][dsub]
    const int dsub = d / M, per = packed ? 2 : 1, m0 = blockIdx.y * per;
    for (int i = threadIdx.x; i < per * 16 * dsub; i += blockDim.x) cb4_s[i] = codebook[(size_t)m0 * 16 * dsub + i];
    __syncthreads();
    const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n) return;
    unsigned byte = 0;
    for (int h = 0; h < per; ++h) {
        const int m = m0 + h;
        const float* xr = x + (size_t)row * d + m * dsub;
        const float* cr = list ? centroids + (size_t)list[row] * d + m * dsub : nullptr;
        float best = FLT_MAX;
        int bj = 0;
        for (int j = 0; j < 16; ++j) {
            float dist = 0.f;
            for (int t = 0; t < dsub; ++t) {
                const float r = cr ? xr[t] - __ldg(cr + t) : xr[t];
                const float df = r - cb4_s[(h * 16 + j) * dsub + t];
                dist = fmaf(df, df, dist);
            }
            if (dist < best) { best = dist; bj = j; }
        }
        byte |= (unsigned)bj << (4 * h);
    }
    codes[(size_t)row * (M / per) + blockIdx.y] = (uint8_t)byte;
}

void launch_pq_encode4(const float* x, int64_t n, int d, const int32_t* list, const float* centroids,
                       const float* codebook, int M, bool packed, uint8_t* codes, cudaStream_t st) {
    if (n <= 0) return;
    const size_t smem = (size_t)(packed ? 2 : 1) * 16 * (d / M) * 4;
    static PerDeviceSize configured;
    if (smem > 48 * 1024 && configured.raise(smem))
        cudaFuncSetAttribute(pq_encode4_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    dim3 grid((unsigned)((n + 127) / 128), packed ? M / 2 : M);
    pq_encode4_kernel<<<grid, 128, smem, st>>>(x, n, d, list, centroids, codebook, M, packed ? 1 : 0, codes);
}

// =============================================================================================================
// k-means update steps (index.train(): faiss Clustering for the coarse quantizer, ProductQuantizer::train for the
// PQ codebooks; reference call sites src/indicies/ivf_flat.py:166, ivf_pq.py:170).  The assignment steps are the
// coarse quantizer itself (tensor-core scorer + exact re-score) and pq_encode_kernel; these accumulate the member sums.
// =============================================================================================================
// Member sums in a fixed order, so that training gives the same centroids / codebooks on every run: the members are
// grouped by cluster with a stable radix sort (ties keep ascending row order), then one warp per cluster adds its
// members' rows in ascending row order.  An "item" is one row (k-means: key = its cluster, its vector = x[item]) or one
// (row, sub-quantizer) pair (PQ: key = m * ksub + code, its vector = the m-th sub-vector of the row).
__global__ void accumulate_keys_kernel(int64_t nitems, int M, const int32_t* __restrict__ assign, int k,
                                       const uint8_t* __restrict__ codes, int ksub, int32_t* __restrict__ keys,
                                       int64_t* __restrict__ items) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nitems; i += (int64_t)gridDim.x * blockDim.x) {
        int key;
        if (codes) key = codes[i] < ksub ? (int)(i % M) * ksub + codes[i] : M * ksub;   // codes >= ksub: ignored
        else key = (assign[i] >= 0 && assign[i] < k) ? assign[i] : k;      // out-of-range assignments: ignored
        keys[i] = key;
        items[i] = i;
    }
}
__global__ void accumulate_bounds_kernel(const int32_t* __restrict__ keys, int64_t nitems, int nkeys,
                                         int64_t* __restrict__ begin, int64_t* __restrict__ end) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nitems; i += (int64_t)gridDim.x * blockDim.x) {
        const int key = keys[i];
        if (key >= nkeys) continue;
        if (i == 0 || keys[i - 1] != key) begin[key] = i;
        if (i == nitems - 1 || keys[i + 1] != key) end[key] = i + 1;
    }
}
// sums[key, 0:w] += sum of the item vectors of `key` in ascending item order, counts[key] += their number
__global__ void accumulate_sums_kernel(const float* __restrict__ x, int d, int M, int w, const int64_t* __restrict__ items,
                                       const int64_t* __restrict__ begin, const int64_t* __restrict__ end, int nkeys,
                                       float* __restrict__ sums, float* __restrict__ counts) {
    const int lane = threadIdx.x & 31;
    const int key = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    if (key >= nkeys) return;
    const int64_t b = begin[key], e = end[key];
    for (int c0 = 0; c0 < w; c0 += 32) {
        const int c = c0 + lane;
        float acc = 0.f;
        for (int64_t j = b; j < e; ++j) {
            const int64_t it = items[j];
            if (c < w) acc += x[(it / M) * d + (it % M) * w + c];
        }
        if (c < w && e > b) sums[(size_t)key * w + c] += acc;
    }
    if (lane == 0 && e > b) counts[key] += (float)(e - b);
}

static cudaError_t accumulate_sorted(const float* x, int64_t n, int d, int M, const int32_t* assign, int k,
                                     const uint8_t* codes, int nkeys, float* sums, float* counts, cudaStream_t st) {
    const int64_t nitems = n * M;
    int bits = 1;
    while ((1 << bits) <= nkeys) ++bits;                                   // key nkeys (ignored items) must fit
    int32_t *keys = nullptr, *keys_sorted = nullptr;
    int64_t *items = nullptr, *items_sorted = nullptr, *bounds = nullptr;
    void* tmp = nullptr;
    size_t tmp_bytes = 0;
    cudaError_t e = cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys, keys_sorted, items, items_sorted, nitems, 0, bits, st);
    if (e == cudaSuccess) e = cudaMallocAsync(&keys, (size_t)nitems * 4, st);
    if (e == cudaSuccess) e = cudaMallocAsync(&keys_sorted, (size_t)nitems * 4, st);
    if (e == cudaSuccess) e = cudaMallocAsync(&items, (size_t)nitems * 8, st);
    if (e == cudaSuccess) e = cudaMallocAsync(&items_sorted, (size_t)nitems * 8, st);
    if (e == cudaSuccess) e = cudaMallocAsync(&bounds, (size_t)nkeys * 2 * 8, st);
    if (e == cudaSuccess) e = cudaMallocAsync(&tmp, tmp_bytes, st);
    if (e == cudaSuccess) {
        const int blocks = (int)std::min<int64_t>(8 * (int64_t)num_sms(), (nitems + 255) / 256);
        accumulate_keys_kernel<<<blocks, 256, 0, st>>>(nitems, M, assign, k, codes, nkeys / M, keys, items);
        e = cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys, keys_sorted, items, items_sorted, nitems, 0, bits, st);
    }
    if (e == cudaSuccess) e = cudaMemsetAsync(bounds, 0, (size_t)nkeys * 2 * 8, st);
    if (e == cudaSuccess) {
        const int blocks = (int)std::min<int64_t>(8 * (int64_t)num_sms(), (nitems + 255) / 256);
        accumulate_bounds_kernel<<<blocks, 256, 0, st>>>(keys_sorted, nitems, nkeys, bounds, bounds + nkeys);
        accumulate_sums_kernel<<<(nkeys + 7) / 8, 256, 0, st>>>(x, d, M, d / M, items_sorted, bounds, bounds + nkeys, nkeys,
                                                              sums, counts);
        e = cudaGetLastError();
    }
    cudaFreeAsync(tmp, st);
    cudaFreeAsync(bounds, st);
    cudaFreeAsync(items_sorted, st);
    cudaFreeAsync(items, st);
    cudaFreeAsync(keys_sorted, st);
    cudaFreeAsync(keys, st);
    return e;
}

// sums[k, d] += x[row] for row's cluster, counts[k] += 1
cudaError_t launch_kmeans_accumulate(const float* x, int64_t n, int d, const int32_t* assign, int k, float* sums, float* counts,
                                     cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    return accumulate_sorted(x, n, d, 1, assign, k, nullptr, k, sums, counts, st);
}

// PQ: sums[m, code, :] += r[row, m*dsub : (m+1)*dsub], counts[m, code] += 1  (sums [M, ksub, dsub], counts [M, ksub])
cudaError_t launch_pq_accumulate(const float* r, int64_t n, int d, int M, int ksub, const uint8_t* codes, float* sums,
                                 float* counts, cudaStream_t st) {
    if (n <= 0) return cudaSuccess;
    return accumulate_sorted(r, n, d, M, nullptr, 0, codes, M * ksub, sums, counts, st);
}

// =============================================================================================================
// layout transforms (build side)
// =============================================================================================================
__device__ __forceinline__ int find_segment(const int64_t* seg_starts, int nseg, int64_t row) {
    int lo = 0, hi = nseg;  // seg_starts has nseg+1 entries; find s with starts[s] <= row < starts[s+1]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (seg_starts[mid] <= row) lo = mid; else hi = mid;
    }
    return lo;
}

__global__ void slot_of_sorted_kernel(const int32_t* __restrict__ sorted_list, int64_t n,
                                      const int64_t* __restrict__ list_nat_off,
                                      const int64_t* __restrict__ list_slot_off, int64_t* __restrict__ dst_row) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int l = sorted_list[i];
        dst_row[i] = list_slot_off[l] + (i - list_nat_off[l]);
    }
}
void launch_slot_of_sorted(const int32_t* sorted_list, int64_t n, const int64_t* list_nat_off,
                           const int64_t* list_slot_off, int64_t* dst_row, cudaStream_t st) {
    if (n <= 0) return;
    const int blocks = (int)std::min<int64_t>(4096, (n + 255) / 256);
    slot_of_sorted_kernel<<<blocks, 256, 0, st>>>(sorted_list, n, list_nat_off, list_slot_off, dst_row);
}

__global__ void pq_interleave_kernel(const uint8_t* const* __restrict__ seg_ptrs,
                                     const int64_t* __restrict__ seg_starts, int nseg,
                                     const int64_t* __restrict__ sorted_src, const int32_t* __restrict__ sorted_list,
                                     int64_t n, const int64_t* __restrict__ list_nat_off,
                                     const int64_t* __restrict__ list_slot_off, int M, uint8_t* __restrict__ codes_il) {
    const int K = M / 16;
    const int64_t total = n * K;
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < total; w += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = w / K;
        const int r = (int)(w % K);
        const int64_t src = sorted_src[i];
        const int seg = find_segment(seg_starts, nseg, src);
        const uint8_t* code = seg_ptrs[seg] + (size_t)(src - seg_starts[seg]) * M;
        const int l = sorted_list[i];
        const int64_t slot = list_slot_off[l] + (i - list_nat_off[l]);
        const int v = (int)(slot & 31);
        const int g = v / K;
        unsigned words[4];
#pragma unroll
        for (int wd = 0; wd < 4; ++wd) {
            unsigned x = 0;
#pragma unroll
            for (int b = 0; b < 4; ++b) x |= (unsigned)code[pq_sub(K, g, r, wd * 4 + b)] << (8 * b);
            words[wd] = x;
        }
        uint8_t* dst = codes_il + (size_t)(slot - v) * M + pq_chunk_off(K, v, r);
        *reinterpret_cast<uint4*>(dst) = make_uint4(words[0], words[1], words[2], words[3]);
    }
}
void launch_pq_interleave(const uint8_t* const* seg_ptrs, const int64_t* seg_starts, int nseg,
                          const int64_t* sorted_src, const int32_t* sorted_list, int64_t n,
                          const int64_t* list_nat_off, const int64_t* list_slot_off, int M, uint8_t* codes_il,
                          cudaStream_t st) {
    if (n <= 0) return;
    const int64_t total = n * (M / 16);
    const int blocks = (int)std::min<int64_t>(8192, (total + 255) / 256);
    pq_interleave_kernel<<<blocks, 256, 0, st>>>(seg_ptrs, seg_starts, nseg, sorted_src, sorted_list, n,
                                                 list_nat_off, list_slot_off, M, codes_il);
}

__global__ void pq_deinterleave_kernel(const uint8_t* __restrict__ codes_il, const int64_t* __restrict__ list_nat_off,
                                       const int64_t* __restrict__ list_slot_off, int nlist, int M,
                                       uint8_t* __restrict__ codes_nat) {
    const int K = M / 16;
    const int64_t n = list_nat_off[nlist];
    const int64_t total = n * K;
    for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < total; w += (int64_t)gridDim.x * blockDim.x) {
        const int64_t i = w / K;
        const int r = (int)(w % K);
        const int l = find_segment(list_nat_off, nlist, i);   // list_nat_off has nlist+1 entries
        const int64_t slot = list_slot_off[l] + (i - list_nat_off[l]);
        const int v = (int)(slot & 31);
        const int g = v / K;
        const uint4 c = *reinterpret_cast<const uint4*>(codes_il + (size_t)(slot - v) * M + pq_chunk_off(K, v, r));
        const unsigned words[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
        for (int s = 0; s < 16; ++s)
            codes_nat[(size_t)i * M + pq_sub(K, g, r, s)] = (uint8_t)(words[s >> 2] >> (8 * (s & 3)));
    }
}
void launch_pq_deinterleave(const uint8_t* codes_il, const int64_t* list_nat_off, const int64_t* list_slot_off,
                            const int* /*list_len*/, int nlist, int M, uint8_t* codes_nat, cudaStream_t st) {
    pq_deinterleave_kernel<<<4096, 256, 0, st>>>(codes_il, list_nat_off, list_slot_off, nlist, M, codes_nat);
}

// empty lists share their offset with the next list: find_segment must return the LAST list whose offset <= i
// among equal offsets only if it is non-empty.  With starts[s] <= row < starts[s+1] the binary search above
// lands on the unique non-empty list containing row, because an empty list has starts[s] == starts[s+1].

__global__ void gather_rows_kernel(const uint8_t* const* __restrict__ seg_ptrs, const int64_t* __restrict__ seg_starts,
                                   int nseg, const int64_t* __restrict__ sorted_src,
                                   const int64_t* __restrict__ dst_row, int64_t n, int row_words,
                                   unsigned* __restrict__ dst) {
    // one warp per row
    const int lane = threadIdx.x & 31;
    const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
    for (int64_t i = wid; i < n; i += nw) {
        const int64_t src = sorted_src[i];
        const int seg = find_segment(seg_starts, nseg, src);
        const unsigned* s = reinterpret_cast<const unsigned*>(seg_ptrs[seg]) + (size_t)(src - seg_starts[seg]) * row_words;
        unsigned* o = dst + (size_t)(dst_row ? dst_row[i] : i) * row_words;
        if ((row_words & 3) == 0) {
            for (int c = lane * 4; c < row_words; c += 128)
                *reinterpret_cast<uint4*>(o + c) = *reinterpret_cast<const uint4*>(s + c);
        } else {
            for (int c = lane; c < row_words; c += 32) o[c] = s[c];
        }
    }
}
void launch_gather_rows(const uint8_t* const* seg_ptrs, const int64_t* seg_starts, int nseg,
                        const int64_t* sorted_src, const int64_t* dst_row, int64_t n, int row_bytes, uint8_t* dst,
                        cudaStream_t st) {
    if (n <= 0) return;
    const int blocks = (int)std::min<int64_t>(8192, (n * 32 + 255) / 256);
    gather_rows_kernel<<<blocks, 256, 0, st>>>(seg_ptrs, seg_starts, nseg, sorted_src, dst_row, n, row_bytes / 4,
                                               reinterpret_cast<unsigned*>(dst));
}

__global__ void gather_ids_kernel(const int64_t* const* __restrict__ seg_ptrs, const int64_t* __restrict__ seg_starts,
                                  int nseg, const int64_t* __restrict__ sorted_src,
                                  const int64_t* __restrict__ dst_row, int64_t n, int64_t* __restrict__ dst) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t src = sorted_src[i];
        const int seg = find_segment(seg_starts, nseg, src);
        dst[dst_row ? dst_row[i] : i] = seg_ptrs[seg][src - seg_starts[seg]];
    }
}
void launch_gather_ids(const int64_t* const* seg_ptrs, const int64_t* seg_starts, int nseg,
                       const int64_t* sorted_src, const int64_t* dst_row, int64_t n, int64_t* dst, cudaStream_t st) {
    if (n <= 0) return;
    const int blocks = (int)std::min<int64_t>(4096, (n + 255) / 256);
    gather_ids_kernel<<<blocks, 256, 0, st>>>(seg_ptrs, seg_starts, nseg, sorted_src, dst_row, n, dst);
}

__global__ void peer_broadcast_kernel(const uint4* __restrict__ src, size_t n16, void* const* __restrict__ dst_ptrs,
                                      int npeers, size_t dst_offset) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x) {
        const uint4 v = src[i];
        for (int p = 0; p < npeers; ++p)
            reinterpret_cast<uint4*>(static_cast<unsigned char*>(dst_ptrs[p]) + dst_offset)[i] = v;
    }
}
void launch_peer_broadcast(const void* src, size_t bytes, void* const* dst_ptrs, int npeers, size_t dst_offset,
                           cudaStream_t st) {
    const size_t n16 = bytes / 16;
    if (n16 == 0 || npeers <= 0) return;
    const int blocks = (int)std::min<size_t>(4 * (size_t)num_sms(), (n16 + 255) / 256);
    peer_broadcast_kernel<<<blocks, 256, 0, st>>>(static_cast<const uint4*>(src), n16, dst_ptrs, npeers, dst_offset);
}

__global__ void fill_i64_kernel(int64_t* p, int64_t n, int64_t v, int64_t step) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        p[i] = v + step * i;
}
void launch_fill_i64(int64_t* p, int64_t n, int64_t v, cudaStream_t st) {
    if (n <= 0) return;
    fill_i64_kernel<<<(int)std::min<int64_t>(4096, (n + 255) / 256), 256, 0, st>>>(p, n, v, 0);
}
void launch_iota_i64(int64_t* p, int64_t n, int64_t start, cudaStream_t st) {
    if (n <= 0) return;
    fill_i64_kernel<<<(int)std::min<int64_t>(4096, (n + 255) / 256), 256, 0, st>>>(p, n, start, 1);
}

// storage conversions of rsb_add: fp32 -> fp16 rounds to nearest even; fp16 -> fp32 is exact
__global__ void f32_to_f16_kernel(const float* __restrict__ src, size_t n, __half* __restrict__ dst) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        dst[i] = __float2half_rn(src[i]);
}
__global__ void f16_to_f32_kernel(const __half* __restrict__ src, size_t n, float* __restrict__ dst) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        dst[i] = __half2float(src[i]);
}
void launch_f32_to_f16(const float* src, size_t n, void* dst, cudaStream_t st) {
    if (n == 0) return;
    f32_to_f16_kernel<<<(int)std::min<size_t>(8192, (n + 255) / 256), 256, 0, st>>>(src, n, static_cast<__half*>(dst));
}
void launch_f16_to_f32(const void* src, size_t n, float* dst, cudaStream_t st) {
    if (n == 0) return;
    f16_to_f32_kernel<<<(int)std::min<size_t>(8192, (n + 255) / 256), 256, 0, st>>>(static_cast<const __half*>(src), n, dst);
}

__global__ void i64_to_i32_kernel(const int64_t* __restrict__ src, int64_t n, int32_t* __restrict__ dst) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        dst[i] = (int32_t)src[i];
}
void launch_i64_to_i32(const int64_t* src, int64_t n, int32_t* dst, cudaStream_t st) {
    if (n <= 0) return;
    i64_to_i32_kernel<<<(int)std::min<int64_t>(4096, (n + 255) / 256), 256, 0, st>>>(src, n, dst);
}

__global__ void list_hist_kernel(const int32_t* __restrict__ list, int64_t n, int nlist, int* hist) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int l = list[i];
        if (l >= 0 && l < nlist) atomicAdd(&hist[l], 1);
    }
}
void launch_list_hist(const int32_t* list, int64_t n, int nlist, int* hist, cudaStream_t st) {
    if (n <= 0) return;
    list_hist_kernel<<<(int)std::min<int64_t>(4096, (n + 255) / 256), 256, 0, st>>>(list, n, nlist, hist);
}

__global__ void compact_slots_i64_kernel(const int64_t* __restrict__ src_slots, const int64_t* __restrict__ list_nat_off,
                                         const int64_t* __restrict__ list_slot_off, int nlist,
                                         int64_t* __restrict__ dst_nat) {
    const int64_t n = list_nat_off[nlist];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int l = find_segment(list_nat_off, nlist, i);
        dst_nat[i] = src_slots[list_slot_off[l] + (i - list_nat_off[l])];
    }
}
void launch_compact_slots_i64(const int64_t* src_slots, const int64_t* list_nat_off, const int64_t* list_slot_off,
                              const int* /*list_len*/, int nlist, int64_t* dst_nat, cudaStream_t st) {
    compact_slots_i64_kernel<<<4096, 256, 0, st>>>(src_slots, list_nat_off, list_slot_off, nlist, dst_nat);
}

}  // namespace rsb
