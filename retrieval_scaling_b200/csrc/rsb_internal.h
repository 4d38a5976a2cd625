// rsb_internal.h -- launcher prototypes shared between the kernel translation units and the C-ABI (rsb_api.cu).
#ifndef RSB_INTERNAL_H_
#define RSB_INTERNAL_H_

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace rsb {

typedef unsigned long long u64;

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) and the SM count are per DEVICE: one process may hold indexes on
// several GPUs (`device=` argument of the Python classes), so "already configured" is remembered per device.
inline int current_device_slot() {
    int d = 0;
    cudaGetDevice(&d);
    return (d < 0 ? 0 : d) & 63;
}
struct PerDeviceSize {
    size_t v[64] = {};
    // true when `bytes` exceeds what this device was configured for (and records it)
    bool raise(size_t bytes) {
        size_t& cur = v[current_device_slot()];
        if (bytes <= cur) return false;
        cur = bytes;
        return true;
    }
};
struct PerDeviceFlag {
    bool done[64] = {};
    bool first() {                       // true exactly once per device
        bool& d = done[current_device_slot()];
        if (d) return false;
        d = true;
        return true;
    }
};
inline int device_num_sms() {
    static int sms[64] = {};
    int& n = sms[current_device_slot()];
    if (!n) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 132;
    }
    return n;
}

// ---- rsb_bert.cu ----------------------------------------------------------------------------------------
// rsb_gemm_f16 (rsb.h) on bf16 A, W, bias, residual and C, for the reader in bf16: epilogue 0 (bias), 1 (bias + GELU)
// or 2 (bias + residual), OR-ed with RSB_GEMM_REVERSED; the same checks and errors (rsb_bert_last_error).
int gemm_bf16(const void* A, const void* W, const void* bias, const void* residual, void* C, int M, int N, int K,
              int epilogue, cudaStream_t stream);

// ---- rsb_dense.cu ---------------------------------------------------------------------------------------
void launch_sgemm_nt(const float* A, int M, const float* B, int N, int K, float* C, int ldc, cudaStream_t st);
void launch_select_rows(const float* S, int nrows, int ncols, int ld, unsigned col_base, int k, int nsplit,
                        u64* out_keys, int* out_cnt, int items_per_row, int item_base, cudaStream_t st);
void launch_merge_items(const u64* keys, const int* cnt, int nq, int nitems, int k_item, int k_out,
                        const int64_t* ids, int64_t id_offset, float* D, int64_t* I, cudaStream_t st);
// X [*, d] rows of elem_bytes 4 (fp32) or 2 (fp16)
int launch_refine_exact(const float* Q, int nq, const void* X, int elem_bytes, int d, const int64_t* I_in, int k_in,
                        int k_out, float* D, int64_t* I, const int64_t* id_map, cudaStream_t st);
int launch_merge_shards(const float* D_all, const int64_t* I_all, int nshards, int nq, int k, int k_out, float* D,
                        int64_t* I, cudaStream_t st);
int launch_merge_shards_peers(const float* const* D_ptrs, const int64_t* const* I_ptrs, int nshards, int nq, int k,
                              int k_out, float* D, int64_t* I, cudaStream_t st);
int launch_merge_shards_peers_scatter(const float* const* D_ptrs, const int64_t* const* I_ptrs, int nshards, int q0,
                                      int nq_slice, int k, int k_out, float* const* D_outs, int64_t* const* I_outs,
                                      int nout, cudaStream_t st);

// ---- rsb_refine.cu (exact re-ranking of candidates against a re-rank store) -------------------------------
struct RefinePlan {
    int nchunks;          // CTAs per query
    int chunk;            // candidates per CTA
    int P;                // sort width (power of two >= chunk)
    int k_item;           // keys a CTA hands to the merge (nchunks > 1)
    size_t ws_bytes;      // partial keys + counts (0 when nchunks == 1)
};
RefinePlan refine_plan(int nq, int k_base, int k);
// P * 8 + d * 4 bytes of shared memory (SQ8, elem_bytes 1: + 2 * d * 4 for vmin / vdiff) <= 200 KB
bool refine_smem_fits(const RefinePlan& p, int d, int elem_bytes);
// The re-rank store [ntotal, d]: rows [0, n_dev) at dev (device memory), rows [n_dev, ntotal) at host (the device
// alias of the mapped page-locked host tier; null when n_dev == ntotal).  elem_bytes 1 (SQ8 codes), 2 (fp16) or 4
// (fp32).  sq: the SQ8 store's [2, d] fp32 (vmin, vdiff), 16-byte aligned (null for fp16 / fp32).
struct RefineStore {
    const void* dev;
    int64_t n_dev;
    const void* host;
    int elem_bytes;
    int d;
    int64_t ntotal;
    const float* sq;
};
// All-device re-rank (s.n_dev == s.ntotal): cand [nq, k_base] ids (-1 = skip); returns <0 if the shared memory the
// kernel needs does not fit (refine_smem_fits)
int launch_refine_rows(const RefinePlan& p, const float* Q, int nq, const RefineStore& s, const int64_t* cand,
                       int k_base, int k, float* D, int64_t* I, void* ws, cudaStream_t st);
// Workspace of a tiered re-rank of nq queries: queries are processed qc at a time, qc = the queries whose worst case
// (k_base * d * elem_bytes each) fits staging_bytes.  qc = 0: staging_bytes is below one query's worst case, or the
// CUB temporary sizes could not be queried.
struct TieredPlan {
    int qc;
    bool smem_ok;
    size_t cub_bytes, ref_bytes;
    size_t off_keys, off_keys2, off_vals, off_vals2, off_slot, off_uniq, off_count, off_cub, off_ref, off_stage, total;
};
TieredPlan tiered_plan(int nq, int k_base, int k, int d, int elem_bytes, size_t staging_bytes);
// Tiered re-rank (s.n_dev < s.ntotal).  host_rows (nullable) += distinct host rows gathered.
cudaError_t launch_refine_tiered(const TieredPlan& p, const float* Q, int nq, const RefineStore& s, const int64_t* cand,
                                 int k_base, int k, float* D, int64_t* I, void* ws, long long* host_rows,
                                 cudaStream_t st);
// SQ8 store (faiss ScalarQuantizer QT_8bit, RS_minmax, per dimension): x [n, d] fp32 (x_f16 = 0) or fp16 (x_f16 = 1);
// sq [2, d] fp32 = (vmin, vdiff).  train: vmin = min over the rows, vdiff = max - vmin.  encode: codes [n, d] uint8;
// with list [n] int32 and centroids [nlist, d] (IVF-SQ8 by residual) row i is encoded as x[i] - centroids[list[i]].
cudaError_t launch_sq8_train(const void* x, int x_f16, int64_t n, int d, float* sq, cudaStream_t st);
cudaError_t launch_sq8_encode(const void* x, int x_f16, int64_t n, int d, const float* sq, uint8_t* codes,
                              cudaStream_t st, const int32_t* list = nullptr, const float* centroids = nullptr);
// enable != 0: time every later tiered chunk's sort / gather / score with events (synchronises per chunk).
// ms3 (nullable) <- the milliseconds accumulated since the previous call, which resets them.
int tiered_profile(int enable, double* ms3);

// ---- rsb_tf32.cu (tensor-core fp32-accurate scores: 3xTF32 on wgmma) ---------------------------------
bool tf32_path_available();
void launch_split_tf32(const float* x, size_t n, float* hi, float* lo, cudaStream_t st);
bool launch_gemm_tf32x3(const float* Ah, const float* Al, int M, const float* Bh, const float* Bl, int N, int K,
                        float* C, int ldc, cudaStream_t st);

// fused scorer + per-half-tile top-8 filter (no score matrix in HBM), see rsb_tf32.cu
size_t fused_cand_per_row(int N);
bool launch_gemm_tf32x3_topt(const float* Ah, const float* Al, int M, const float* Bh, const float* Bl, int N, int K,
                             unsigned col_base, u64* cand, unsigned* xbound, cudaStream_t st);
// rsb_dense.cu: top-kc of a row's candidates + exactness check (flag) ; exhaustive fp32 re-do of flagged rows
int launch_select_cands(const u64* cand, int nrows, int ncand, const unsigned* xbound, int nx, int kc, u64* out_keys,
                        int* out_cnt, int items_per_row, int item, unsigned char* flags, cudaStream_t st);
void launch_exact_rows(const float* Q, int nrows, const void* X, int elem_bytes, int ncols, int d, unsigned col_base,
                       const unsigned char* flags, int kc, u64* out_keys, int* out_cnt, int items_per_row, int item,
                       cudaStream_t st);

// ---- rsb_tf32.cu, fp16 forms: Flat with fp16 storage (the database rows are the fp16 B operand as stored) and the
// IVF coarse quantizer (the centroids split once, as the queries are) ------
// rows [M, K] fp32 -> per row a power-of-two scale s (largest |element| * s in [2^14, 2^15)), hi = fp16(x s),
// lo = fp16(x s - hi), inv = 1 / s
void launch_split_f16(const float* q, int M, int K, void* hi, void* lo, float* inv, cudaStream_t st);
// as launch_gemm_tf32x3 / _topt with S = (Ah + Al) . B^T * inv[row] * inv_b[col]: B [N, K] fp16 rows as stored
// (Bl = inv_b = nullptr, K % 64 == 0), or Bh + Bl with inv_b [N] from launch_split_f16 (K % 8 == 0)
bool launch_gemm_f16(const void* Ah, const void* Al, const float* inv, int M, const void* Bh, const void* Bl,
                     const float* inv_b, int N, int K, float* C, int ldc, cudaStream_t st);
bool launch_gemm_f16_topt(const void* Ah, const void* Al, const float* inv, int M, const void* Bh, const void* Bl,
                          const float* inv_b, int N, int K, unsigned col_base, u64* cand, unsigned* xbound,
                          cudaStream_t st);

// ---- rsb_ivf.cu -----------------------------------------------------------------------------------------
// (query, list) work list, sorted by list so that concurrently running blocks share inverted lists in L2.
struct PairWork {
    int* hist;            // [2 * nlist + 1] scratch (zeroed by the launcher)
    int* cursor;          // [2 * nlist] scratch
    int* icursor;         // [2 * nlist] scratch (paired items)
    int* order;           // [nq * nprobe] out: pair index (q * nprobe + j), list-major
    int2* items;          // [nq * nprobe] out (paired items): (pair a, pair b or -1), list-major
    int* n_items;         // [1] out: number of scan items (= n_pairs unless paired)
    int* n_pairs;         // [1] out: number of valid pairs
    int* item_counter;    // [1] zeroed: dynamic scheduler of the scan kernel
    u64* scan_bytes;      // [1] out: sum over valid pairs of list_len (elements; caller scales by row bytes)
};
size_t pair_work_bytes(int nq, int nprobe, int nlist);
PairWork carve_pair_work(void* base, int nq, int nprobe, int nlist);
// list_rank[l] = position of list l in the order the lists should be visited (may be null: list id order)
// lead_mode 0: a query's lead pair = its best-ranked list that is non-empty HERE; 1: its probe-rank-0 list only
// paired: also build `items`, where two non-lead pairs of the same list form one item (IVF-PQ paired scan)
void launch_pair_setup(const int64_t* coarse_ids, int nq, int nprobe, int nlist, const int* list_len,
                       const int* list_rank, PairWork w, cudaStream_t st, int lead_mode = 0, bool paired = false);

// Per-query constants of the 10-bit quantised table Q (IVF-PQ paired scan).  For every look-up-table entry T of
// sub-quantizer m:  T = lo_m + delta * Q + e,  |e| <= resid_m.
struct PQQuant {
    double base;          // sum_m lo_m
    double delta;         // quantisation step (fp32 value)
    double err;           // sum_m max_j resid_m (evaluated in fp64)
    double amax;          // sum_m max_j |T[m][j]|
};

struct ScanArgs {
    const int64_t* coarse_ids;    // [nq * nprobe]
    const float* coarse_scores;   // [nq * nprobe]
    int nprobe;
    const int* order;
    const int* n_items;
    int* item_counter;
    const int* list_len;          // [nlist]
    const int64_t* list_off;      // [nlist] first slot of the list (IVFPQ: multiple of 32; IVFFLAT: CSR offset)
    unsigned* tau;                // [nq] running per-query threshold (ordered uint, zeroed by launcher)
    // Multi-GPU threshold exchange (rsb_search_preassigned with tau_local_dev set): `tau` then points into THIS GPU's
    // symmetric-memory threshold array (owned and zeroed by the caller) and every raise of tau[q] is also pushed to
    // tau_peers[p][q] of the other GPUs with a fire-and-forget system-scope reduction over NVLink, so every GPU filters
    // with the best k-th-best bound any GPU has found for that query.  Exact: a bound is always the k-th best of real
    // candidates.
    unsigned* const* tau_peers;   // device array of n_peers pointers (entries equal to `tau`'s base are skipped); or null
    int n_peers;
    int tau_external;             // 1: the caller owns and zeroes `tau`
    int k;
    u64* out_keys;                // [nq * nprobe, k]
    int* out_cnt;                 // [nq * nprobe]
    unsigned* dbg_flag;           // nullable: 1 = literal-offset LDS path ran, 2 = generic path
    // IVF-PQ paired scan (null: every item is one pair, a.order[item])
    const int2* items;            // [n_items] (pair a, pair b or -1)
    const int* n_pairs;           // [1] valid pairs (n_items < n_pairs iff some item is paired)
    const unsigned short* qlut;   // [nq][256][64] 10-bit quantised tables
    const PQQuant* quant;         // [nq]
    u64* rescored;                // nullable: += vectors re-scored exactly after the quantised filter
};

// IVF-Flat: rows of d elements, fp32 (elem_bytes 4), fp16 (elem_bytes 2) or SQ8 codes (elem_bytes 1, with sq [2, d]
// fp32 = (vmin, vdiff); by_residual: each score is a.coarse_scores[pair] + the score of the decoded codes); queries
// [nq, d] fp32.  The rows of list l are vecs[list_data[l] + v] (the all-device index: list_data = a.list_off, vecs in
// CSR order); candidate slots are a.list_off[l] + v.  The caller zeroes a.tau (unless external) and a.out_cnt before
// the first scan of a query batch: several scans of one batch (the pieces of a tiered index) share them.
void launch_ivfflat_scan(const ScanArgs& a, const float* queries, const void* vecs, const int64_t* list_data,
                         int elem_bytes, int d, int nq, cudaStream_t st, const float* sq = nullptr,
                         bool by_residual = false);
// Tiered IVF-Flat (rsb_reserve_lists; lists [0, l_dev) in device memory, the rest in page-locked host memory).
// flags [nlist] <- 1 for the host lists (l >= l_dev, non-empty) that a valid pair of coarse_ids [npairs] probes, else 0
void launch_ivf_probed_flags(const int64_t* coarse_ids, int npairs, int nlist, int l_dev, const int* list_len,
                             unsigned char* flags, cudaStream_t st);
// a host piece: len_out[l] = list_len[l] and data_out[l] = stage_off[l] where chunk_of[l] == chunk, else 0
void launch_ivf_piece_tables(const int* list_len, const int64_t* stage_off, const int* chunk_of, int nlist, int chunk,
                             int* len_out, int64_t* data_out, cudaStream_t st);
// placement of a batch sorted by list (stable): see ivf_place_rows_kernel in rsb_ivf.cu.  row_bytes % 16 == 0
void launch_ivf_place_rows(const int32_t* sorted_list, const int64_t* sorted_src, int64_t n, const int64_t* batch_start,
                           const int64_t* dst_base, int l_dev, int64_t host_begin, const void* src_rows,
                           const int64_t* src_ids, int row_bytes, void* dev_rows, void* host_stage, int64_t* ids_slots,
                           cudaStream_t st);

// IVF-PQ
void launch_pq_lut(const float* queries, int nq, int d, int M, const float* codebook_t, float* lut,
                   cudaStream_t st);                                 // lut [nq, 256, 64]
// lut [nq, 256, 64] -> qlut [nq, 256, 64] u16 and quant [nq] (tables for the paired scan)
void launch_pq_lut_quant(const float* lut, int nq, int M, unsigned short* qlut, PQQuant* quant, cudaStream_t st);
int launch_ivfpq_scan(const ScanArgs& a, const float* lut, const uint8_t* codes, int M, int nq,
                      cudaStream_t st);                              // returns <0 if M unsupported
// generic-M path (M not in {16, 32, 64}): table [nq][M][256], codes in natural [slot][M] order
inline bool pq_interleaved_layout(int M) { return M == 16 || M == 32 || M == 64; }
void launch_pq_lut_generic(const float* queries, int nq, int d, int M, const float* codebook, float* lut, cudaStream_t st);
void launch_compact_slots_rows(const uint8_t* src_slots, const int64_t* list_nat_off, const int64_t* list_slot_off, int nlist,
                               int row_bytes, uint8_t* dst_nat, cudaStream_t st);
unsigned probe_dynamic_smem_base(cudaStream_t st);   // shared-window address of dynamic smem in a kernel without static smem
// codebook [M,256,dsub] -> transposed [256, d] (cbT[j][m*dsub + t] = cb[m][j][t]) used by the LUT kernel
void launch_codebook_transpose(const float* cb, int M, int dsub, float* cbT, cudaStream_t st);
// residual PQ encoding: codes[n, M] = argmin_j || (x - centroid[list])_m - cb[m][j] ||^2
void launch_pq_encode(const float* x, int64_t n, int d, const int32_t* list, const float* centroids,
                      const float* codebook, int M, uint8_t* codes, cudaStream_t st);
// 4-bit sub-quantizers (nbits = 4, M_b = M / 2 code bytes per vector), codebook [M, 16, dsub] as stored.
// Table of the byte sub-quantizers T'[b][j] = T[2b][j & 15] + T[2b+1][j >> 4], written in the layout the scan of M_b
// bytes reads: [nq, 256, 64] when pq_interleaved_layout(M_b), else [nq][M_b][256].
void launch_pq_lut4(const float* queries, int nq, int d, int M, const float* codebook, float* lut, cudaStream_t st);
// nearest of the 16 entries per sub-quantizer (x - centroid[list]; list null: x is the residual).  packed: codes
// [n, M/2] with byte b = c[2b] | c[2b+1] << 4 (faiss PQEncoderGeneric order); else codes [n, M], one code per byte.
void launch_pq_encode4(const float* x, int64_t n, int d, const int32_t* list, const float* centroids,
                       const float* codebook, int M, bool packed, uint8_t* codes, cudaStream_t st);
// k-means update steps of index.train(): member sums / counts (float atomics)
cudaError_t launch_kmeans_accumulate(const float* x, int64_t n, int d, const int32_t* assign, int k, float* sums, float* counts,
                              cudaStream_t st);
// codes [n, M] one code per byte (< ksub; larger codes are skipped); sums [M, ksub, d/M], counts [M, ksub]
cudaError_t launch_pq_accumulate(const float* r, int64_t n, int d, int M, int ksub, const uint8_t* codes, float* sums,
                                 float* counts, cudaStream_t st);
// natural codes -> interleaved blocks (see rsb_layout.h).  src_row[i] = row in `codes_nat` of the i-th vector in
// list-sorted order; rank/list via list_of_sorted + list_nat_off.
void launch_pq_interleave(const uint8_t* const* seg_ptrs, const int64_t* seg_starts, int nseg,
                          const int64_t* sorted_src, const int32_t* sorted_list, int64_t n,
                          const int64_t* list_nat_off, const int64_t* list_slot_off, int M,
                          uint8_t* codes_il, cudaStream_t st);
void launch_pq_deinterleave(const uint8_t* codes_il, const int64_t* list_nat_off, const int64_t* list_slot_off,
                            const int* list_len, int nlist, int M, uint8_t* codes_nat, cudaStream_t st);
// gather rows of `row_bytes` bytes (multiple of 4) from segmented storage into dst[dst_row[i]]
void launch_gather_rows(const uint8_t* const* seg_ptrs, const int64_t* seg_starts, int nseg,
                        const int64_t* sorted_src, const int64_t* dst_row, int64_t n, int row_bytes,
                        uint8_t* dst, cudaStream_t st);
void launch_gather_ids(const int64_t* const* seg_ptrs, const int64_t* seg_starts, int nseg,
                       const int64_t* sorted_src, const int64_t* dst_row, int64_t n, int64_t* dst,
                       cudaStream_t st);
// dst_row for PQ slots: slot = list_slot_off[list] + (i - list_nat_off[list]); for CSR: dst_row = i
void launch_slot_of_sorted(const int32_t* sorted_list, int64_t n, const int64_t* list_nat_off,
                           const int64_t* list_slot_off, int64_t* dst_row, cudaStream_t st);
void launch_fill_i64(int64_t* p, int64_t n, int64_t v, cudaStream_t st);
void launch_iota_i64(int64_t* p, int64_t n, int64_t start, cudaStream_t st);
void launch_i64_to_i32(const int64_t* src, int64_t n, int32_t* dst, cudaStream_t st);
void launch_f32_to_f16(const float* src, size_t n, void* dst, cudaStream_t st);   // round to nearest even
void launch_f16_to_f32(const void* src, size_t n, float* dst, cudaStream_t st);
// copy `bytes` (multiple of 16) from src to dst_ptrs[p] + dst_offset for every p < npeers (peer-mapped destinations)
void launch_peer_broadcast(const void* src, size_t bytes, void* const* dst_ptrs, int npeers, size_t dst_offset,
                           cudaStream_t st);
void launch_list_hist(const int32_t* list, int64_t n, int nlist, int* hist, cudaStream_t st);  // hist += counts
// compact slot-space ids (with -1 padding) to natural order
void launch_compact_slots_i64(const int64_t* src_slots, const int64_t* list_nat_off, const int64_t* list_slot_off,
                              const int* list_len, int nlist, int64_t* dst_nat, cudaStream_t st);

}  // namespace rsb
#endif
