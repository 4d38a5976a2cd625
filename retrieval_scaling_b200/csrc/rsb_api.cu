// rsb_api.cu -- the C-ABI of librsb (include/rsb.h): opaque index handle, population / finalisation into the
// searchable layout, and the host-side orchestration of a search (coarse scan -> work list -> LUT -> list scan
// -> merge), everything enqueued on the caller's stream.
#include "../../include/rsb.h"
#include "rsb_internal.h"
#include "rsb_layout.h"

#include <cub/device/device_radix_sort.cuh>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <string>
#include <vector>

using namespace rsb;

// ---------------------------------------------------------------------------------------------------------
// errors
// ---------------------------------------------------------------------------------------------------------
static thread_local std::string g_err;
static int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}
#define CU(expr)                                                                                     \
    do {                                                                                             \
        cudaError_t e__ = (expr);                                                                    \
        if (e__ != cudaSuccess)                                                                      \
            return fail(e__ == cudaErrorMemoryAllocation ? RSB_ERR_OOM : RSB_ERR_CUDA, "%s: %s (%s:%d)", #expr, \
                        cudaGetErrorString(e__), __FILE__, __LINE__);                                \
    } while (0)
#define CHECK_LAUNCH() CU(cudaPeekAtLastError())
#define RSB_TRY(expr)              \
    do {                           \
        int rc__ = (expr);         \
        if (rc__ != RSB_OK) return rc__; \
    } while (0)

static inline size_t align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

// ---------------------------------------------------------------------------------------------------------
// handle
// ---------------------------------------------------------------------------------------------------------
struct Segment {
    void* payload = nullptr;   // [n, d] in the storage dtype (FLAT / IVFFLAT) or uint8 [n, M] (IVFPQ)
    int64_t* ids = nullptr;    // [n]
    int32_t* list = nullptr;   // [n] (IVF only)
    int64_t n = 0;
};

// A page-locked host block of a tiered index: rows [r0, r0 + n) of the index, exactly n * row_bytes bytes
struct HostBlock {
    void* p = nullptr;
    int64_t r0 = 0, n = 0;
};
static const size_t kDefaultStagingBytes = (size_t)256 << 20;   // RSB_OPT_STAGING_BYTES default (per buffer)

// The split of a tiered index between device and page-locked host memory: rows [0, dev_rows) live in the handle's
// `payload`, rows [dev_rows, rows) in `blocks`.  A tiered Flat index (RSB_OPT_DEVICE_ROWS, fp16 only) allocates the
// device tier once, at dev_rows rows, and adds one block per add; a reserved IVFFLAT index (rsb_reserve_lists) counts
// CSR slots, with dev_rows the slots of lists [0, l_dev) and one block for the other lists.  Search streams the host
// rows through two staging buffers of the workspace on copy_st (StagePipe).
struct HostTier {
    int64_t dev_rows = -1;                 // -1: not tiered
    int64_t rows = 0;                      // Flat: rows added (ntotal + n_staged); IVFFLAT: slots reserved
    std::vector<HostBlock> blocks;         // in row order
    // one staging buffer of the search: Flat: as requested (clamped per search); IVFFLAT: clamped at reservation to
    // [largest host list, host tier], in bytes that need not be whole rows
    size_t staging_bytes = kDefaultStagingBytes;
    cudaStream_t copy_st = nullptr;
    cudaEvent_t stage_ready[2] = {}, stage_free[2] = {}, copy_start = nullptr, copy_done = nullptr, flags_ready = nullptr;
    unsigned char* pinned = nullptr;       // IVFFLAT, page-locked: the per-batch table the search copies to the device
                                           // (stage_off int64 [nlist], chunk_of int32 [nlist]), then probed flags [nlist]
};

struct rsb_index {
    // IVFPQ: M sub-quantizers of nbits bits each (faiss' values: codebook, encoding, training, rsb_info) and
    // Mb = M * nbits / 8 code bytes per vector (layout, interleave, tables, scan, export).  nbits = 4 packs two codes
    // per byte and is scanned as an 8-bit index of Mb byte sub-quantizers (rsb_ivf.cu, pq_lut4_kernel).
    int kind = 0, d = 0, nlist = 0, M = 0, nbits = 0, dsub = 0, Mb = 0;
    int dtype = RSB_DTYPE_F32;   // storage of FLAT / IVFFLAT rows: RSB_DTYPE_F32, RSB_DTYPE_F16 or (IVFFLAT) RSB_DTYPE_SQ8
    // IVFFLAT with RSB_DTYPE_SQ8 (faiss IndexIVFScalarQuantizer, QT_8bit): sq [2, d] = (vmin, vdiff); by_residual encodes
    // x - c_list and adds the list's coarse score to every score of the list
    float* sq = nullptr;
    bool has_sq = false, by_residual = false;
    float* centroids = nullptr;
    float* codebook = nullptr;
    float* codebook_t = nullptr;
    // fp16 hi/lo split of the centroids and their inverse row scales (launch_split_f16): the B operand of the
    // tensor-core coarse scan, [nlist, d] fp16 each and [nlist] fp32
    uint16_t *cent_hi = nullptr, *cent_lo = nullptr;
    float* cent_inv = nullptr;
    bool coarse_tensor = true;
    float *flat_hi = nullptr, *flat_lo = nullptr;   // FLAT: tf32 hi/lo split of the database rows
    bool flat_tensor = true;
    bool has_centroids = false, has_codebook = false;

    std::vector<Segment> staging;
    int64_t n_staged = 0;
    int64_t next_id = 0;       // sequential id for adds without ids

    // searchable layout
    int64_t ntotal = 0;        // vectors in the searchable layout
    int64_t nslots = 0;        // slots (IVFPQ: lists padded to 32)
    uint8_t* payload = nullptr;
    size_t payload_bytes = 0;
    int64_t* ids_slots = nullptr;
    int* list_len = nullptr;           // [nlist]
    int* list_rank = nullptr;          // [nlist] position of the list in descending-length order (work-list order)
    int64_t* list_slot_off = nullptr;  // [nlist + 1]
    int64_t* list_nat_off = nullptr;   // [nlist + 1]
    int max_list_len = 0;

    // tiered Flat: only the ids go through the staging segments.  Reserved IVFFLAT: the CSR layout is fixed up front
    // from the reserved list sizes; ids, list tables, centroids and the SQ8 range stay on the device.  rsb_add /
    // rsb_add_preassigned / rsb_add_codes place every row in its final slot; ntotal counts the rows placed so far
    // (nslots the rows reserved).
    HostTier tier;
    int l_dev = 0;
    std::vector<int> ivf_len;              // [nlist] reserved sizes
    std::vector<int64_t> ivf_off;          // [nlist + 1] CSR offsets
    std::vector<int64_t> ivf_fill;         // [nlist] rows placed so far
    int* dev_len = nullptr;                // [nlist] device: list_len on lists [0, l_dev), 0 elsewhere
    bool tiered() const { return tier.dev_rows >= 0; }
    bool ivf_reserved() const { return kind == RSB_IVFFLAT && tiered(); }
    // rows in device memory (RSB_INFO_DEVICE_ROWS) and in the host tier
    int64_t device_rows() const { return tiered() ? std::min(tier.dev_rows, tier.rows) : ntotal + n_staged; }
    int64_t host_rows() const { return tiered() ? tier.rows - device_rows() : 0; }

    // profiling
    bool prof = false;
    // ring of event sets: one set per profiled search since the last rsb_get_profile (which averages them), so a
    // benchmark can time many back-to-back searches without synchronising between them
    static const int kProfSets = 64;
    cudaEvent_t evs[kProfSets][6] = {};
    cudaEvent_t* ev = evs[0];
    int ev_done = 0;
    unsigned long long* prof_dev = nullptr;  // [4]: scan elements, pairs, scan path flag, re-scored vectors
    long launches = 0;
    int elem_bytes() const { return dtype == RSB_DTYPE_SQ8 ? 1 : dtype == RSB_DTYPE_F16 ? 2 : 4; }
    size_t row_bytes() const { return kind == RSB_IVFPQ ? (size_t)Mb : (size_t)d * elem_bytes(); }
    int ksub() const { return 1 << nbits; }
};

static void free_segment(Segment& s) {
    cudaFree(s.payload); cudaFree(s.ids); cudaFree(s.list);
    s = Segment();
}
static void free_layout(rsb_index* h) {
    cudaFree(h->payload); cudaFree(h->ids_slots); cudaFree(h->list_len); cudaFree(h->list_rank);
    cudaFree(h->dev_len); h->dev_len = nullptr;
    cudaFree(h->flat_hi); cudaFree(h->flat_lo);
    h->flat_hi = nullptr; h->flat_lo = nullptr; h->list_rank = nullptr;
    cudaFree(h->list_slot_off); cudaFree(h->list_nat_off);
    h->payload = nullptr; h->ids_slots = nullptr; h->list_len = nullptr;
    h->list_slot_off = nullptr; h->list_nat_off = nullptr;
    h->ntotal = 0; h->nslots = 0; h->payload_bytes = 0; h->max_list_len = 0;
}
static void free_tier(HostTier& t) {
    if (t.copy_st) {   // a search in flight may still copy from the host blocks
        cudaStreamSynchronize(t.copy_st);
        cudaStreamDestroy(t.copy_st);
    }
    for (cudaEvent_t e : {t.stage_ready[0], t.stage_ready[1], t.stage_free[0], t.stage_free[1], t.copy_start, t.copy_done,
                          t.flags_ready})
        if (e) cudaEventDestroy(e);
    for (auto& b : t.blocks) if (b.p) cudaFreeHost(b.p);
    if (t.pinned) cudaFreeHost(t.pinned);
    t = HostTier();
}

extern "C" int rsb_version(void) { return RSB_VERSION; }
extern "C" const char* rsb_last_error(void) { return g_err.c_str(); }

static int create_common(int kind, int d, int nlist, int M, int nbits, int dtype, rsb_index_t** out) {
    if (!out) return fail(RSB_ERR_INVALID, "out is NULL");
    *out = nullptr;
    if (d <= 0 || (d & 3)) return fail(RSB_ERR_INVALID, "dimension must be a positive multiple of 4, got %d", d);
    if (dtype != RSB_DTYPE_F32 && dtype != RSB_DTYPE_F16 && !(dtype == RSB_DTYPE_SQ8 && kind == RSB_IVFFLAT))
        return fail(RSB_ERR_INVALID, "dtype must be RSB_DTYPE_F32 or RSB_DTYPE_F16%s, got %d",
                    kind == RSB_IVFFLAT ? " or RSB_DTYPE_SQ8" : "", dtype);
    if (dtype == RSB_DTYPE_SQ8 && d % 16)
        return fail(RSB_ERR_INVALID, "SQ8 storage needs whole 16-byte rows: d = %d is not a multiple of 16", d);
    if (dtype == RSB_DTYPE_F16) {
        if (d % 8) return fail(RSB_ERR_INVALID, "fp16 storage needs 16-byte rows: d = %d is not a multiple of 8", d);
        if (kind == RSB_FLAT && d % 64)
            return fail(RSB_ERR_UNSUPPORTED, "the fp16 Flat scorer (wgmma, 64 fp16 per K step) needs d %% 64 == 0, got %d", d);
    }
    if (kind != RSB_FLAT && nlist <= 0) return fail(RSB_ERR_INVALID, "nlist must be > 0, got %d", nlist);
    if (kind == RSB_IVFPQ) {
        if (nbits != 8 && nbits != 4) return fail(RSB_ERR_UNSUPPORTED, "nbits must be 8 or 4, got %d", nbits);
        if (M <= 0 || d % M) return fail(RSB_ERR_INVALID, "d = %d is not divisible by M = %d", d, M);
        if (nbits == 8 && !pq_interleaved_layout(M) && ((M & 3) || M > 128))
            return fail(RSB_ERR_UNSUPPORTED, "n_subquantizers must be 16, 32, 64 (tuned path) or a multiple of 4 up to 128 (got %d)", M);
        if (nbits == 4 && ((M & 7) || M / 2 > 128))
            return fail(RSB_ERR_INVALID, "4-bit codes need M %% 8 == 0 and M / 2 <= 128 code bytes (got M = %d)", M);
    }
    rsb_index* h = new rsb_index();
    h->kind = kind; h->d = d; h->nlist = kind == RSB_FLAT ? 1 : nlist; h->M = M; h->nbits = nbits; h->dtype = dtype;
    h->dsub = M ? d / M : 0;
    h->Mb = M * nbits / 8;
    for (auto& set : h->evs) for (auto& e : set) cudaEventCreate(&e);
    if (cudaMalloc(&h->prof_dev, 32) != cudaSuccess) { delete h; return fail(RSB_ERR_OOM, "cudaMalloc failed"); }
    cudaMemset(h->prof_dev, 0, 32);
    *out = h;
    return RSB_OK;
}
extern "C" int rsb_flat_create(int d, int dtype, rsb_index_t** out) {
    return create_common(RSB_FLAT, d, 1, 0, 0, dtype, out);
}
extern "C" int rsb_ivfflat_create(int d, int nlist, int dtype, rsb_index_t** out) {
    return create_common(RSB_IVFFLAT, d, nlist, 0, 0, dtype, out);
}
extern "C" int rsb_ivfpq_create(int d, int nlist, int M, int nbits, rsb_index_t** out) {
    return create_common(RSB_IVFPQ, d, nlist, M, nbits, RSB_DTYPE_F32, out);
}
extern "C" int rsb_free(rsb_index_t* h) {
    if (!h) return RSB_OK;
    for (auto& s : h->staging) free_segment(s);
    free_layout(h);
    cudaFree(h->centroids); cudaFree(h->codebook); cudaFree(h->codebook_t); cudaFree(h->prof_dev); cudaFree(h->sq);
    cudaFree(h->cent_hi); cudaFree(h->cent_lo); cudaFree(h->cent_inv);
    for (auto& set : h->evs) for (auto& e : set) if (e) cudaEventDestroy(e);
    free_tier(h->tier);
    delete h;
    return RSB_OK;
}

// ---------------------------------------------------------------------------------------------------------
// trained state
// ---------------------------------------------------------------------------------------------------------
extern "C" int rsb_set_centroids(rsb_index_t* h, const float* c, rsb_stream_t stream) {
    if (!h || !c) return fail(RSB_ERR_INVALID, "null argument");
    if (h->kind == RSB_FLAT) return fail(RSB_ERR_INVALID, "a Flat index has no centroids");
    if (h->ntotal || h->n_staged || h->ivf_reserved())
        return fail(RSB_ERR_STATE, "cannot change centroids of a populated (or reserved) index");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t bytes = (size_t)h->nlist * h->d * 4;
    if (!h->centroids) CU(cudaMalloc(&h->centroids, bytes));
    CU(cudaMemcpyAsync(h->centroids, c, bytes, cudaMemcpyDeviceToDevice, st));
    if (!h->cent_hi) CU(cudaMalloc(&h->cent_hi, bytes / 2));
    if (!h->cent_lo) CU(cudaMalloc(&h->cent_lo, bytes / 2));
    if (!h->cent_inv) CU(cudaMalloc(&h->cent_inv, (size_t)h->nlist * 4));
    launch_split_f16(h->centroids, h->nlist, h->d, h->cent_hi, h->cent_lo, h->cent_inv, st);
    CHECK_LAUNCH();
    h->has_centroids = true;
    return RSB_OK;
}
extern "C" int rsb_set_pq_codebook(rsb_index_t* h, const float* cb, rsb_stream_t stream) {
    if (!h || !cb) return fail(RSB_ERR_INVALID, "null argument");
    if (h->kind != RSB_IVFPQ) return fail(RSB_ERR_INVALID, "not an IVFPQ index");
    if (h->ntotal || h->n_staged) return fail(RSB_ERR_STATE, "cannot change the codebook of a populated index");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t bytes = (size_t)h->M * h->ksub() * h->dsub * 4;
    if (!h->codebook) CU(cudaMalloc(&h->codebook, bytes));
    CU(cudaMemcpyAsync(h->codebook, cb, bytes, cudaMemcpyDeviceToDevice, st));
    if (h->nbits == 8) {   // the 8-bit table kernels read the codebook transposed; pq_lut4_kernel reads it as stored
        if (!h->codebook_t) CU(cudaMalloc(&h->codebook_t, bytes));
        launch_codebook_transpose(h->codebook, h->M, h->dsub, h->codebook_t, st);
        CHECK_LAUNCH();
    }
    h->has_codebook = true;
    return RSB_OK;
}
extern "C" int rsb_get_centroids(rsb_index_t* h, float* out, rsb_stream_t stream) {
    if (!h || !out) return fail(RSB_ERR_INVALID, "null argument");
    if (!h->has_centroids) return fail(RSB_ERR_STATE, "index has no centroids");
    CU(cudaMemcpyAsync(out, h->centroids, (size_t)h->nlist * h->d * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return RSB_OK;
}
extern "C" int rsb_get_pq_codebook(rsb_index_t* h, float* out, rsb_stream_t stream) {
    if (!h || !out) return fail(RSB_ERR_INVALID, "null argument");
    if (!h->has_codebook) return fail(RSB_ERR_STATE, "index has no PQ codebook");
    CU(cudaMemcpyAsync(out, h->codebook, (size_t)h->M * h->ksub() * h->dsub * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return RSB_OK;
}

static bool is_sq8_ivf(const rsb_index* h) { return h->kind == RSB_IVFFLAT && h->dtype == RSB_DTYPE_SQ8; }
extern "C" int rsb_set_sq_range(rsb_index_t* h, const float* sq, rsb_stream_t stream) {
    if (!h || !sq) return fail(RSB_ERR_INVALID, "null argument");
    if (!is_sq8_ivf(h)) return fail(RSB_ERR_INVALID, "only an IVFFLAT index with RSB_DTYPE_SQ8 storage has a scalar-quantizer range");
    if (h->ntotal || h->n_staged || h->ivf_reserved())
        return fail(RSB_ERR_STATE, "cannot change the range of a populated (or reserved) index (its codes use it)");
    const size_t bytes = (size_t)2 * h->d * 4;
    if (!h->sq) CU(cudaMalloc(&h->sq, bytes));
    CU(cudaMemcpyAsync(h->sq, sq, bytes, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    h->has_sq = true;
    return RSB_OK;
}
extern "C" int rsb_get_sq_range(rsb_index_t* h, float* out, rsb_stream_t stream) {
    if (!h || !out) return fail(RSB_ERR_INVALID, "null argument");
    if (!is_sq8_ivf(h)) return fail(RSB_ERR_INVALID, "only an IVFFLAT index with RSB_DTYPE_SQ8 storage has a scalar-quantizer range");
    if (!h->has_sq) return fail(RSB_ERR_STATE, "the scalar-quantizer range is not set");
    CU(cudaMemcpyAsync(out, h->sq, (size_t)2 * h->d * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return RSB_OK;
}

static bool is_trained(const rsb_index* h) {
    if (h->kind == RSB_FLAT) return true;
    if (h->kind == RSB_IVFFLAT) return h->has_centroids && (h->dtype != RSB_DTYPE_SQ8 || h->has_sq);
    return h->has_centroids && h->has_codebook;
}

// ---------------------------------------------------------------------------------------------------------
// dense exact k-NN by inner product (IndexFlatIP semantics): sgemm tiles -> row select -> item merge
// ---------------------------------------------------------------------------------------------------------
// RSB_NO_FUSED_COARSE=1: score matrix + select_rows path (A/B switch for the fused scorer of rsb_tf32.cu)
static const bool g_no_fused = getenv("RSB_NO_FUSED_COARSE") != nullptr;

struct KnnPlan {
    int qb;          // queries per batch
    int chunk;       // database columns per sgemm call (multiple of 4)
    int nchunks, nsplit, items;
    size_t off_S, off_keys, off_cnt, total;
};
static KnnPlan knn_plan(int nq, int64_t n, int k) {
    KnnPlan p;
    p.qb = std::max(1, std::min(nq, 16384));
    const size_t budget = (size_t)1 << 30;  // score tile budget
    int64_t chunk = (int64_t)(budget / ((size_t)p.qb * 4));
    chunk = std::max<int64_t>(1024, chunk / 256 * 256);
    const int64_t n4 = std::max<int64_t>(4, (n + 3) / 4 * 4);
    chunk = std::min(chunk, n4);
    p.chunk = (int)chunk;
    p.nchunks = (int)std::max<int64_t>(1, (n + chunk - 1) / chunk);
    int want = (2 * device_num_sms() + p.qb - 1) / p.qb;
    p.nsplit = std::max(1, std::min(want, std::max(1, p.chunk / 4096)));
    p.items = p.nchunks * p.nsplit;
    size_t o = 0;
    p.off_S = o;    o += align_up((size_t)p.qb * p.chunk * 4);
    p.off_keys = o; o += align_up((size_t)p.qb * p.items * k * 8);
    p.off_cnt = o;  o += align_up((size_t)p.qb * p.items * 4);
    p.total = o;
    return p;
}

// optional tensor-core operands: database rows pre-split into hi/lo parts + scratch for the split queries.
//   tf32 (f16 false, xinv null): xh / xl the tf32 split of fp32 rows, qh / ql the tf32 query split;
//   f16: the database rows x are fp16 and are the B operand themselves (xh / xl unused);
//   xinv set: xh / xl the scaled fp16 split of fp32 rows and xinv [n] their inverse scales (launch_split_f16).
// In both fp16 forms qh / ql hold the scaled fp16 query split and qinv [min(nq, qb)] the inverse scales.
struct TensorOperands {
    const void* xh;
    const void* xl;
    float* qh;   // [min(nq, qb), d]
    float* ql;
    bool f16 = false;
    float* qinv = nullptr;
    const float* xinv = nullptr;
};

// x: [n, d] fp32 rows, or fp16 rows when tc->f16
static int knn_ip_device(rsb_index* h, const float* q, int nq, const void* x, int64_t n, int d, int k,
                         const int64_t* ids, int64_t id_offset, float* D, int64_t* I, void* ws, size_t ws_bytes,
                         cudaStream_t st, const TensorOperands* tc = nullptr) {
    if (nq <= 0) return RSB_OK;
    if (n >= ((int64_t)1 << 32)) return fail(RSB_ERR_UNSUPPORTED, "more than 2^32 rows in one dense scan");
    const KnnPlan p = knn_plan(nq, n, k);
    if (ws_bytes < p.total) return fail(RSB_ERR_OOM, "workspace too small: need %zu bytes, got %zu", p.total, ws_bytes);
    unsigned char* w = static_cast<unsigned char*>(ws);
    float* S = reinterpret_cast<float*>(w + p.off_S);
    u64* keys = reinterpret_cast<u64*>(w + p.off_keys);
    int* cnt = reinterpret_cast<int*>(w + p.off_cnt);
    const bool f16 = tc && tc->f16;                   // fp16 rows
    const bool h16 = tc && (tc->f16 || tc->xinv);     // fp16 operands on wgmma
    const int eb = f16 ? 2 : 4;
    const unsigned char* xb8 = static_cast<const unsigned char*>(x);
    // the B operand of columns [c0, c0 + cols)
    auto bh = [&](int64_t c0) -> const void* {
        return f16 ? xb8 + (size_t)c0 * d * 2
                   : static_cast<const unsigned char*>(tc->xh) + (size_t)c0 * d * (tc->xinv ? 2 : 4);
    };
    auto bl = [&](int64_t c0) -> const void* {
        return f16 ? nullptr : static_cast<const unsigned char*>(tc->xl) + (size_t)c0 * d * (tc->xinv ? 2 : 4);
    };
    auto binv = [&](int64_t c0) -> const float* { return tc->xinv ? tc->xinv + c0 : nullptr; };
    for (int q0 = 0; q0 < nq; q0 += p.qb) {
        const int nb = std::min(p.qb, nq - q0);
        if (n == 0) {
            CU(cudaMemsetAsync(cnt, 0, (size_t)nb * p.items * 4, st));
        }
        if (tc && n > 0) {
            if (h16) launch_split_f16(q + (size_t)q0 * d, nb, d, tc->qh, tc->ql, tc->qinv, st);
            else launch_split_tf32(q + (size_t)q0 * d, (size_t)nb * d, tc->qh, tc->ql, st);
            if (h) h->launches += 1;
        }
        for (int c = 0; c < p.nchunks && n > 0; ++c) {
            const int64_t c0 = (int64_t)c * p.chunk;
            const int cols = (int)std::min<int64_t>(p.chunk, n - c0);
            bool on_tensor = false;
            if (tc && p.nsplit == 1 && k <= 256 && !g_no_fused) {
                // fused scorer + filter: 8 candidates per row per 128-column half tile instead of the score matrix.
                // Worth it when a row's top k spreads thinly over the half tiles (else too many rows need the
                // exhaustive re-do); the candidate arrays live in the region the score tile would have used.
                const size_t ncand = fused_cand_per_row(cols);
                const size_t nx = ncand / 8;
                const size_t need = align_up((size_t)nb * ncand * 8) + align_up((size_t)nb * nx * 4) + align_up((size_t)nb);
                if ((size_t)k <= 2 * nx && ncand <= 16384 && need <= align_up((size_t)p.qb * p.chunk * 4)) {
                    u64* cand = reinterpret_cast<u64*>(w + p.off_S);
                    unsigned* xb = reinterpret_cast<unsigned*>(w + p.off_S + align_up((size_t)nb * ncand * 8));
                    unsigned char* flags = w + p.off_S + align_up((size_t)nb * ncand * 8) + align_up((size_t)nb * nx * 4);
                    const bool scored =
                        h16 ? launch_gemm_f16_topt(tc->qh, tc->ql, tc->qinv, nb, bh(c0), bl(c0), binv(c0), cols, d,
                                                   (unsigned)c0, cand, xb, st)
                            : launch_gemm_tf32x3_topt(tc->qh, tc->ql, nb, static_cast<const float*>(bh(c0)),
                                                      static_cast<const float*>(bl(c0)), cols, d, (unsigned)c0, cand, xb, st);
                    if (scored && launch_select_cands(cand, nb, (int)ncand, xb, (int)nx, k, keys, cnt, p.items, c, flags, st) == 0) {
                        launch_exact_rows(q + (size_t)q0 * d, nb, xb8 + (size_t)c0 * d * eb, eb, cols, d, (unsigned)c0, flags, k,
                                          keys, cnt, p.items, c, st);
                        if (h) h->launches += 3;
                        continue;
                    }
                }
            }
            if (h16)  // fp16 hi/lo query split on wgmma; there is no CUDA-core fp16 path
                on_tensor = launch_gemm_f16(tc->qh, tc->ql, tc->qinv, nb, bh(c0), bl(c0), binv(c0), cols, d, S, p.chunk, st);
            else if (tc)  // 3xTF32 on wgmma (fp32-equivalent accuracy); CUDA-core fp32 tiles otherwise
                on_tensor = launch_gemm_tf32x3(tc->qh, tc->ql, nb, static_cast<const float*>(bh(c0)),
                                               static_cast<const float*>(bl(c0)), cols, d, S, p.chunk, st);
            if (h16 && !on_tensor) return fail(RSB_ERR_CUDA, "the fp16 tensor-core scorer could not be set up (tensor map encoding failed)");
            if (!on_tensor)
                launch_sgemm_nt(q + (size_t)q0 * d, nb, static_cast<const float*>(x) + (size_t)c0 * d, cols, d, S, p.chunk, st);
            launch_select_rows(S, nb, cols, p.chunk, (unsigned)c0, k, p.nsplit, keys, cnt, p.items, c * p.nsplit, st);
            if (h) h->launches += 2;
        }
        launch_merge_items(keys, cnt, nb, p.items, k, k, ids, id_offset, D + (size_t)q0 * k, I + (size_t)q0 * k, st);
        if (h) h->launches += 1;
        CHECK_LAUNCH();
    }
    return RSB_OK;
}

extern "C" size_t rsb_knn_workspace_bytes(int nq, int64_t n, int k) {
    return knn_plan(std::max(nq, 1), std::max<int64_t>(n, 1), std::max(k, 1)).total;
}
extern "C" int rsb_knn_ip(const float* q, int nq, const float* x, int64_t n, int d, int k, int64_t id_offset,
                          float* D, int64_t* I, void* ws, size_t ws_bytes, rsb_stream_t stream) {
    if (nq < 0 || n < 0 || k <= 0 || d <= 0 || (d & 3)) return fail(RSB_ERR_INVALID, "bad shape nq=%d n=%lld d=%d k=%d", nq, (long long)n, d, k);
    if (k > 4096) return fail(RSB_ERR_UNSUPPORTED, "k = %d > 4096 is not supported", k);
    return knn_ip_device(nullptr, q, nq, x, n, d, k, nullptr, id_offset, D, I, ws, ws_bytes, (cudaStream_t)stream);
}

// the copy stream and stage events of a tiered index, on the device current now (which holds the index)
static int ensure_copy_stream(HostTier& t) {
    if (t.copy_st) return RSB_OK;
    CU(cudaStreamCreateWithFlags(&t.copy_st, cudaStreamNonBlocking));
    for (cudaEvent_t* e : {&t.stage_ready[0], &t.stage_ready[1], &t.stage_free[0], &t.stage_free[1], &t.copy_start,
                           &t.copy_done, &t.flags_ready})
        CU(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    return RSB_OK;
}

// bytes of one staging buffer of a tiered search: the requested size, but at least min_rows rows and at most the host
// tier's host_rows (min_rows <= host_rows)
static size_t staging_size(size_t requested, size_t rb, int64_t min_rows, int64_t host_rows) {
    return std::min(std::max(requested, (size_t)min_rows * rb), (size_t)host_rows * rb);
}

// ---------------------------------------------------------------------------------------------------------
// population
// ---------------------------------------------------------------------------------------------------------
static const int kAssignRows = 16384;  // rows per coarse-assignment batch inside rsb_add

// list = argmax_c <x, c> for `n` rows through the index's coarse quantizer (tensor-core candidates + exact fp32
// re-score, or CUDA-core fp32 tiles: coarse_impl below); defined after the search plan
static size_t assign_workspace_bytes(const rsb_index* h, int64_t n);
static int assign_lists(rsb_index* h, const float* x, int64_t n, int32_t* list_out, void* ws, size_t ws_bytes, cudaStream_t st,
                        int64_t r_begin = 0);

extern "C" size_t rsb_add_workspace_bytes(rsb_index_t* h, int64_t n) {
    if (!h || h->kind == RSB_FLAT) return 256;
    return assign_workspace_bytes(h, n);
}

static int stage_common(rsb_index* h, Segment& seg, const int64_t* ids, int64_t n, cudaStream_t st) {
    CU(cudaMalloc(&seg.ids, (size_t)n * 8));
    if (ids) CU(cudaMemcpyAsync(seg.ids, ids, (size_t)n * 8, cudaMemcpyDeviceToDevice, st));
    else launch_iota_i64(seg.ids, n, h->next_id, st);
    h->next_id += n;
    seg.n = n;
    return RSB_OK;
}

// fp32 -> fp16 on the host, rounded to nearest even like launch_f32_to_f16 (nan becomes a quiet nan): fp32 rows of a
// tiered Flat index that land in its host tier are converted where they are
static uint16_t f32_to_f16_host(float v) {
    uint32_t f;
    memcpy(&f, &v, 4);
    const uint32_t sign = (f >> 16) & 0x8000u;
    f &= 0x7fffffffu;
    uint32_t o;
    if (f >= 0x47800000u) {                      // |v| >= 65536, inf or nan
        o = f > 0x7f800000u ? 0x7e00u : 0x7c00u;
    } else if (f < 0x38800000u) {                // |v| < 2^-14: an fp16 subnormal or zero
        float a, s;                              // adding 0.5f rounds (to nearest even) at the subnormal step 2^-24
        memcpy(&a, &f, 4);
        s = a + 0.5f;
        uint32_t su;
        memcpy(&su, &s, 4);
        o = su - 0x3f000000u;
    } else {                                     // rebias the exponent (-112 << 23), round to nearest even
        o = (f + 0xc8000fffu + ((f >> 13) & 1u)) >> 13;
    }
    return (uint16_t)(sign | o);
}

// tiered Flat: rows [pos, pos + n) go to the device tier up to dev_rows and to one new page-locked host block after
// it.  x is device or host memory (pageable or pinned); host rows bound for the host tier are copied (or converted)
// host to host.  Only the ids are staged for rsb_finalize.
static int add_tiered(rsb_index* h, const void* x, int x_dtype, int64_t n, const int64_t* ids, cudaStream_t st) {
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, x) != cudaSuccess) {
        cudaGetLastError();
        attr.type = cudaMemoryTypeUnregistered;
    }
    const bool x_dev = attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged;
    const bool f32 = x_dtype == RSB_DTYPE_F32;
    const int d = h->d;
    const size_t rb = h->row_bytes(), xrb = (size_t)d * (f32 ? 4 : 2);
    const int64_t pos = h->tier.rows;
    const int64_t n_to_dev = std::max<int64_t>(0, std::min<int64_t>(n, h->tier.dev_rows - pos));
    const int64_t n_host = n - n_to_dev;
    const uint8_t* xb = static_cast<const uint8_t*>(x);
    if (n_to_dev && !h->payload) {   // the device tier, once, at its full size
        CU(cudaMalloc(&h->payload, (size_t)h->tier.dev_rows * rb));
        h->payload_bytes = (size_t)h->tier.dev_rows * rb;
    }
    HostBlock blk;
    if (n_host) {
        blk.r0 = pos + n_to_dev;
        blk.n = n_host;
        CU(cudaHostAlloc(&blk.p, (size_t)n_host * rb, cudaHostAllocPortable));
    }
    const int64_t conv_rows = std::max<int64_t>(1, ((int64_t)16 << 20) / (int64_t)rb);   // 16 MB conversion steps
    std::vector<uint16_t> hbuf;
    void* dbuf = nullptr;
    auto run = [&]() -> int {
        // device tier
        uint8_t* dst = h->payload + (size_t)pos * rb;
        if (n_to_dev && !f32) CU(cudaMemcpyAsync(dst, xb, (size_t)n_to_dev * rb, cudaMemcpyDefault, st));
        else if (n_to_dev && x_dev) launch_f32_to_f16(static_cast<const float*>(x), (size_t)n_to_dev * d, dst, st);
        else if (n_to_dev) {
            hbuf.resize((size_t)std::min(n_to_dev, conv_rows) * d);
            for (int64_t r = 0; r < n_to_dev; r += conv_rows) {
                const int64_t m = std::min(conv_rows, n_to_dev - r);
                const float* src = reinterpret_cast<const float*>(xb + (size_t)r * xrb);
                for (size_t i = 0; i < (size_t)m * d; ++i) hbuf[i] = f32_to_f16_host(src[i]);
                // from pageable memory: returns once hbuf has been consumed
                CU(cudaMemcpyAsync(dst + (size_t)r * rb, hbuf.data(), (size_t)m * rb, cudaMemcpyHostToDevice, st));
            }
        }
        if (!n_host) return RSB_OK;
        // host tier
        const uint8_t* src0 = xb + (size_t)n_to_dev * xrb;
        uint8_t* hdst = static_cast<uint8_t*>(blk.p);
        if (!f32 && x_dev) CU(cudaMemcpyAsync(hdst, src0, (size_t)n_host * rb, cudaMemcpyDeviceToHost, st));
        else if (!f32) memcpy(hdst, src0, (size_t)n_host * rb);
        else if (!x_dev) {
            const float* src = reinterpret_cast<const float*>(src0);
            uint16_t* out = static_cast<uint16_t*>(blk.p);
            for (size_t i = 0; i < (size_t)n_host * d; ++i) out[i] = f32_to_f16_host(src[i]);
        } else {   // fp32 rows on the device: converted there, 16 MB of fp16 at a time
            const int64_t step = std::min(conv_rows, n_host);
            CU(cudaMalloc(&dbuf, (size_t)step * rb));
            for (int64_t r = 0; r < n_host; r += step) {
                const int64_t m = std::min(step, n_host - r);
                launch_f32_to_f16(reinterpret_cast<const float*>(src0 + (size_t)r * xrb), (size_t)m * d, dbuf, st);
                CU(cudaMemcpyAsync(hdst + (size_t)r * rb, dbuf, (size_t)m * rb, cudaMemcpyDeviceToHost, st));
            }
            CU(cudaStreamSynchronize(st));
        }
        return RSB_OK;
    };
    int rc = run();
    cudaFree(dbuf);
    Segment seg;
    if (rc == RSB_OK) rc = stage_common(h, seg, ids, n, st);
    if (rc == RSB_OK && cudaPeekAtLastError() != cudaSuccess)
        rc = fail(RSB_ERR_CUDA, "tiered add: %s", cudaGetErrorString(cudaGetLastError()));
    if (rc != RSB_OK) {
        cudaStreamSynchronize(st);
        free_segment(seg);
        cudaFreeHost(blk.p);
        return rc;
    }
    if (n_host) h->tier.blocks.push_back(blk);
    h->staging.push_back(seg);
    h->n_staged += n;
    h->tier.rows += n;
    return RSB_OK;
}

// x: [n, d] in x_dtype (RSB_DTYPE_F32 / RSB_DTYPE_F16); stored in the handle's dtype (fp32 -> fp16 rounds to nearest
// even, fp16 -> fp32 is exact).  IVF list assignment runs on fp32 values (fp16 input is upcast 16384 rows at a time).
static int place_segment(rsb_index* h, const Segment& seg, cudaStream_t st);

static int add_impl(rsb_index* h, const void* x, int x_dtype, const uint8_t* codes_in, int64_t n, const int64_t* ids,
                    const int32_t* list_in, void* ws, size_t ws_bytes, cudaStream_t st) {
    if (!h) return fail(RSB_ERR_INVALID, "null handle");
    if (x_dtype != RSB_DTYPE_F32 && x_dtype != RSB_DTYPE_F16)
        return fail(RSB_ERR_INVALID, "x_dtype must be RSB_DTYPE_F32 or RSB_DTYPE_F16, got %d", x_dtype);
    if (x_dtype == RSB_DTYPE_F16 && h->kind == RSB_IVFPQ)
        return fail(RSB_ERR_UNSUPPORTED, "IVFPQ encodes fp32 rows: pass x as RSB_DTYPE_F32");
    if (n < 0) return fail(RSB_ERR_INVALID, "n < 0");
    if (n == 0) return RSB_OK;
    if (!x && !codes_in) return fail(RSB_ERR_INVALID, "null data pointer");
    if (!is_trained(h))
        return fail(RSB_ERR_STATE, "index is not trained (set centroids%s first)",
                    h->kind == RSB_IVFPQ ? " and PQ codebook" : is_sq8_ivf(h) ? " and the SQ8 range" : "");
    // slots are 32-bit in the candidate keys (2^32) and rsb_finalize sorts (list, row) pairs with a 32-bit item count
    if (h->ntotal + h->n_staged + n >= ((int64_t)1 << 31) - 64 * (int64_t)h->nlist)
        return fail(RSB_ERR_UNSUPPORTED, "more than 2^31 vectors per index shard (shard the datastore across GPUs)");
    if (h->kind == RSB_FLAT && h->tiered()) return add_tiered(h, x, x_dtype, n, ids, st);
    const int64_t next_id0 = h->next_id;
    Segment seg;
    int rc = stage_common(h, seg, ids, n, st);
    if (rc != RSB_OK) { free_segment(seg); return rc; }
    auto bail = [&](int code) { free_segment(seg); return code; };
#define CUB_(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) return bail(fail(e__ == cudaErrorMemoryAllocation ? RSB_ERR_OOM : RSB_ERR_CUDA, "%s: %s", #expr, cudaGetErrorString(e__))); } while (0)
    if (h->kind != RSB_FLAT) {
        CUB_(cudaMalloc(&seg.list, (size_t)n * 4));
        if (list_in) {
            CUB_(cudaMemcpyAsync(seg.list, list_in, (size_t)n * 4, cudaMemcpyDeviceToDevice, st));
        } else if (x_dtype == RSB_DTYPE_F32) {
            // list = argmax_c <x, c>  (fp32-exact, IndexFlatIP quantizer semantics)
            rc = assign_lists(h, static_cast<const float*>(x), n, seg.list, ws, ws_bytes, st);
            if (rc != RSB_OK) return bail(rc);
        } else {
            // fp16 rows: the same quantizer on the upcast values (exact), so the lists are those of the fp32 rows
            const int64_t rows = std::min<int64_t>(n, kAssignRows);
            float* up = nullptr;
            CUB_(cudaMalloc(&up, (size_t)rows * h->d * 4));
            for (int64_t r0 = 0; r0 < n && rc == RSB_OK; r0 += rows) {
                const int64_t nb = std::min<int64_t>(rows, n - r0);
                launch_f16_to_f32(static_cast<const uint16_t*>(x) + (size_t)r0 * h->d, (size_t)nb * h->d, up, st);
                rc = assign_lists(h, up, nb, seg.list, ws, ws_bytes, st, r0);
            }
            cudaStreamSynchronize(st);
            cudaFree(up);
            if (rc != RSB_OK) return bail(rc);
        }
    }
    if (codes_in) {     // IVFPQ codes or SQ8 codes, as stored
        CUB_(cudaMalloc(&seg.payload, (size_t)n * h->row_bytes()));
        CUB_(cudaMemcpyAsync(seg.payload, codes_in, (size_t)n * h->row_bytes(), cudaMemcpyDeviceToDevice, st));
    } else if (is_sq8_ivf(h)) {
        // encode on the device; by residual: x - c_list of the list just assigned (fp16 rows widen exactly)
        CUB_(cudaMalloc(&seg.payload, (size_t)n * h->d));
        CUB_(launch_sq8_encode(x, x_dtype == RSB_DTYPE_F16, n, h->d, h->sq, static_cast<uint8_t*>(seg.payload), st,
                               h->by_residual ? seg.list : nullptr, h->centroids));
    } else if (h->kind == RSB_IVFPQ) {
        CUB_(cudaMalloc(&seg.payload, (size_t)n * h->Mb));
        if (h->nbits == 4)
            launch_pq_encode4(static_cast<const float*>(x), n, h->d, seg.list, h->centroids, h->codebook, h->M, true,
                              static_cast<uint8_t*>(seg.payload), st);
        else launch_pq_encode(static_cast<const float*>(x), n, h->d, seg.list, h->centroids, h->codebook, h->M,
                              static_cast<uint8_t*>(seg.payload), st);
    } else {
        const size_t elems = (size_t)n * h->d;
        CUB_(cudaMalloc(&seg.payload, elems * h->elem_bytes()));
        if (x_dtype == h->dtype)
            CUB_(cudaMemcpyAsync(seg.payload, x, elems * h->elem_bytes(), cudaMemcpyDeviceToDevice, st));
        else if (h->dtype == RSB_DTYPE_F16)
            launch_f32_to_f16(static_cast<const float*>(x), elems, seg.payload, st);
        else
            launch_f16_to_f32(x, elems, static_cast<float*>(seg.payload), st);
    }
    CUB_(cudaPeekAtLastError());
#undef CUB_
    if (h->ivf_reserved()) {   // the rows go to their final slots now; the segment was only the encoded batch
        rc = place_segment(h, seg, st);
        cudaStreamSynchronize(st);
        free_segment(seg);
        if (rc != RSB_OK) h->next_id = next_id0;
        return rc;
    }
    h->staging.push_back(seg);
    h->n_staged += n;
    return RSB_OK;
}

extern "C" int rsb_add(rsb_index_t* h, const void* x, int x_dtype, int64_t n, const int64_t* ids, void* ws,
                       size_t ws_bytes, rsb_stream_t stream) {
    return add_impl(h, x, x_dtype, nullptr, n, ids, nullptr, ws, ws_bytes, (cudaStream_t)stream);
}
extern "C" int rsb_add_preassigned(rsb_index_t* h, const void* x, int x_dtype, int64_t n, const int64_t* ids,
                                   const int32_t* list, rsb_stream_t stream) {
    if (h && h->kind == RSB_FLAT) return fail(RSB_ERR_INVALID, "a Flat index has no lists");
    if (!list) return fail(RSB_ERR_INVALID, "list_dev is NULL");
    return add_impl(h, x, x_dtype, nullptr, n, ids, list, nullptr, 0, (cudaStream_t)stream);
}
extern "C" int rsb_add_codes(rsb_index_t* h, const uint8_t* codes, int64_t n, const int64_t* ids,
                             const int32_t* list, rsb_stream_t stream) {
    if (!h || (h->kind != RSB_IVFPQ && !is_sq8_ivf(h)))
        return fail(RSB_ERR_INVALID, "rsb_add_codes needs an IVFPQ index or an IVFFLAT index with SQ8 storage");
    if (!list || !codes) return fail(RSB_ERR_INVALID, "null argument");
    return add_impl(h, nullptr, RSB_DTYPE_F32, codes, n, ids, list, nullptr, 0, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------------------
// tiered IVFFLAT: reserve the lists, then place every added row in its final slot
// ---------------------------------------------------------------------------------------------------------
extern "C" int rsb_reserve_lists(rsb_index_t* h, const int64_t* sizes, int64_t device_rows, size_t staging_bytes,
                                 rsb_stream_t stream) {
    if (!h) return fail(RSB_ERR_INVALID, "null handle");
    if (h->kind != RSB_IVFFLAT)
        return fail(RSB_ERR_INVALID, "rsb_reserve_lists splits the lists of an IVFFLAT index (any dtype), not an %s index",
                    h->kind == RSB_IVFPQ ? "IVFPQ" : "FLAT");
    if (!sizes) return fail(RSB_ERR_INVALID, "sizes is NULL");
    if (device_rows < 0) return fail(RSB_ERR_INVALID, "device_rows must be >= 0, got %lld", (long long)device_rows);
    const int nlist = h->nlist;
    std::vector<int> len(nlist);
    std::vector<int64_t> off(nlist + 1, 0);
    for (int l = 0; l < nlist; ++l) {
        if (sizes[l] < 0) return fail(RSB_ERR_INVALID, "list %d has a negative size %lld", l, (long long)sizes[l]);
        if (sizes[l] >= ((int64_t)1 << 31) || off[l] + sizes[l] >= ((int64_t)1 << 31) - 64 * (int64_t)nlist)
            return fail(RSB_ERR_UNSUPPORTED, "more than 2^31 vectors per index shard (shard the datastore across GPUs)");
        len[l] = (int)sizes[l];
        off[l + 1] = off[l] + sizes[l];
    }
    if (!is_trained(h))
        return fail(RSB_ERR_STATE, "index is not trained (set centroids%s first)", is_sq8_ivf(h) ? " and the SQ8 range" : "");
    if (h->ivf_reserved()) return fail(RSB_ERR_STATE, "the lists are already reserved (one reservation per index)");
    if (h->ntotal || h->n_staged) return fail(RSB_ERR_STATE, "rows were already added: reserve the lists of an empty index");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t rb = h->row_bytes();
    const int64_t total = off[nlist];
    int l_dev = 0;                                  // the largest list count whose rows fit device_rows
    while (l_dev < nlist && off[l_dev + 1] <= device_rows) ++l_dev;
    const int64_t dev_rows = off[l_dev], host_rows = total - dev_rows;
    int max_len = 0, max_host = 0;
    for (int l = 0; l < nlist; ++l) {
        max_len = std::max(max_len, len[l]);
        if (l >= l_dev) max_host = std::max(max_host, len[l]);
    }
    std::vector<int> dlen(nlist), by_len(nlist), rank_of(nlist);
    for (int l = 0; l < nlist; ++l) { dlen[l] = l < l_dev ? len[l] : 0; by_len[l] = l; }
    std::stable_sort(by_len.begin(), by_len.end(), [&](int a, int b) { return len[a] > len[b]; });
    for (int i = 0; i < nlist; ++i) rank_of[by_len[i]] = i;

    auto undo = [&](int rc) {
        cudaStreamSynchronize(st);
        free_layout(h);
        free_tier(h->tier);
        return rc;
    };
#define CUR(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) return undo(fail(e__ == cudaErrorMemoryAllocation ? RSB_ERR_OOM : RSB_ERR_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__)); } while (0)
    free_layout(h);
    CUR(cudaMalloc(&h->list_len, (size_t)nlist * 4));
    CUR(cudaMalloc(&h->dev_len, (size_t)nlist * 4));
    CUR(cudaMalloc(&h->list_rank, (size_t)nlist * 4));
    CUR(cudaMalloc(&h->list_nat_off, (size_t)(nlist + 1) * 8));
    CUR(cudaMalloc(&h->list_slot_off, (size_t)(nlist + 1) * 8));
    CUR(cudaMemcpyAsync(h->list_len, len.data(), (size_t)nlist * 4, cudaMemcpyHostToDevice, st));
    CUR(cudaMemcpyAsync(h->dev_len, dlen.data(), (size_t)nlist * 4, cudaMemcpyHostToDevice, st));
    CUR(cudaMemcpyAsync(h->list_rank, rank_of.data(), (size_t)nlist * 4, cudaMemcpyHostToDevice, st));
    CUR(cudaMemcpyAsync(h->list_nat_off, off.data(), (size_t)(nlist + 1) * 8, cudaMemcpyHostToDevice, st));
    CUR(cudaMemcpyAsync(h->list_slot_off, off.data(), (size_t)(nlist + 1) * 8, cudaMemcpyHostToDevice, st));
    CUR(cudaMalloc(&h->payload, std::max<size_t>((size_t)dev_rows * rb, 256)));     // the device tier, once
    CUR(cudaMalloc(&h->ids_slots, std::max<size_t>((size_t)total * 8, 256)));
    launch_fill_i64(h->ids_slots, total, -1, st);
    CUR(cudaPeekAtLastError());
    if (host_rows) {
        h->tier.blocks.push_back(HostBlock{nullptr, dev_rows, host_rows});
        CUR(cudaHostAlloc(&h->tier.blocks[0].p, (size_t)host_rows * rb, cudaHostAllocPortable));
    }
    CUR(cudaHostAlloc((void**)&h->tier.pinned, (size_t)nlist * 13, cudaHostAllocPortable));
    if (ensure_copy_stream(h->tier) != RSB_OK) return undo(RSB_ERR_CUDA);
    CUR(cudaStreamSynchronize(st));
#undef CUR
    h->tier.dev_rows = dev_rows;
    h->tier.rows = total;
    h->tier.staging_bytes = staging_size(staging_bytes ? staging_bytes : kDefaultStagingBytes, rb, max_host, host_rows);
    h->l_dev = l_dev;
    h->ivf_len = len; h->ivf_off = off; h->ivf_fill.assign(nlist, 0);
    h->payload_bytes = (size_t)dev_rows * rb;
    h->nslots = total; h->ntotal = 0; h->max_list_len = max_len;
    return RSB_OK;
}

// rsb_search / rsb_export_* of a reserved index: every reserved row must have arrived
static int ivf_check_complete(const rsb_index* h) {
    if (h->ivf_reserved() && h->ntotal < h->nslots)
        return fail(RSB_ERR_STATE, "%lld of the %lld reserved rows have been added: add the rest first",
                    (long long)h->ntotal, (long long)h->nslots);
    return RSB_OK;
}

// One add batch of a reserved index (seg: ids, lists, rows in the storage dtype, on the device): refused whole when a
// list would overflow its reservation; else stably sorted by list (insertion order inside a list is kept), device-tier
// rows scattered to list_slot_off[l] + fill[l] + rank, host-tier rows gathered in list order and copied device to host,
// one copy per run of consecutive slots.  Synchronises st.
static int place_segment(rsb_index* h, const Segment& seg, cudaStream_t st) {
    const int64_t n = seg.n;
    const int nlist = h->nlist;
    const size_t rb = h->row_bytes();
    int* hist = nullptr;
    int32_t* sorted_list = nullptr;
    int64_t *src_idx = nullptr, *sorted_src = nullptr, *tabs = nullptr;
    uint8_t* host_stage = nullptr;
    void* cub_tmp = nullptr;
    auto cleanup = [&](int rc) {
        cudaStreamSynchronize(st);
        cudaFree(hist); cudaFree(sorted_list); cudaFree(src_idx); cudaFree(sorted_src); cudaFree(tabs);
        cudaFree(host_stage); cudaFree(cub_tmp);
        return rc;
    };
#define CUP(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) return cleanup(fail(e__ == cudaErrorMemoryAllocation ? RSB_ERR_OOM : RSB_ERR_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__)); } while (0)
    CUP(cudaMalloc(&hist, (size_t)nlist * 4));
    CUP(cudaMemsetAsync(hist, 0, (size_t)nlist * 4, st));
    launch_list_hist(seg.list, n, nlist, hist, st);
    std::vector<int> cnt(nlist);
    CUP(cudaMemcpyAsync(cnt.data(), hist, (size_t)nlist * 4, cudaMemcpyDeviceToHost, st));
    CUP(cudaStreamSynchronize(st));
    int64_t in_range = 0;
    for (int l = 0; l < nlist; ++l) in_range += cnt[l];
    if (in_range != n)
        return cleanup(fail(RSB_ERR_INVALID, "list ids out of range [0, %d): %lld of %lld rows assigned", nlist,
                            (long long)in_range, (long long)n));
    for (int l = 0; l < nlist; ++l)
        if (h->ivf_fill[l] + cnt[l] > h->ivf_len[l])
            return cleanup(fail(RSB_ERR_STATE, "the batch adds %d rows to list %d, which holds %lld of its %d reserved rows: "
                                "nothing of the batch was added", cnt[l], l, (long long)h->ivf_fill[l], h->ivf_len[l]));
    // batch_start [nlist] (first sorted row of list l in the batch), dst_base [nlist] (its slot)
    std::vector<int64_t> tab(2 * (size_t)nlist);
    int64_t acc = 0;
    for (int l = 0; l < nlist; ++l) {
        tab[l] = acc;
        tab[nlist + l] = h->ivf_off[l] + h->ivf_fill[l];
        acc += cnt[l];
    }
    const int64_t host_begin = h->l_dev < nlist ? tab[h->l_dev] : n;
    CUP(cudaMalloc(&tabs, (size_t)2 * nlist * 8));
    CUP(cudaMemcpyAsync(tabs, tab.data(), (size_t)2 * nlist * 8, cudaMemcpyHostToDevice, st));
    CUP(cudaMalloc(&sorted_list, (size_t)n * 4));
    CUP(cudaMalloc(&src_idx, (size_t)n * 8));
    CUP(cudaMalloc(&sorted_src, (size_t)n * 8));
    launch_iota_i64(src_idx, n, 0, st);
    int bits = 1;
    while ((1 << bits) < nlist) ++bits;
    size_t tmp_bytes = 0;
    CUP(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, seg.list, sorted_list, src_idx, sorted_src, n, 0, bits, st));
    CUP(cudaMalloc(&cub_tmp, tmp_bytes));
    CUP(cub::DeviceRadixSort::SortPairs(cub_tmp, tmp_bytes, seg.list, sorted_list, src_idx, sorted_src, n, 0, bits, st));
    if (n > host_begin) CUP(cudaMalloc(&host_stage, (size_t)(n - host_begin) * rb));
    launch_ivf_place_rows(sorted_list, sorted_src, n, tabs, tabs + nlist, h->l_dev, host_begin, seg.payload, seg.ids,
                          (int)rb, h->payload, host_stage, h->ids_slots, st);
    CUP(cudaPeekAtLastError());
    // host-tier rows: one device-to-host copy per run of slots that are consecutive in both buffers
    for (int l = h->l_dev; l < nlist;) {
        if (!cnt[l]) { ++l; continue; }
        const HostBlock& hb = h->tier.blocks[0];
        const int64_t s0 = tab[l] - host_begin, d0 = tab[nlist + l] - hb.r0;
        int64_t rows = cnt[l];
        int e = l + 1;
        for (; e < nlist; ++e) {
            if (!cnt[e]) continue;
            if (tab[e] - host_begin != s0 + rows || tab[nlist + e] - hb.r0 != d0 + rows) break;
            rows += cnt[e];
        }
        CUP(cudaMemcpyAsync(static_cast<uint8_t*>(hb.p) + (size_t)d0 * rb, host_stage + (size_t)s0 * rb, (size_t)rows * rb,
                            cudaMemcpyDeviceToHost, st));
        l = e;
    }
    CUP(cudaStreamSynchronize(st));
#undef CUP
    for (int l = 0; l < nlist; ++l) h->ivf_fill[l] += cnt[l];
    h->ntotal += n;
    return cleanup(RSB_OK);
}

// rows [r0, r0 + n) of a Flat or IVFFLAT index (IVFFLAT: CSR slots), from whichever tier holds them, to dst (device
// or host memory): one copy for the device rows and one per host block the range overlaps
static int tier_copy_rows(rsb_index* h, int64_t r0, int64_t n, void* dst, cudaStream_t st) {
    const size_t rb = h->row_bytes();
    uint8_t* out = static_cast<uint8_t*>(dst);
    const int64_t n_dev = h->device_rows(), r1 = r0 + n;
    if (r0 < n_dev && n > 0)
        CU(cudaMemcpyAsync(out, h->payload + (size_t)r0 * rb, (size_t)std::min(n, n_dev - r0) * rb, cudaMemcpyDefault, st));
    const std::vector<HostBlock>& blocks = h->tier.blocks;
    auto b = std::partition_point(blocks.begin(), blocks.end(), [&](const HostBlock& blk) { return blk.r0 + blk.n <= r0; });
    for (; b != blocks.end() && b->r0 < r1; ++b) {
        const int64_t a = std::max(r0, b->r0), e = std::min(r1, b->r0 + b->n);
        CU(cudaMemcpyAsync(out + (size_t)(a - r0) * rb, static_cast<const uint8_t*>(b->p) + (size_t)(a - b->r0) * rb,
                           (size_t)(e - a) * rb, cudaMemcpyDefault, st));
    }
    return RSB_OK;
}

// ---------------------------------------------------------------------------------------------------------
// finalize: staging segments (+ an existing layout) -> CSR lists / interleaved PQ blocks
// ---------------------------------------------------------------------------------------------------------
__global__ void expand_list_ids_kernel(const int64_t* __restrict__ nat_off, int nlist, int64_t n, int32_t* out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int lo = 0, hi = nlist;
        while (hi - lo > 1) {
            const int mid = (lo + hi) >> 1;
            if (nat_off[mid] <= i) lo = mid; else hi = mid;
        }
        out[i] = lo;
    }
}

static int export_impl(rsb_index* h, int64_t* offsets, void* payload, int64_t* ids, cudaStream_t st);

static int layout_to_segment(rsb_index* h, cudaStream_t st) {
    // turn the current searchable layout back into one staging segment (natural order), then drop it
    if (h->ntotal == 0) { free_layout(h); return RSB_OK; }
    Segment seg;
    seg.n = h->ntotal;
    CU(cudaMalloc(&seg.payload, (size_t)seg.n * h->row_bytes()));
    CU(cudaMalloc(&seg.ids, (size_t)seg.n * 8));
    RSB_TRY(export_impl(h, nullptr, seg.payload, seg.ids, st));
    if (h->kind != RSB_FLAT) {
        CU(cudaMalloc(&seg.list, (size_t)seg.n * 4));
        expand_list_ids_kernel<<<4096, 256, 0, st>>>(h->list_nat_off, h->nlist, seg.n, seg.list);
        CHECK_LAUNCH();
    }
    CU(cudaStreamSynchronize(st));
    free_layout(h);
    h->staging.insert(h->staging.begin(), seg);
    h->n_staged += seg.n;
    return RSB_OK;
}

// tiered Flat: the rows are already in place; only the staged ids are appended to the id array
static int finalize_tiered(rsb_index* h, cudaStream_t st) {
    const int64_t n = h->ntotal + h->n_staged;
    int64_t* ids = nullptr;
    CU(cudaMalloc(&ids, (size_t)n * 8));
    cudaError_t e = h->ntotal ? cudaMemcpyAsync(ids, h->ids_slots, (size_t)h->ntotal * 8, cudaMemcpyDeviceToDevice, st)
                              : cudaSuccess;
    int64_t o = h->ntotal;
    for (const Segment& s : h->staging) {
        if (e == cudaSuccess) e = cudaMemcpyAsync(ids + o, s.ids, (size_t)s.n * 8, cudaMemcpyDeviceToDevice, st);
        o += s.n;
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) {
        cudaFree(ids);
        return fail(RSB_ERR_CUDA, "tiered finalize: %s", cudaGetErrorString(e));
    }
    for (auto& s : h->staging) free_segment(s);
    h->staging.clear(); h->n_staged = 0;
    cudaFree(h->ids_slots);
    h->ids_slots = ids;
    h->ntotal = n; h->nslots = n; h->max_list_len = (int)std::min<int64_t>(n, 0x7fffffff);
    return RSB_OK;
}

extern "C" int rsb_finalize(rsb_index_t* h, rsb_stream_t stream) {
    if (!h) return fail(RSB_ERR_INVALID, "null handle");
    cudaStream_t st = (cudaStream_t)stream;
    if (h->staging.empty()) return RSB_OK;
    if (h->tiered()) return finalize_tiered(h, st);
    if (h->ntotal > 0) RSB_TRY(layout_to_segment(h, st));
    else free_layout(h);
    const int64_t n = h->n_staged;
    const int nseg = (int)h->staging.size();
    const size_t rb = h->row_bytes();

    std::vector<int64_t> starts(nseg + 1, 0);
    for (int s = 0; s < nseg; ++s) starts[s + 1] = starts[s] + h->staging[s].n;

    if (h->kind == RSB_FLAT) {
        uint8_t* payload = nullptr;
        int64_t* ids = nullptr;
        if (nseg == 1) {  // adopt
            payload = static_cast<uint8_t*>(h->staging[0].payload);
            ids = h->staging[0].ids;
            h->staging[0].payload = nullptr; h->staging[0].ids = nullptr;
        } else {
            CU(cudaMalloc(&payload, (size_t)n * rb));
            CU(cudaMalloc(&ids, (size_t)n * 8));
            for (int s = 0; s < nseg; ++s) {
                CU(cudaMemcpyAsync(payload + (size_t)starts[s] * rb, h->staging[s].payload, (size_t)h->staging[s].n * rb, cudaMemcpyDeviceToDevice, st));
                CU(cudaMemcpyAsync(ids + starts[s], h->staging[s].ids, (size_t)h->staging[s].n * 8, cudaMemcpyDeviceToDevice, st));
            }
        }
        CU(cudaStreamSynchronize(st));
        for (auto& s : h->staging) free_segment(s);
        h->staging.clear(); h->n_staged = 0;
        h->payload = payload; h->payload_bytes = (size_t)n * rb; h->ids_slots = ids;
        h->ntotal = n; h->nslots = n; h->max_list_len = (int)std::min<int64_t>(n, 0x7fffffff);
        // tensor-core scoring needs the rows split into tf32 hi/lo parts (2x the fp32 footprint): only below 8 GB.
        // fp16 rows are the tensor-core operand as stored: no split copy at any size.
        if (h->dtype == RSB_DTYPE_F32 && h->flat_tensor && (h->d % 32 == 0) && n > 0 && (size_t)n * rb <= ((size_t)8 << 30) && tf32_path_available()) {
            if (cudaMalloc(&h->flat_hi, (size_t)n * rb) == cudaSuccess && cudaMalloc(&h->flat_lo, (size_t)n * rb) == cudaSuccess) {
                launch_split_tf32(reinterpret_cast<const float*>(payload), (size_t)n * h->d, h->flat_hi, h->flat_lo, st);
                CU(cudaStreamSynchronize(st));
            } else {
                cudaFree(h->flat_hi); cudaFree(h->flat_lo);
                h->flat_hi = nullptr; h->flat_lo = nullptr;
                cudaGetLastError();
            }
        }
        return RSB_OK;
    }

    // ---- IVF: sort (list, source row) pairs by list (stable radix sort keeps insertion order inside a list)
    int32_t *list_all = nullptr, *sorted_list = nullptr;
    int64_t *src_idx = nullptr, *sorted_src = nullptr, *dst_row = nullptr;
    void* cub_tmp = nullptr;
    int* hist = nullptr;
    const uint8_t** seg_payload_dev = nullptr;
    const int64_t** seg_ids_dev = nullptr;
    int64_t* seg_starts_dev = nullptr;
    auto cleanup = [&]() {
        cudaFree(list_all); cudaFree(sorted_list); cudaFree(src_idx); cudaFree(sorted_src); cudaFree(dst_row);
        cudaFree(cub_tmp); cudaFree(hist); cudaFree((void*)seg_payload_dev); cudaFree((void*)seg_ids_dev);
        cudaFree(seg_starts_dev);
    };
#define CUF(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) { cleanup(); return fail(e__ == cudaErrorMemoryAllocation ? RSB_ERR_OOM : RSB_ERR_CUDA, "%s: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); } } while (0)
    CUF(cudaMalloc(&list_all, (size_t)n * 4));
    CUF(cudaMalloc(&sorted_list, (size_t)n * 4));
    CUF(cudaMalloc(&src_idx, (size_t)n * 8));
    CUF(cudaMalloc(&sorted_src, (size_t)n * 8));
    for (int s = 0; s < nseg; ++s)
        CUF(cudaMemcpyAsync(list_all + starts[s], h->staging[s].list, (size_t)h->staging[s].n * 4, cudaMemcpyDeviceToDevice, st));
    launch_iota_i64(src_idx, n, 0, st);
    int bits = 1;
    while ((1 << bits) < h->nlist) ++bits;
    size_t tmp_bytes = 0;
    CUF(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, list_all, sorted_list, src_idx, sorted_src, (int64_t)n, 0, bits, st));
    CUF(cudaMalloc(&cub_tmp, tmp_bytes));
    CUF(cub::DeviceRadixSort::SortPairs(cub_tmp, tmp_bytes, list_all, sorted_list, src_idx, sorted_src, (int64_t)n, 0, bits, st));

    CUF(cudaMalloc(&hist, (size_t)h->nlist * 4));
    CUF(cudaMemsetAsync(hist, 0, (size_t)h->nlist * 4, st));
    launch_list_hist(list_all, n, h->nlist, hist, st);
    std::vector<int> len(h->nlist);
    CUF(cudaMemcpyAsync(len.data(), hist, (size_t)h->nlist * 4, cudaMemcpyDeviceToHost, st));
    CUF(cudaStreamSynchronize(st));

    std::vector<int64_t> nat(h->nlist + 1, 0), slot(h->nlist + 1, 0);
    int max_len = 0;
    const bool pq = h->kind == RSB_IVFPQ;
    for (int l = 0; l < h->nlist; ++l) {
        nat[l + 1] = nat[l] + len[l];
        slot[l + 1] = slot[l] + (pq ? (int64_t)((len[l] + 31) / 32 * 32) : (int64_t)len[l]);
        max_len = std::max(max_len, len[l]);
    }
    if (nat[h->nlist] != n) { cleanup(); return fail(RSB_ERR_INVALID, "list ids out of range [0, %d): %lld of %lld rows assigned", h->nlist, (long long)nat[h->nlist], (long long)n); }
    const int64_t nslots = slot[h->nlist];

    CUF(cudaMalloc(&h->list_len, (size_t)h->nlist * 4));
    CUF(cudaMalloc(&h->list_nat_off, (size_t)(h->nlist + 1) * 8));
    CUF(cudaMalloc(&h->list_slot_off, (size_t)(h->nlist + 1) * 8));
    CUF(cudaMemcpyAsync(h->list_len, len.data(), (size_t)h->nlist * 4, cudaMemcpyHostToDevice, st));
    {
        // work-list order: longest lists first (longest-processing-time scheduling of the persistent scan blocks)
        std::vector<int> by_len(h->nlist), rank_of(h->nlist);
        for (int l = 0; l < h->nlist; ++l) by_len[l] = l;
        std::stable_sort(by_len.begin(), by_len.end(), [&](int a, int b) { return len[a] > len[b]; });
        for (int i = 0; i < h->nlist; ++i) rank_of[by_len[i]] = i;
        CUF(cudaMalloc(&h->list_rank, (size_t)h->nlist * 4));
        CUF(cudaMemcpy(h->list_rank, rank_of.data(), (size_t)h->nlist * 4, cudaMemcpyHostToDevice));
    }
    CUF(cudaMemcpyAsync(h->list_nat_off, nat.data(), (size_t)(h->nlist + 1) * 8, cudaMemcpyHostToDevice, st));
    CUF(cudaMemcpyAsync(h->list_slot_off, slot.data(), (size_t)(h->nlist + 1) * 8, cudaMemcpyHostToDevice, st));

    h->payload_bytes = std::max<size_t>((size_t)nslots * rb, 256);
    CUF(cudaMalloc(&h->payload, h->payload_bytes));
    CUF(cudaMalloc(&h->ids_slots, std::max<size_t>((size_t)nslots * 8, 256)));
    if (pq) CUF(cudaMemsetAsync(h->payload, 0, h->payload_bytes, st));
    launch_fill_i64(h->ids_slots, nslots, -1, st);

    std::vector<const uint8_t*> sp(nseg);
    std::vector<const int64_t*> si(nseg);
    for (int s = 0; s < nseg; ++s) { sp[s] = static_cast<const uint8_t*>(h->staging[s].payload); si[s] = h->staging[s].ids; }
    CUF(cudaMalloc((void**)&seg_payload_dev, (size_t)nseg * 8));
    CUF(cudaMalloc((void**)&seg_ids_dev, (size_t)nseg * 8));
    CUF(cudaMalloc(&seg_starts_dev, (size_t)(nseg + 1) * 8));
    CUF(cudaMemcpyAsync((void*)seg_payload_dev, sp.data(), (size_t)nseg * 8, cudaMemcpyHostToDevice, st));
    CUF(cudaMemcpyAsync((void*)seg_ids_dev, si.data(), (size_t)nseg * 8, cudaMemcpyHostToDevice, st));
    CUF(cudaMemcpyAsync(seg_starts_dev, starts.data(), (size_t)(nseg + 1) * 8, cudaMemcpyHostToDevice, st));

    if (pq) {
        CUF(cudaMalloc(&dst_row, (size_t)n * 8));
        launch_slot_of_sorted(sorted_list, n, h->list_nat_off, h->list_slot_off, dst_row, st);
        if (pq_interleaved_layout(h->Mb))
            launch_pq_interleave(seg_payload_dev, seg_starts_dev, nseg, sorted_src, sorted_list, n, h->list_nat_off,
                                 h->list_slot_off, h->Mb, h->payload, st);
        else   // generic M: natural [slot][Mb] rows
            launch_gather_rows(seg_payload_dev, seg_starts_dev, nseg, sorted_src, dst_row, n, (int)rb, h->payload, st);
        launch_gather_ids(seg_ids_dev, seg_starts_dev, nseg, sorted_src, dst_row, n, h->ids_slots, st);
    } else {
        launch_gather_rows(seg_payload_dev, seg_starts_dev, nseg, sorted_src, nullptr, n, (int)rb, h->payload, st);
        launch_gather_ids(seg_ids_dev, seg_starts_dev, nseg, sorted_src, nullptr, n, h->ids_slots, st);
    }
    CUF(cudaPeekAtLastError());
    CUF(cudaStreamSynchronize(st));
#undef CUF
    cleanup();
    for (auto& s : h->staging) free_segment(s);
    h->staging.clear(); h->n_staged = 0;
    h->ntotal = n; h->nslots = nslots; h->max_list_len = max_len;
    return RSB_OK;
}

// ---------------------------------------------------------------------------------------------------------
// introspection / export
// ---------------------------------------------------------------------------------------------------------
extern "C" int rsb_info(rsb_index_t* h, int what, int64_t* out) {
    if (!h || !out) return fail(RSB_ERR_INVALID, "null argument");
    switch (what) {
        case RSB_INFO_KIND: *out = h->kind; break;
        case RSB_INFO_D: *out = h->d; break;
        case RSB_INFO_NLIST: *out = h->kind == RSB_FLAT ? 0 : h->nlist; break;
        case RSB_INFO_M: *out = h->M; break;
        case RSB_INFO_NBITS: *out = h->nbits; break;
        case RSB_INFO_NTOTAL: *out = h->ntotal + h->n_staged; break;
        case RSB_INFO_IS_TRAINED: *out = is_trained(h) ? 1 : 0; break;
        case RSB_INFO_MAX_LIST_LEN: *out = h->max_list_len; break;
        case RSB_INFO_INDEX_BYTES: *out = (int64_t)(h->payload_bytes + (size_t)h->nslots * 8); break;
        case RSB_INFO_DTYPE: *out = h->dtype; break;
        case RSB_INFO_BY_RESIDUAL: *out = h->by_residual ? 1 : 0; break;
        case RSB_INFO_HOST_BYTES: *out = h->host_rows() * (int64_t)h->row_bytes(); break;
        case RSB_INFO_DEVICE_ROWS: *out = h->device_rows(); break;
        default: return fail(RSB_ERR_INVALID, "unknown info key %d", what);
    }
    return RSB_OK;
}

__global__ void widen_i32_kernel(const int* __restrict__ src, int n, int64_t* __restrict__ dst) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) dst[i] = src[i];
}

extern "C" int rsb_list_sizes(rsb_index_t* h, int64_t* sizes, rsb_stream_t stream) {
    if (!h || !sizes) return fail(RSB_ERR_INVALID, "null argument");
    if (h->kind == RSB_FLAT) return fail(RSB_ERR_INVALID, "a Flat index has no lists");
    cudaStream_t st = (cudaStream_t)stream;
    if (!h->staging.empty()) RSB_TRY(rsb_finalize(h, stream));
    if (!h->list_len) { CU(cudaMemsetAsync(sizes, 0, (size_t)h->nlist * 8, st)); return RSB_OK; }
    widen_i32_kernel<<<(h->nlist + 255) / 256, 256, 0, st>>>(h->list_len, h->nlist, sizes);
    CHECK_LAUNCH();
    return RSB_OK;
}

static int export_impl(rsb_index* h, int64_t* offsets, void* payload, int64_t* ids, cudaStream_t st) {
    if (h->kind == RSB_FLAT) {
        if (offsets) {
            const int64_t o[2] = {0, h->ntotal};
            CU(cudaMemcpyAsync(offsets, o, 16, cudaMemcpyHostToDevice, st));
            CU(cudaStreamSynchronize(st));
        }
    } else if (!h->list_nat_off) {
        if (offsets) CU(cudaMemsetAsync(offsets, 0, (size_t)(h->nlist + 1) * 8, st));
        return RSB_OK;
    } else if (offsets) {
        CU(cudaMemcpyAsync(offsets, h->list_nat_off, (size_t)(h->nlist + 1) * 8, cudaMemcpyDeviceToDevice, st));
    }
    if (h->ntotal == 0) return RSB_OK;
    if (h->kind == RSB_IVFPQ) {
        if (payload && pq_interleaved_layout(h->Mb))
            launch_pq_deinterleave(h->payload, h->list_nat_off, h->list_slot_off, h->list_len, h->nlist, h->Mb, static_cast<uint8_t*>(payload), st);
        else if (payload)
            launch_compact_slots_rows(h->payload, h->list_nat_off, h->list_slot_off, h->nlist, h->Mb, static_cast<uint8_t*>(payload), st);
        if (ids) launch_compact_slots_i64(h->ids_slots, h->list_nat_off, h->list_slot_off, h->list_len, h->nlist, ids, st);
        CHECK_LAUNCH();
        return RSB_OK;
    }
    // Flat and IVFFLAT slots are the natural order; rows from either tier, to device or host memory
    if (payload) RSB_TRY(tier_copy_rows(h, 0, h->ntotal, payload, st));
    if (ids) CU(cudaMemcpyAsync(ids, h->ids_slots, (size_t)h->ntotal * 8, cudaMemcpyDefault, st));
    return RSB_OK;
}

extern "C" int rsb_export_lists(rsb_index_t* h, int64_t* offsets, void* payload, int64_t* ids, rsb_stream_t stream) {
    if (!h) return fail(RSB_ERR_INVALID, "null handle");
    if (!h->staging.empty()) RSB_TRY(rsb_finalize(h, stream));
    RSB_TRY(ivf_check_complete(h));
    return export_impl(h, offsets, payload, ids, (cudaStream_t)stream);
}

extern "C" int rsb_export_rows(rsb_index_t* h, int64_t r0, int64_t n, void* dst, rsb_stream_t stream) {
    if (!h) return fail(RSB_ERR_INVALID, "null handle");
    if (h->kind == RSB_IVFPQ)
        return fail(RSB_ERR_INVALID, "rsb_export_rows reads the rows of a Flat or IVFFLAT index, not IVFPQ codes");
    if (!h->staging.empty()) RSB_TRY(rsb_finalize(h, stream));
    RSB_TRY(ivf_check_complete(h));
    if (r0 < 0 || n < 0 || r0 + n > h->ntotal)
        return fail(RSB_ERR_INVALID, "rows [%lld, %lld) are outside [0, %lld)", (long long)r0, (long long)(r0 + n),
                    (long long)h->ntotal);
    if (n == 0) return RSB_OK;
    if (!dst) return fail(RSB_ERR_INVALID, "dst is NULL");
    return tier_copy_rows(h, r0, n, dst, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------------------
// search
// ---------------------------------------------------------------------------------------------------------
// IVF-PQ with the interleaved layout scans two queries of a list per item (rsb_ivf.cu).  RSB_PQ_SINGLE_ITEMS=1
// (read once) scans every (query, list) pair on its own: the reference the tests compare the paired scan against.
static bool pq_paired_scan(const rsb_index* h) {
    static const bool single = getenv("RSB_PQ_SINGLE_ITEMS") != nullptr;
    return h->kind == RSB_IVFPQ && pq_interleaved_layout(h->Mb) && !single;
}

struct SearchPlan {
    int qb, nprobe;          // queries per batch, effective nprobe
    int kc;                  // candidates taken from the tensor-core coarse scan before the exact re-score
    KnnPlan coarse;
    size_t off_coarse_ws, off_cD, off_cI, off_pair, off_lut, off_qlut, off_quant, off_keys, off_cnt, off_tau, off_qsplit,
        off_cD2, off_cI2, total;
};
static SearchPlan search_plan(const rsb_index* h, int nq, int k, int nprobe) {
    SearchPlan p;
    p.nprobe = std::max(1, std::min(nprobe, h->nlist));
    int qb = std::max(1, std::min(nq, 16384));
    const size_t per_q = (size_t)p.nprobe * k * 8;
    const size_t cap = (size_t)2 << 30;
    if (per_q * qb > cap) qb = (int)std::max<size_t>(1, cap / per_q);
    p.qb = qb;
    p.kc = std::min(h->nlist, p.nprobe + 8);
    p.coarse = knn_plan(qb, h->nlist, p.kc);
    size_t o = 0;
    p.off_coarse_ws = o; o += align_up(p.coarse.total);
    p.off_cD = o;        o += align_up((size_t)qb * p.nprobe * 4);
    p.off_cI = o;        o += align_up((size_t)qb * p.nprobe * 8);
    p.off_pair = o;      o += align_up(pair_work_bytes(qb, p.nprobe, h->nlist));
    const size_t lut_words = pq_interleaved_layout(h->Mb) ? (size_t)kLutWords : (size_t)h->Mb * 256;
    p.off_lut = o;       o += h->kind == RSB_IVFPQ ? align_up((size_t)qb * lut_words * 4) : 0;
    const bool paired = pq_paired_scan(h);
    p.off_qlut = o;      o += paired ? align_up((size_t)qb * kLutWords * 2) : 0;
    p.off_quant = o;     o += paired ? align_up((size_t)qb * sizeof(PQQuant)) : 0;
    p.off_keys = o;      o += align_up((size_t)qb * p.nprobe * k * 8);
    p.off_cnt = o;       o += align_up((size_t)qb * p.nprobe * 4);
    p.off_tau = o;       o += align_up((size_t)qb * 4);
    p.off_qsplit = o;    o += align_up((size_t)2 * qb * h->d * 4);
    p.off_cD2 = o;       o += align_up((size_t)qb * p.kc * 4);
    p.off_cI2 = o;       o += align_up((size_t)qb * p.kc * 8);
    p.total = o;
    return p;
}

struct FlatPlan {
    bool tensor;
    int kc;
    KnnPlan knn;
    size_t off_qsplit, off_D2, off_I2, total;
};
static FlatPlan flat_plan(const rsb_index* h, int nq, int k) {
    FlatPlan p;
    const int64_t n = std::max<int64_t>(h->ntotal + h->n_staged, 1);
    if (h->dtype == RSB_DTYPE_F16) {
        // always the tensor-core scorer; k + 8 candidates, at most 4096 (the select / re-score limit)
        p.tensor = true;
        p.kc = (int)std::min<int64_t>(n, std::min(k + 8, 4096));
    } else {
        p.tensor = h->flat_tensor && h->flat_hi && h->flat_lo && h->n_staged == 0 && (h->d % 32 == 0) && k + 8 <= 4096 &&
                   tf32_path_available();
        p.kc = p.tensor ? (int)std::min<int64_t>(n, (int64_t)k + 8) : k;
    }
    p.knn = knn_plan(nq, n, p.kc);
    size_t o = align_up(p.knn.total);
    p.off_qsplit = o; o += p.tensor ? align_up((size_t)2 * p.knn.qb * h->d * 4) : 0;
    p.off_D2 = o;     o += p.tensor ? align_up((size_t)p.knn.qb * p.kc * 4) : 0;
    p.off_I2 = o;     o += p.tensor ? align_up((size_t)p.knn.qb * p.kc * 8) : 0;
    p.total = o;
    return p;
}

// The staging pipeline of both tiered searches: host chunk c is copied by the tier's copy stream into staging buffer
// c % 2 while the caller's stream scores chunk c - 1.  Per query batch the caller runs begin, prefetch, then
// acquire / score / release for every chunk; end joins the copy stream back to the caller's stream after the last
// batch.  `copy(c, buf)` enqueues chunk c's copies into buf on tier.copy_st.
struct StagePipe {
    HostTier& t;
    uint8_t* buf[2];
    std::function<int(int64_t, uint8_t*)> copy;
    int64_t nchunks = 0;

    uint8_t* buffer(int64_t c) const { return buf[c & 1]; }
    // copies of this batch start after everything enqueued on st before (adds, the previous batch's use of the buffers)
    int begin(cudaStream_t st) {
        CU(cudaEventRecord(t.copy_start, st));
        CU(cudaStreamWaitEvent(t.copy_st, t.copy_start, 0));
        return RSB_OK;
    }
    int fill(int64_t c) {
        RSB_TRY(copy(c, buffer(c)));
        CU(cudaEventRecord(t.stage_ready[c & 1], t.copy_st));
        return RSB_OK;
    }
    int prefetch(int64_t n) {
        nchunks = n;
        for (int64_t c = 0; c < std::min<int64_t>(2, n); ++c) RSB_TRY(fill(c));
        return RSB_OK;
    }
    int acquire(int64_t c, cudaStream_t st) {
        CU(cudaStreamWaitEvent(st, t.stage_ready[c & 1], 0));
        return RSB_OK;
    }
    // chunk c's buffer is free once st has scored it: it takes chunk c + 2
    int release(int64_t c, cudaStream_t st) {
        CU(cudaEventRecord(t.stage_free[c & 1], st));
        if (c + 2 < nchunks) {
            CU(cudaStreamWaitEvent(t.copy_st, t.stage_free[c & 1], 0));
            RSB_TRY(fill(c + 2));
        }
        return RSB_OK;
    }
    int end(cudaStream_t st) {
        CU(cudaEventRecord(t.copy_done, t.copy_st));
        CU(cudaStreamWaitEvent(st, t.copy_done, 0));
        return RSB_OK;
    }
};
// two staging buffers of `bytes` each from workspace offset o; returns the offset after them
static size_t plan_staging(size_t o, size_t bytes, size_t off_stage[2]) {
    for (int b = 0; b < 2; ++b) {
        off_stage[b] = o;
        o += align_up(bytes);
    }
    return o;
}

// Tiered Flat search (rows past dev_rows in host memory).  The rows are scored in pieces: the device tier in place,
// then the host tier in chunks of chunk_rows, staged by StagePipe while the previous piece is scored.  Each piece
// runs the fp16 candidate path (kc = min(k + 8, 4096, rows) candidates) and the exact fp32 re-score of its own rows,
// and is merged into the running top-k (ties: the earlier piece, i.e. the lower row).
struct TieredFlatPlan {
    int qb, kc;
    int64_t n_dev, chunk_rows, nchunks;
    size_t knn_bytes, off_qsplit, off_D2, off_I2, off_mD, off_mI, off_stage[2], total;
};
static TieredFlatPlan tiered_flat_plan(const rsb_index* h, int nq, int k) {
    TieredFlatPlan p;
    const size_t rb = h->row_bytes();
    p.n_dev = h->device_rows();
    const int64_t n_host = h->host_rows();
    p.chunk_rows = (int64_t)(staging_size(h->tier.staging_bytes, rb, 1, n_host) / rb);
    p.nchunks = (n_host + p.chunk_rows - 1) / p.chunk_rows;
    p.kc = std::min(k + 8, 4096);
    const int64_t rows = std::max<int64_t>({p.n_dev, p.chunk_rows, 1});
    const KnnPlan kp = knn_plan(nq, rows, p.kc);
    p.qb = kp.qb;
    p.knn_bytes = kp.total;
    if (nq % p.qb) p.knn_bytes = std::max(p.knn_bytes, knn_plan(nq % p.qb, rows, p.kc).total);   // the last batch
    size_t o = align_up(p.knn_bytes);
    p.off_qsplit = o; o += align_up((size_t)2 * p.qb * h->d * 4);
    p.off_D2 = o;     o += align_up((size_t)p.qb * p.kc * 4);
    p.off_I2 = o;     o += align_up((size_t)p.qb * p.kc * 8);
    p.off_mD = o;     o += align_up((size_t)2 * p.qb * k * 4);   // merge input [2, nb, k]: running top-k, new piece
    p.off_mI = o;     o += align_up((size_t)2 * p.qb * k * 8);
    p.total = plan_staging(o, (size_t)p.chunk_rows * rb, p.off_stage);
    return p;
}

static int search_flat_tiered(rsb_index* h, const float* q, int nq, int k, float* D, int64_t* I, void* ws,
                              size_t ws_bytes, cudaStream_t st) {
    const TieredFlatPlan p = tiered_flat_plan(h, nq, k);
    if (ws_bytes < p.total) return fail(RSB_ERR_OOM, "workspace too small: need %zu bytes, got %zu", p.total, ws_bytes);
    unsigned char* w = static_cast<unsigned char*>(ws);
    TensorOperands tc;   // [qb, d] fp16 hi, [qb, d] fp16 lo, [qb] fp32 inverse scales
    tc.xh = tc.xl = nullptr;
    tc.f16 = true;
    tc.qh = reinterpret_cast<float*>(w + p.off_qsplit);
    tc.ql = reinterpret_cast<float*>(reinterpret_cast<uint16_t*>(tc.qh) + (size_t)p.qb * h->d);
    tc.qinv = reinterpret_cast<float*>(reinterpret_cast<uint16_t*>(tc.qh) + (size_t)2 * p.qb * h->d);
    float* D2 = reinterpret_cast<float*>(w + p.off_D2);
    int64_t* I2 = reinterpret_cast<int64_t*>(w + p.off_I2);
    float* mD = reinterpret_cast<float*>(w + p.off_mD);
    int64_t* mI = reinterpret_cast<int64_t*>(w + p.off_mI);
    StagePipe pipe{h->tier, {w + p.off_stage[0], w + p.off_stage[1]}, [&](int64_t c, uint8_t* buf) -> int {
        const int64_t r0 = p.n_dev + c * p.chunk_rows;
        return tier_copy_rows(h, r0, std::min(p.chunk_rows, h->ntotal - r0), buf, h->tier.copy_st);
    }};

    // rows X [rows, d] = index rows [r0, r0 + rows) -> exact top-k of nb queries
    auto score_piece = [&](const float* qb, int nb, const void* X, int64_t rows, int64_t r0, float* Do, int64_t* Io) -> int {
        const int kc = (int)std::min<int64_t>(rows, p.kc);
        RSB_TRY(knn_ip_device(h, qb, nb, X, rows, h->d, kc, nullptr, 0, D2, I2, w, p.knn_bytes, st, &tc));
        if (launch_refine_exact(qb, nb, X, 2, h->d, I2, kc, k, Do, Io, h->ids_slots + r0, st) != 0)
            return fail(RSB_ERR_UNSUPPORTED, "k = %d is too large for the re-score kernel", k);
        h->launches += 1;
        return RSB_OK;
    };
    const int64_t pieces = (p.n_dev > 0 ? 1 : 0) + p.nchunks;
    for (int q0 = 0; q0 < nq; q0 += p.qb) {
        const int nb = std::min(p.qb, nq - q0);
        const float* qb = q + (size_t)q0 * h->d;
        float* Dq = D + (size_t)q0 * k;
        int64_t* Iq = I + (size_t)q0 * k;
        int64_t done = 0;
        // piece `done` writes the final result (a single piece), the running slot (first piece) or the new-piece slot
        auto outD = [&]() { return pieces == 1 ? Dq : mD + (done ? (size_t)nb * k : 0); };
        auto outI = [&]() { return pieces == 1 ? Iq : mI + (done ? (size_t)nb * k : 0); };
        auto merge = [&]() -> int {
            if (done++ == 0) return RSB_OK;
            if (launch_merge_shards(mD, mI, 2, nb, k, k, Dq, Iq, st) != 0)
                return fail(RSB_ERR_UNSUPPORTED, "k = %d is too large for the merge kernel", k);
            h->launches += 1;
            if (done < pieces) {   // the merged top-k is the running slot of the next merge
                CU(cudaMemcpyAsync(mD, Dq, (size_t)nb * k * 4, cudaMemcpyDeviceToDevice, st));
                CU(cudaMemcpyAsync(mI, Iq, (size_t)nb * k * 8, cudaMemcpyDeviceToDevice, st));
            }
            return RSB_OK;
        };
        RSB_TRY(pipe.begin(st));
        RSB_TRY(pipe.prefetch(p.nchunks));
        if (p.n_dev > 0) {   // the device tier, in place, while the first chunks cross PCIe
            RSB_TRY(score_piece(qb, nb, h->payload, p.n_dev, 0, outD(), outI()));
            RSB_TRY(merge());
        }
        for (int64_t c = 0; c < p.nchunks; ++c) {
            const int64_t r0 = p.n_dev + c * p.chunk_rows;
            RSB_TRY(pipe.acquire(c, st));
            RSB_TRY(score_piece(qb, nb, pipe.buffer(c), std::min(p.chunk_rows, h->ntotal - r0), r0, outD(), outI()));
            RSB_TRY(pipe.release(c, st));
            RSB_TRY(merge());
        }
    }
    RSB_TRY(pipe.end(st));
    CHECK_LAUNCH();
    return RSB_OK;
}

// Tiered IVFFLAT search (lists past l_dev in host memory): the search plan's workspace, then the probed-list flags
// [nlist], one piece's masked list_len [nlist] int32 and staging offsets [nlist] int64, the per-batch table (stage_off
// [nlist] int64, chunk_of [nlist] int32) and two staging buffers of tier.staging_bytes.
struct IvfTierPlan {
    size_t off_flags, off_plen, off_pdata, off_table, off_stage[2], total;
};
static IvfTierPlan ivf_tier_plan(const rsb_index* h, size_t base) {
    IvfTierPlan t;
    size_t o = align_up(base);
    t.off_flags = o; o += align_up((size_t)h->nlist);
    t.off_plen = o;  o += align_up((size_t)h->nlist * 4);
    t.off_pdata = o; o += align_up((size_t)h->nlist * 8);
    t.off_table = o; o += align_up((size_t)h->nlist * 12);
    t.total = plan_staging(o, h->tier.staging_bytes, t.off_stage);
    return t;
}

extern "C" size_t rsb_workspace_bytes(rsb_index_t* h, int nq, int k, int nprobe) {
    if (!h) return 0;
    nq = std::max(nq, 1); k = std::max(k, 1);
    if (h->kind == RSB_FLAT && h->host_rows() > 0) return tiered_flat_plan(h, nq, k).total;
    if (h->kind == RSB_FLAT) {
        // pending adds are finalised by the search itself, which may switch the tensor path on: size for both
        const size_t plain = knn_plan(nq, std::max<int64_t>(h->ntotal + h->n_staged, 1), k).total;
        const int kc = std::min(k + 8, 4096);
        const KnnPlan kp = knn_plan(nq, std::max<int64_t>(h->ntotal + h->n_staged, 1), kc);
        const size_t tens = align_up(kp.total) + align_up((size_t)2 * kp.qb * h->d * 4) + align_up((size_t)kp.qb * kc * 4) +
                            align_up((size_t)kp.qb * kc * 8);
        return std::max(plain, tens);
    }
    if (h->host_rows() > 0) return ivf_tier_plan(h, search_plan(h, nq, k, nprobe).total).total;
    return search_plan(h, nq, k, nprobe).total;
}

static int coarse_impl(rsb_index* h, const float* q, int nq, const SearchPlan& p, unsigned char* w, cudaStream_t st) {
    float* cD = reinterpret_cast<float*>(w + p.off_cD);
    int64_t* cI = reinterpret_cast<int64_t*>(w + p.off_cI);
    TensorOperands tc;
    const bool use_tc = h->coarse_tensor && h->cent_hi && h->cent_lo && (h->d % 32 == 0) && tf32_path_available();
    if (use_tc) {
        // [qb, d] fp16 hi, [qb, d] fp16 lo, [qb] fp32 inverse scales
        tc.xh = h->cent_hi; tc.xl = h->cent_lo; tc.xinv = h->cent_inv;
        tc.qh = reinterpret_cast<float*>(w + p.off_qsplit);
        tc.ql = reinterpret_cast<float*>(reinterpret_cast<uint16_t*>(tc.qh) + (size_t)p.qb * h->d);
        tc.qinv = reinterpret_cast<float*>(reinterpret_cast<uint16_t*>(tc.qh) + (size_t)2 * p.qb * h->d);
    }
    if (!use_tc)
        return knn_ip_device(h, q, nq, h->centroids, h->nlist, h->d, p.nprobe, nullptr, 0, cD, cI, w + p.off_coarse_ws,
                             p.coarse.total, st, nullptr);
    // tensor-core candidates (nprobe + 8), then exact fp32 re-score -> top-nprobe (fp32-exact ids and scores)
    float* cD2 = reinterpret_cast<float*>(w + p.off_cD2);
    int64_t* cI2 = reinterpret_cast<int64_t*>(w + p.off_cI2);
    RSB_TRY(knn_ip_device(h, q, nq, h->centroids, h->nlist, h->d, p.kc, nullptr, 0, cD2, cI2, w + p.off_coarse_ws,
                          p.coarse.total, st, &tc));
    if (launch_refine_exact(q, nq, h->centroids, 4, h->d, cI2, p.kc, p.nprobe, cD, cI, nullptr, st) != 0)
        return fail(RSB_ERR_UNSUPPORTED, "nprobe = %d is too large for the coarse re-score kernel", p.nprobe);
    h->launches += 1;
    CHECK_LAUNCH();
    return RSB_OK;
}

static size_t assign_workspace_bytes(const rsb_index* h, int64_t n) {
    const int rows = (int)std::min<int64_t>(std::max<int64_t>(n, 1), kAssignRows);
    return search_plan(h, rows, 1, 1).total + 256;
}
// rows x[0, n) get lists list_out[r_begin + i]
static int assign_lists(rsb_index* h, const float* x, int64_t n, int32_t* list_out, void* ws, size_t ws_bytes, cudaStream_t st,
                        int64_t r_begin) {
    const int rows = (int)std::min<int64_t>(std::max<int64_t>(n, 1), kAssignRows);
    const SearchPlan p = search_plan(h, rows, 1, 1);
    if (ws_bytes < p.total) return fail(RSB_ERR_OOM, "add workspace too small: need %zu, got %zu", p.total, ws_bytes);
    unsigned char* w = static_cast<unsigned char*>(ws);
    for (int64_t r0 = 0; r0 < n; r0 += p.qb) {
        const int nb = (int)std::min<int64_t>(p.qb, n - r0);
        RSB_TRY(coarse_impl(h, x + (size_t)r0 * h->d, nb, p, w, st));
        launch_i64_to_i32(reinterpret_cast<const int64_t*>(w + p.off_cI), nb, list_out + r_begin + r0, st);
    }
    CHECK_LAUNCH();
    return RSB_OK;
}

extern "C" int rsb_coarse(rsb_index_t* h, const float* q, int nq, int nprobe, int64_t* list_out, float* score_out,
                          void* ws, size_t ws_bytes, rsb_stream_t stream) {
    if (!h || !q || !list_out) return fail(RSB_ERR_INVALID, "null argument");
    if (h->kind == RSB_FLAT) return fail(RSB_ERR_INVALID, "a Flat index has no coarse quantizer");
    if (!h->has_centroids) return fail(RSB_ERR_STATE, "index has no centroids");
    if (nprobe <= 0 || nprobe > h->nlist) return fail(RSB_ERR_INVALID, "nprobe must be in [1, nlist]");
    cudaStream_t st = (cudaStream_t)stream;
    const SearchPlan p = search_plan(h, nq, 1, nprobe);
    if (ws_bytes < p.total) return fail(RSB_ERR_OOM, "workspace too small: need %zu bytes, got %zu", p.total, ws_bytes);
    unsigned char* w = static_cast<unsigned char*>(ws);
    for (int q0 = 0; q0 < nq; q0 += p.qb) {
        const int nb = std::min(p.qb, nq - q0);
        RSB_TRY(coarse_impl(h, q + (size_t)q0 * h->d, nb, p, w, st));
        CU(cudaMemcpyAsync(list_out + (size_t)q0 * nprobe, w + p.off_cI, (size_t)nb * nprobe * 8, cudaMemcpyDeviceToDevice, st));
        if (score_out) CU(cudaMemcpyAsync(score_out + (size_t)q0 * nprobe, w + p.off_cD, (size_t)nb * nprobe * 4, cudaMemcpyDeviceToDevice, st));
    }
    return RSB_OK;
}

struct SharedTau {
    unsigned* local = nullptr;            // this GPU's threshold array [nq] (symmetric memory, zeroed by the caller)
    unsigned* const* peers = nullptr;     // device array of npeers base pointers (one per GPU, own entry included)
    int npeers = 0;
};

// The IVFPQ look-up tables for queries q [nq, d], as the scan reads them (Mb byte sub-quantizers).  The search and
// the rsb_pq_tables diagnostic both build them here, so the tables a test reads are the ones the scan reads.
static void launch_pq_tables(const rsb_index* h, const float* q, int nq, float* lut, cudaStream_t st) {
    if (h->nbits == 4) launch_pq_lut4(q, nq, h->d, h->M, h->codebook, lut, st);
    else if (pq_interleaved_layout(h->M)) launch_pq_lut(q, nq, h->d, h->M, h->codebook_t, lut, st);
    else launch_pq_lut_generic(q, nq, h->d, h->M, h->codebook, lut, st);
}

// Tiered IVFFLAT search, per query batch:
//   1. the coarse step (or the caller's lists), then the probed host lists are flagged on the device and the [nlist]
//      flags copied to page-locked memory;
//   2. the device lists are scanned in place (list_len masked to lists [0, l_dev)), enqueued before the host waits;
//   3. the host waits for the flags -- the one host synchronisation per batch, by design: only the host can drive the
//      copy engine -- and packs the probed host lists, in list order, into chunks of at most one staging buffer
//      (adjacent lists coalesced into one copy).  StagePipe copies chunk c into staging buffer c % 2 while the caller's
//      stream scans chunk c - 1, as in search_flat_tiered; a small kernel derives each chunk's masked list_len and
//      staging offsets from one per-batch table, copied by copy_st ahead of the chunks;
//   4. every piece shares the batch's thresholds tau and writes disjoint (query, probe) slots of out_keys / out_cnt,
//      so one merge_items gives the result, as in the all-device search.
// The pinned flags / table are rewritten only after the host has waited for this batch's flags, which the caller's
// stream orders after every use of them by the previous batch.
static int search_ivf_tiered(rsb_index* h, const float* q, int nq, int k, const SearchPlan& p, const IvfTierPlan& t,
                             const int64_t* pre_lists, const float* pre_dis, float* D, int64_t* I, unsigned char* w,
                             cudaStream_t st) {
    const int nlist = h->nlist;
    const size_t rb = h->row_bytes();
    const int64_t stage_rows = (int64_t)(h->tier.staging_bytes / rb);
    unsigned char* dflags = w + t.off_flags;
    int* plen = reinterpret_cast<int*>(w + t.off_plen);
    int64_t* pdata = reinterpret_cast<int64_t*>(w + t.off_pdata);
    int64_t* dtab = reinterpret_cast<int64_t*>(w + t.off_table);
    int64_t* stage_off = reinterpret_cast<int64_t*>(h->tier.pinned);
    int* chunk_of = reinterpret_cast<int*>(stage_off + nlist);
    unsigned char* hflags = h->tier.pinned + (size_t)nlist * 12;
    struct Run { int64_t chunk, slot, stage_row, rows; };
    std::vector<Run> runs;
    StagePipe pipe{h->tier, {w + t.off_stage[0], w + t.off_stage[1]}, [&](int64_t c, uint8_t* buf) -> int {
        for (const Run& r : runs)
            if (r.chunk == c) RSB_TRY(tier_copy_rows(h, r.slot, r.rows, buf + (size_t)r.stage_row * rb, h->tier.copy_st));
        return RSB_OK;
    }};
    for (int q0 = 0; q0 < nq; q0 += p.qb) {
        const int nb = std::min(p.qb, nq - q0);
        const float* qb = q + (size_t)q0 * h->d;
        if (pre_lists) {
            CU(cudaMemcpyAsync(w + p.off_cI, pre_lists + (size_t)q0 * p.nprobe, (size_t)nb * p.nprobe * 8, cudaMemcpyDeviceToDevice, st));
            CU(cudaMemcpyAsync(w + p.off_cD, pre_dis + (size_t)q0 * p.nprobe, (size_t)nb * p.nprobe * 4, cudaMemcpyDeviceToDevice, st));
        } else {
            RSB_TRY(coarse_impl(h, qb, nb, p, w, st));
        }
        const int64_t* cI = reinterpret_cast<const int64_t*>(w + p.off_cI);
        ScanArgs a;
        a.coarse_ids = cI; a.coarse_scores = reinterpret_cast<const float*>(w + p.off_cD); a.nprobe = p.nprobe;
        a.list_off = h->list_slot_off;
        a.tau = reinterpret_cast<unsigned*>(w + p.off_tau);
        a.tau_peers = nullptr; a.n_peers = 0; a.tau_external = 0;
        a.k = k;
        a.out_keys = reinterpret_cast<u64*>(w + p.off_keys);
        a.out_cnt = reinterpret_cast<int*>(w + p.off_cnt);
        a.dbg_flag = reinterpret_cast<unsigned*>(h->prof_dev + 2);
        a.items = nullptr; a.qlut = nullptr; a.quant = nullptr; a.rescored = nullptr;
        // the pieces of this batch share tau and out_cnt: zeroed once, here
        CU(cudaMemsetAsync(a.tau, 0, (size_t)nb * 4, st));
        CU(cudaMemsetAsync(a.out_cnt, 0, (size_t)nb * p.nprobe * 4, st));
        launch_ivf_probed_flags(cI, nb * p.nprobe, nlist, h->l_dev, h->list_len, dflags, st);
        CU(cudaMemcpyAsync(hflags, dflags, (size_t)nlist, cudaMemcpyDeviceToHost, st));
        CU(cudaEventRecord(h->tier.flags_ready, st));
        RSB_TRY(pipe.begin(st));
        static const bool lpt_env = getenv("RSB_LIST_ORDER_LPT") != nullptr;
        const bool lpt_order = lpt_env || ((long)nb * p.nprobe < 64L * 3 * device_num_sms());
        PairWork pw = carve_pair_work(w + p.off_pair, nb, p.nprobe, nlist);
        a.order = pw.order; a.n_items = pw.n_items; a.item_counter = pw.item_counter; a.n_pairs = pw.n_pairs;
        auto scan_piece = [&](const int* len, const void* vecs, const int64_t* data) {
            launch_pair_setup(cI, nb, p.nprobe, nlist, len, lpt_order ? h->list_rank : nullptr, pw, st, 0, false);
            a.list_len = len;
            launch_ivfflat_scan(a, qb, vecs, data, h->elem_bytes(), h->d, nb, st, h->sq, h->by_residual);
            h->launches += 4;
        };
        if (h->tier.dev_rows > 0) scan_piece(h->dev_len, h->payload, h->list_slot_off);   // the device lists, in place
        CU(cudaEventSynchronize(h->tier.flags_ready));
        runs.clear();
        int nchunks = 0;
        int64_t used = stage_rows;
        for (int l = 0; l < nlist; ++l) { chunk_of[l] = -1; stage_off[l] = 0; }
        for (int l = h->l_dev; l < nlist; ++l) {
            if (!hflags[l]) continue;
            const int64_t len = h->ivf_len[l], slot = h->ivf_off[l];
            if (used + len > stage_rows) { ++nchunks; used = 0; }
            chunk_of[l] = nchunks - 1;
            stage_off[l] = used;
            Run* last = runs.empty() ? nullptr : &runs.back();
            if (last && last->chunk == nchunks - 1 && last->slot + last->rows == slot) last->rows += len;
            else runs.push_back(Run{nchunks - 1, slot, used, len});
            used += len;
        }
        if (nchunks > 0) {
            // on the copy stream, ahead of the chunks: an H2D on `st` would queue behind the device-piece scan and
            // hold up the chunk copies behind it on the copy engine.  st reads it after waiting for stage_ready.
            CU(cudaMemcpyAsync(dtab, stage_off, (size_t)nlist * 12, cudaMemcpyHostToDevice, h->tier.copy_st));
            RSB_TRY(pipe.prefetch(nchunks));
            for (int c = 0; c < nchunks; ++c) {
                RSB_TRY(pipe.acquire(c, st));
                launch_ivf_piece_tables(h->list_len, dtab, reinterpret_cast<const int*>(dtab + nlist), nlist, c, plen,
                                        pdata, st);
                scan_piece(plen, pipe.buffer(c), pdata);
                RSB_TRY(pipe.release(c, st));
            }
        }
        launch_merge_items(a.out_keys, a.out_cnt, nb, p.nprobe, k, k, h->ids_slots, 0, D + (size_t)q0 * k,
                           I + (size_t)q0 * k, st);
        h->launches += 3;
        CHECK_LAUNCH();
    }
    return pipe.end(st);
}

// shared: the multi-GPU threshold exchange, or nullptr for thresholds kept in the workspace
static int search_impl(rsb_index_t* h, const float* q, int nq, int k, int nprobe, const int64_t* pre_lists,
                       const float* pre_dis, float* D, int64_t* I, void* ws, size_t ws_bytes, rsb_stream_t stream,
                       const SharedTau* shared = nullptr) {
    if (!h) return fail(RSB_ERR_INVALID, "null handle");
    if (nq < 0 || k <= 0) return fail(RSB_ERR_INVALID, "bad nq = %d / k = %d", nq, k);
    if (k > 4096) return fail(RSB_ERR_UNSUPPORTED, "k = %d > 4096 is not supported", k);
    if (nq == 0) return RSB_OK;
    if (!q || !D || !I) return fail(RSB_ERR_INVALID, "null argument");
    if (!is_trained(h)) return fail(RSB_ERR_STATE, "index is not trained");
    cudaStream_t st = (cudaStream_t)stream;
    if (!h->staging.empty()) RSB_TRY(rsb_finalize(h, stream));
    h->launches = 0;
    h->ev = h->evs[h->ev_done % rsb_index::kProfSets];

    if (h->kind == RSB_FLAT) {
        if (h->prof) CU(cudaEventRecord(h->ev[0], st));
        const FlatPlan fp = flat_plan(h, nq, k);
        if (h->host_rows() > 0) {
            RSB_TRY(search_flat_tiered(h, q, nq, k, D, I, ws, ws_bytes, st));
        } else if (fp.tensor && h->ntotal > 0) {
            // tensor-core candidates (k + 8 per query; 3xTF32 on wgmma, or the scaled fp16 query split against fp16
            // rows), then exact fp32 re-score -> top-k
            if (ws_bytes < fp.total) return fail(RSB_ERR_OOM, "workspace too small: need %zu bytes, got %zu", fp.total, ws_bytes);
            unsigned char* w = static_cast<unsigned char*>(ws);
            TensorOperands tc;
            tc.xh = h->flat_hi; tc.xl = h->flat_lo;
            tc.qh = reinterpret_cast<float*>(w + fp.off_qsplit);
            tc.ql = tc.qh + (size_t)fp.knn.qb * h->d;
            if (h->dtype == RSB_DTYPE_F16) {   // [qb, d] fp16 hi, [qb, d] fp16 lo, [qb] fp32 inverse scales
                tc.f16 = true;
                tc.ql = reinterpret_cast<float*>(reinterpret_cast<uint16_t*>(tc.qh) + (size_t)fp.knn.qb * h->d);
                tc.qinv = reinterpret_cast<float*>(reinterpret_cast<uint16_t*>(tc.qh) + (size_t)2 * fp.knn.qb * h->d);
            }
            float* D2 = reinterpret_cast<float*>(w + fp.off_D2);
            int64_t* I2 = reinterpret_cast<int64_t*>(w + fp.off_I2);
            for (int q0 = 0; q0 < nq; q0 += fp.knn.qb) {
                const int nb = std::min(fp.knn.qb, nq - q0);
                const float* qb = q + (size_t)q0 * h->d;
                RSB_TRY(knn_ip_device(h, qb, nb, h->payload, h->ntotal, h->d, fp.kc, nullptr, 0, D2, I2, w, fp.knn.total, st, &tc));
                if (launch_refine_exact(qb, nb, h->payload, h->elem_bytes(), h->d, I2, fp.kc, k, D + (size_t)q0 * k,
                                        I + (size_t)q0 * k, h->ids_slots, st) != 0)
                    return fail(RSB_ERR_UNSUPPORTED, "k = %d is too large for the re-score kernel", k);
                h->launches += 1;
            }
            CHECK_LAUNCH();
        } else {
            // fp32 rows on CUDA cores (or an empty index of either dtype: all padding, no row is read)
            RSB_TRY(knn_ip_device(h, q, nq, h->payload, h->ntotal, h->d, k, h->ids_slots, 0,
                                  D, I, ws, ws_bytes, st));
        }
        if (h->prof) {
            for (int i = 1; i < 6; ++i) CU(cudaEventRecord(h->ev[i], st));
            h->ev_done++;
        }
        return RSB_OK;
    }

    if (nprobe <= 0) return fail(RSB_ERR_INVALID, "nprobe must be > 0, got %d", nprobe);
    RSB_TRY(ivf_check_complete(h));
    if (h->ivf_reserved() && shared)
        return fail(RSB_ERR_UNSUPPORTED, "shared thresholds (a multi-GPU partition) are not implemented for an IVFFLAT "
                                         "index with reserved, tiered lists");
    const SearchPlan p = search_plan(h, nq, k, nprobe);
    if (ws_bytes < p.total) return fail(RSB_ERR_OOM, "workspace too small: need %zu bytes, got %zu", p.total, ws_bytes);
    unsigned char* w = static_cast<unsigned char*>(ws);

    if (h->ntotal == 0) {  // empty index: all padding
        launch_merge_items(nullptr, nullptr, 0, 0, k, k, nullptr, 0, D, I, st);
        std::vector<float> dpad((size_t)nq * k, -3.402823466e+38f);
        std::vector<int64_t> ipad((size_t)nq * k, -1);
        CU(cudaMemcpyAsync(D, dpad.data(), dpad.size() * 4, cudaMemcpyHostToDevice, st));
        CU(cudaMemcpyAsync(I, ipad.data(), ipad.size() * 8, cudaMemcpyHostToDevice, st));
        CU(cudaStreamSynchronize(st));
        return RSB_OK;
    }
    if (h->host_rows() > 0) {
        const IvfTierPlan t = ivf_tier_plan(h, p.total);
        if (pre_lists && p.nprobe != nprobe)
            return fail(RSB_ERR_INVALID, "preassigned nprobe %d exceeds nlist %d", nprobe, h->nlist);
        if (ws_bytes < t.total) return fail(RSB_ERR_OOM, "workspace too small: need %zu bytes, got %zu", t.total, ws_bytes);
        if (h->prof) CU(cudaEventRecord(h->ev[0], st));
        RSB_TRY(search_ivf_tiered(h, q, nq, k, p, t, pre_lists, pre_dis, D, I, w, st));
        if (h->prof) {
            for (int i = 1; i < 6; ++i) CU(cudaEventRecord(h->ev[i], st));
            h->ev_done++;
        }
        return RSB_OK;
    }

    for (int q0 = 0; q0 < nq; q0 += p.qb) {
        const int nb = std::min(p.qb, nq - q0);
        const float* qb = q + (size_t)q0 * h->d;
        const bool prof = h->prof && (q0 + p.qb >= nq);  // time the last batch
        if (prof) CU(cudaEventRecord(h->ev[0], st));
        if (pre_lists) {
            // faiss search_preassigned: the caller supplies the probed lists and their coarse scores
            if (p.nprobe != nprobe) return fail(RSB_ERR_INVALID, "preassigned nprobe %d exceeds nlist %d", nprobe, h->nlist);
            CU(cudaMemcpyAsync(w + p.off_cI, pre_lists + (size_t)q0 * nprobe, (size_t)nb * nprobe * 8, cudaMemcpyDeviceToDevice, st));
            CU(cudaMemcpyAsync(w + p.off_cD, pre_dis + (size_t)q0 * nprobe, (size_t)nb * nprobe * 4, cudaMemcpyDeviceToDevice, st));
        } else {
            RSB_TRY(coarse_impl(h, qb, nb, p, w, st));
        }
        if (prof) CU(cudaEventRecord(h->ev[1], st));

        PairWork pw = carve_pair_work(w + p.off_pair, nb, p.nprobe, h->nlist);
        const int64_t* cI = reinterpret_cast<const int64_t*>(w + p.off_cI);
        const float* cD = reinterpret_cast<const float*>(w + p.off_cD);
        // Large batches visit the lists in id order; when a persistent block only gets a few dozen items (small
        // batches, the full-sweep micro-benchmark) the lists are visited longest-first so that the blocks finish on
        // short items (longest-first helps the full sweep but slows large batches, hence the threshold).
        // RSB_LIST_ORDER_LPT=1 forces longest-first.
        static const bool lpt_env = getenv("RSB_LIST_ORDER_LPT") != nullptr;
        const bool lpt_order = lpt_env || ((long)nb * p.nprobe < 64L * 3 * device_num_sms());
        // Thresholds shared between GPUs: ONE lead pair per query job-wide -- only the GPU that holds the query's rank-0 list
        // leads it, the others get their first bound for that query over NVLink (see pair_bin): fewer cold top-k
        // selections per GPU.  RSB_LOCAL_LEADS=1: a lead pair per query on every GPU (its best-ranked list that is
        // non-empty there), the single-GPU rule.
        static const bool local_leads = getenv("RSB_LOCAL_LEADS") != nullptr;
        const int lead_mode = (shared && shared->npeers > 1 && !local_leads) ? 1 : 0;
        const bool paired = pq_paired_scan(h) && nb > 1;          // one query: no list is probed twice
        launch_pair_setup(cI, nb, p.nprobe, h->nlist, h->list_len, lpt_order ? h->list_rank : nullptr, pw, st, lead_mode,
                          paired);
        h->launches += paired ? 5 : 3;
        if (prof) CU(cudaEventRecord(h->ev[2], st));

        ScanArgs a;
        a.coarse_ids = cI; a.coarse_scores = cD; a.nprobe = p.nprobe;
        a.order = pw.order; a.n_items = pw.n_items; a.item_counter = pw.item_counter;
        a.list_len = h->list_len; a.list_off = h->list_slot_off;
        a.tau = reinterpret_cast<unsigned*>(w + p.off_tau);
        a.tau_peers = nullptr; a.n_peers = 0; a.tau_external = 0;
        if (shared) {
            if (nq > p.qb) return fail(RSB_ERR_UNSUPPORTED, "shared thresholds need the whole batch in one pass (nq = %d > %d)", nq, p.qb);
            a.tau = shared->local; a.tau_peers = shared->peers; a.n_peers = shared->npeers; a.tau_external = 1;
        }
        a.k = k;
        a.out_keys = reinterpret_cast<u64*>(w + p.off_keys);
        a.out_cnt = reinterpret_cast<int*>(w + p.off_cnt);
        a.dbg_flag = reinterpret_cast<unsigned*>(h->prof_dev + 2);
        a.items = paired ? pw.items : nullptr;
        a.n_pairs = pw.n_pairs;
        a.qlut = paired ? reinterpret_cast<const unsigned short*>(w + p.off_qlut) : nullptr;
        a.quant = paired ? reinterpret_cast<const PQQuant*>(w + p.off_quant) : nullptr;
        a.rescored = prof ? h->prof_dev + 3 : nullptr;
        if (prof) CU(cudaMemsetAsync(h->prof_dev + 3, 0, 8, st));

        if (h->kind == RSB_IVFPQ) {
            float* lut = reinterpret_cast<float*>(w + p.off_lut);
            // from here on the index is scanned as Mb byte sub-quantizers (Mb = M for 8-bit codes)
            launch_pq_tables(h, qb, nb, lut, st);
            h->launches += 1;
            if (paired) {
                launch_pq_lut_quant(lut, nb, h->Mb, reinterpret_cast<unsigned short*>(w + p.off_qlut),
                                    reinterpret_cast<PQQuant*>(w + p.off_quant), st);
                h->launches += 1;
            }
            if (prof) CU(cudaEventRecord(h->ev[3], st));
            if (launch_ivfpq_scan(a, lut, h->payload, h->Mb, nb, st) != 0)
                return fail(RSB_ERR_UNSUPPORTED, "no scan kernel for %d code bytes per vector", h->Mb);
        } else {
            if (prof) CU(cudaEventRecord(h->ev[3], st));
            if (!a.tau_external) CU(cudaMemsetAsync(a.tau, 0, (size_t)nb * 4, st));
            CU(cudaMemsetAsync(a.out_cnt, 0, (size_t)nb * p.nprobe * 4, st));
            launch_ivfflat_scan(a, qb, h->payload, h->list_slot_off, h->elem_bytes(), h->d, nb, st, h->sq, h->by_residual);
        }
        h->launches += paired ? 2 : 1;                 // paired work list: both scan variants, one returns at once
        if (prof) CU(cudaEventRecord(h->ev[4], st));
        launch_merge_items(a.out_keys, a.out_cnt, nb, p.nprobe, k, k, h->ids_slots, 0, D + (size_t)q0 * k,
                           I + (size_t)q0 * k, st);
        h->launches += 1;
        if (prof) {
            CU(cudaEventRecord(h->ev[5], st));
            CU(cudaMemcpyAsync(h->prof_dev, pw.scan_bytes, 8, cudaMemcpyDeviceToDevice, st));
            CU(cudaMemcpyAsync(h->prof_dev + 1, pw.n_pairs, 4, cudaMemcpyDeviceToDevice, st));
            h->ev_done++;
        }
        CHECK_LAUNCH();
    }
    return RSB_OK;
}

extern "C" int rsb_search(rsb_index_t* h, const float* q, int nq, int k, int nprobe, float* D, int64_t* I, void* ws,
                          size_t ws_bytes, rsb_stream_t stream) {
    return search_impl(h, q, nq, k, nprobe, nullptr, nullptr, D, I, ws, ws_bytes, stream);
}
extern "C" int rsb_search_preassigned(rsb_index_t* h, const float* q, int nq, int k, int nprobe,
                                      const int64_t* list_dev, const float* coarse_dis_dev, float* D, int64_t* I,
                                      void* ws, size_t ws_bytes, uint32_t* tau_local_dev,
                                      uint32_t* const* tau_peers_dev, int npeers, rsb_stream_t stream) {
    if (h && h->kind == RSB_FLAT) return fail(RSB_ERR_INVALID, "a Flat index has no lists");
    if (!list_dev || !coarse_dis_dev) return fail(RSB_ERR_INVALID, "null argument");
    if (npeers < 0 || (npeers > 0 && !tau_peers_dev) || (!tau_local_dev && (npeers != 0 || tau_peers_dev)))
        return fail(RSB_ERR_INVALID, "inconsistent threshold arrays: tau_local_dev %s, tau_peers_dev %s, npeers = %d",
                    tau_local_dev ? "set" : "NULL", tau_peers_dev ? "set" : "NULL", npeers);
    SharedTau sh;
    sh.local = tau_local_dev; sh.peers = tau_peers_dev; sh.npeers = npeers;
    return search_impl(h, q, nq, k, nprobe, list_dev, coarse_dis_dev, D, I, ws, ws_bytes, stream,
                       tau_local_dev ? &sh : nullptr);
}

// ---- exact re-ranking (faiss IndexRefine::search) -----------------------------------------------------------
// The store [ntotal, d] in fp32, fp16 or SQ8 codes: rows [0, n_dev) in device memory, rows [n_dev, ntotal) in mapped
// page-locked host memory (n_dev < ntotal: the tiered store).
extern "C" int rsb_host_alloc(size_t bytes, void** out) {
    if (!out) return fail(RSB_ERR_INVALID, "out is NULL");
    *out = nullptr;
    if (bytes == 0) return RSB_OK;
    CU(cudaHostAlloc(out, bytes, cudaHostAllocPortable | cudaHostAllocMapped));
    return RSB_OK;
}

extern "C" int rsb_host_free(void* p) {
    if (p) CU(cudaFreeHost(p));
    return RSB_OK;
}

static bool misaligned16(const void* p) { return reinterpret_cast<uintptr_t>(p) & 15; }

// The checks of the store that need no pointer (the workspace queries run these alone); *s gets its shape.
static int store_shape(RefineStore* s, int store_dtype, int64_t n_dev, int64_t ntotal, int d, int k_base, int k,
                       size_t staging_bytes) {
    if (store_dtype != RSB_DTYPE_F32 && store_dtype != RSB_DTYPE_F16 && store_dtype != RSB_DTYPE_SQ8)
        return fail(RSB_ERR_INVALID, "store_dtype must be RSB_DTYPE_F32, RSB_DTYPE_F16 or RSB_DTYPE_SQ8, got %d", store_dtype);
    if (n_dev < 0 || n_dev > ntotal)
        return fail(RSB_ERR_INVALID, "n_dev = %lld must be in [0, ntotal = %lld]", (long long)n_dev, (long long)ntotal);
    if (k <= 0 || k_base < k) return fail(RSB_ERR_INVALID, "need 0 < k <= k_base, got k = %d, k_base = %d", k, k_base);
    if (k_base > 4096) return fail(RSB_ERR_UNSUPPORTED, "k_base = k * k_factor = %d > 4096 is not supported", k_base);
    if (ntotal > ((int64_t)1 << 31)) return fail(RSB_ERR_INVALID, "store rows must be in [0, 2^31], got %lld", (long long)ntotal);
    if (d <= 0 || d % 8) return fail(RSB_ERR_INVALID, "d = %d must be a positive multiple of 8 for the re-rank store", d);
    const bool sq8 = store_dtype == RSB_DTYPE_SQ8;
    if (sq8 && d % 16) return fail(RSB_ERR_INVALID, "d = %d must be a multiple of 16 for an SQ8 store (whole 16-byte rows)", d);
    const int eb = sq8 ? 1 : store_dtype == RSB_DTYPE_F16 ? 2 : 4;
    const size_t per_q = (size_t)k_base * d * eb;
    if (n_dev < ntotal && staging_bytes < per_q)
        return fail(RSB_ERR_INVALID, "staging_bytes = %zu is below one query's worst case (k_base * d * elem = %zu)",
                    staging_bytes, per_q);
    *s = RefineStore{nullptr, n_dev, nullptr, eb, d, ntotal, nullptr};
    return RSB_OK;
}

// Every check of the store that needs no CUDA call; *s gets the store, its host tier as the caller's pointer until
// map_host_tier replaces it by the device alias.
static int refine_store(RefineStore* s, const void* store_dev, int64_t n_dev, const void* store_host, int store_dtype,
                        const float* sq, int d, int64_t ntotal, int k_base, int k, size_t staging_bytes) {
    RSB_TRY(store_shape(s, store_dtype, n_dev, ntotal, d, k_base, k, staging_bytes));
    if (n_dev > 0 && (!store_dev || misaligned16(store_dev)))
        return fail(RSB_ERR_INVALID, "the re-rank store must be a 16-byte aligned device pointer");
    if (n_dev < ntotal && (!store_host || misaligned16(store_host)))
        return fail(RSB_ERR_INVALID, "the host tier must be a 16-byte aligned page-locked host pointer");
    if (store_dtype == RSB_DTYPE_SQ8 && (!sq || misaligned16(sq)))
        return fail(RSB_ERR_INVALID, "the SQ8 range sq_dev [2, d] must be a 16-byte aligned device pointer");
    s->dev = store_dev;
    s->host = n_dev < ntotal ? store_host : nullptr;
    s->sq = store_dtype == RSB_DTYPE_SQ8 ? sq : nullptr;
    return RSB_OK;
}

// A tiered store's host tier must be page-locked and mapped: both ends are checked, and s->host becomes the device
// alias the kernels read it through.  Pageable memory and device memory are refused.
static int map_host_tier(RefineStore* s) {
    if (s->n_dev == s->ntotal) return RSB_OK;
    const size_t bytes = (size_t)(s->ntotal - s->n_dev) * s->d * s->elem_bytes;
    const unsigned char* p[2] = {static_cast<const unsigned char*>(s->host), static_cast<const unsigned char*>(s->host) + bytes - 1};
    void* dp[2] = {nullptr, nullptr};
    for (int i = 0; i < 2; ++i) {
        cudaPointerAttributes a{};
        if (cudaPointerGetAttributes(&a, p[i]) != cudaSuccess || a.type != cudaMemoryTypeHost) {
            cudaGetLastError();
            return fail(RSB_ERR_INVALID, "the host tier is not page-locked host memory (rsb_host_alloc / cudaHostAlloc)");
        }
        if (cudaHostGetDevicePointer(&dp[i], const_cast<unsigned char*>(p[i]), 0) != cudaSuccess) {
            cudaGetLastError();
            return fail(RSB_ERR_INVALID, "the host tier is not mapped into the device address space (cudaHostAllocMapped)");
        }
    }
    if (static_cast<unsigned char*>(dp[1]) != static_cast<unsigned char*>(dp[0]) + bytes - 1)
        return fail(RSB_ERR_INVALID, "the host tier is not one mapped allocation");
    s->host = dp[0];
    return RSB_OK;
}

// Workspace of one re-rank of nq queries: the plain kernel's for an all-device store, the tiered plan of the store's
// element size otherwise (0: the tiered plan could not be sized).
static size_t refine_ws(const RefineStore& s, int nq, int k_base, int k, size_t staging_bytes) {
    if (s.n_dev == s.ntotal) return refine_plan(nq, k_base, k).ws_bytes;
    const TieredPlan p = tiered_plan(nq, k_base, k, s.d, s.elem_bytes, staging_bytes);
    return p.qc ? p.total : 0;
}

// Validated: the re-rank of nq queries, by the plain kernel (all-device store) or the tiered launcher.
static int refine_batch(const RefineStore& s, const float* q, int nq, const int64_t* cand, int k_base, int k, float* D,
                        int64_t* I, void* ws, size_t ws_bytes, size_t staging_bytes, int64_t* host_rows, cudaStream_t st) {
    const size_t need = refine_ws(s, nq, k_base, k, staging_bytes);
    if (ws_bytes < need) return fail(RSB_ERR_OOM, "workspace too small: need %zu bytes, got %zu", need, ws_bytes);
    if (s.n_dev == s.ntotal) {
        if (launch_refine_rows(refine_plan(nq, k_base, k), q, nq, s, cand, k_base, k, D, I, ws, st) != 0)
            return fail(RSB_ERR_UNSUPPORTED, "d = %d with k_base = %d needs more shared memory than the re-rank kernel has",
                        s.d, k_base);
        CHECK_LAUNCH();
        return RSB_OK;
    }
    const TieredPlan p = tiered_plan(nq, k_base, k, s.d, s.elem_bytes, staging_bytes);
    if (!p.qc) return fail(RSB_ERR_CUDA, "could not size the tiered re-rank workspace: %s", cudaGetErrorString(cudaGetLastError()));
    if (!p.smem_ok)
        return fail(RSB_ERR_UNSUPPORTED, "d = %d with k_base = %d needs more shared memory than the re-rank kernel has", s.d, k_base);
    const cudaError_t e = launch_refine_tiered(p, q, nq, s, cand, k_base, k, D, I, ws, reinterpret_cast<long long*>(host_rows), st);
    if (e != cudaSuccess) return fail(RSB_ERR_CUDA, "tiered re-rank: %s", cudaGetErrorString(e));
    return RSB_OK;
}

extern "C" size_t rsb_refine_workspace_bytes(int nq, int k_base, int k, int d, int store_dtype, int64_t n_dev,
                                             int64_t ntotal, size_t staging_bytes) {
    RefineStore s;
    if (nq <= 0 || store_shape(&s, store_dtype, n_dev, ntotal, d, k_base, k, staging_bytes) != RSB_OK) return 0;
    return refine_ws(s, nq, k_base, k, staging_bytes);
}

extern "C" int rsb_refine(const float* q, int nq, const void* store_dev, int64_t n_dev, const void* store_host,
                          int store_dtype, const float* sq, int d, int64_t ntotal, const int64_t* cand, int k_base, int k,
                          float* D, int64_t* I, void* ws, size_t ws_bytes, size_t staging_bytes, int64_t* host_rows,
                          rsb_stream_t stream) {
    RefineStore s;
    RSB_TRY(refine_store(&s, store_dev, n_dev, store_host, store_dtype, sq, d, ntotal, k_base, k, staging_bytes));
    if (nq < 0) return fail(RSB_ERR_INVALID, "bad nq = %d", nq);
    if (nq == 0) return RSB_OK;
    if (!q || !cand || !D || !I) return fail(RSB_ERR_INVALID, "null argument");
    RSB_TRY(map_host_tier(&s));
    return refine_batch(s, q, nq, cand, k_base, k, D, I, ws, ws_bytes, staging_bytes, host_rows, (cudaStream_t)stream);
}

// Queries are processed in batches of qb: base search at k_base into [qb, k_base] candidate buffers, then the re-rank.
struct SearchRefinePlan {
    int qb;
    size_t search_ws, off_D, off_I, off_ref, total;
};
static SearchRefinePlan search_refine_plan(rsb_index* h, const RefineStore& s, int nq, int k, int k_base, int nprobe,
                                           size_t staging_bytes) {
    SearchRefinePlan p;
    nq = std::max(nq, 1);
    p.qb = std::min(nq, 16384);
    const int last = nq % p.qb ? nq % p.qb : p.qb;     // the last batch may split its queries into more chunks
    p.search_ws = align_up(rsb_workspace_bytes(h, p.qb, k_base, nprobe));
    p.off_D = p.search_ws;
    p.off_I = p.off_D + align_up((size_t)p.qb * k_base * 4);
    p.off_ref = p.off_I + align_up((size_t)p.qb * k_base * 8);
    p.total = p.off_ref + align_up(std::max(refine_ws(s, p.qb, k_base, k, staging_bytes),
                                            refine_ws(s, last, k_base, k, staging_bytes)));
    return p;
}

extern "C" size_t rsb_search_refine_workspace_bytes(rsb_index_t* h, int nq, int k, int k_factor, int nprobe,
                                                    int store_dtype, int64_t n_dev, int64_t ntotal,
                                                    size_t staging_bytes) {
    if (!h || k <= 0 || k_factor <= 0 || (int64_t)k * k_factor > 4096) return 0;
    RefineStore s;
    if (store_shape(&s, store_dtype, n_dev, ntotal, h->d, k * k_factor, k, staging_bytes) != RSB_OK) return 0;
    return search_refine_plan(h, s, nq, k, k * k_factor, nprobe, staging_bytes).total;
}

extern "C" int rsb_search_refine(rsb_index_t* h, const float* q, int nq, int k, int k_factor, int nprobe,
                                 const void* store_dev, int64_t n_dev, const void* store_host, int store_dtype,
                                 const float* sq, int64_t ntotal, float* D, int64_t* I, void* ws, size_t ws_bytes,
                                 size_t staging_bytes, int64_t* host_rows, rsb_stream_t stream) {
    if (!h) return fail(RSB_ERR_INVALID, "null handle");
    if (h->kind != RSB_IVFPQ) return fail(RSB_ERR_INVALID, "re-ranking is for IVFPQ indexes: Flat / IVFFlat scores are already exact");
    if (k <= 0 || k_factor <= 0) return fail(RSB_ERR_INVALID, "bad k = %d / k_factor = %d", k, k_factor);
    if ((int64_t)k * k_factor > 4096) return fail(RSB_ERR_UNSUPPORTED, "k * k_factor = %lld > 4096 is not supported", (long long)k * k_factor);
    const int k_base = k * k_factor;
    RefineStore s;
    RSB_TRY(refine_store(&s, store_dev, n_dev, store_host, store_dtype, sq, h->d, ntotal, k_base, k, staging_bytes));
    if (ntotal != h->ntotal + h->n_staged)
        return fail(RSB_ERR_INVALID, "the re-rank store has %lld rows, the index holds %lld vectors", (long long)ntotal,
                    (long long)(h->ntotal + h->n_staged));
    if (nq < 0) return fail(RSB_ERR_INVALID, "bad nq = %d", nq);
    if (nq == 0) return RSB_OK;
    if (!q || !D || !I) return fail(RSB_ERR_INVALID, "null argument");
    RSB_TRY(map_host_tier(&s));
    const SearchRefinePlan p = search_refine_plan(h, s, nq, k, k_base, nprobe, staging_bytes);
    if (ws_bytes < p.total) return fail(RSB_ERR_OOM, "workspace too small: need %zu bytes, got %zu", p.total, ws_bytes);
    unsigned char* w = static_cast<unsigned char*>(ws);
    float* Db = reinterpret_cast<float*>(w + p.off_D);
    int64_t* Ib = reinterpret_cast<int64_t*>(w + p.off_I);
    for (int q0 = 0; q0 < nq; q0 += p.qb) {
        const int nb = std::min(p.qb, nq - q0);
        const float* qb = q + (size_t)q0 * h->d;
        RSB_TRY(rsb_search(h, qb, nb, k_base, nprobe, Db, Ib, w, p.search_ws, stream));
        RSB_TRY(refine_batch(s, qb, nb, Ib, k_base, k, D + (size_t)q0 * k, I + (size_t)q0 * k, w + p.off_ref,
                             p.total - p.off_ref, staging_bytes, host_rows, (cudaStream_t)stream));
    }
    return RSB_OK;
}

extern "C" int rsb_refine_tiered_profile(int enable, double* ms_out) {
    if (tiered_profile(enable, ms_out) != 0) return fail(RSB_ERR_CUDA, "cudaEventCreate failed");
    return RSB_OK;
}

// ---- SQ8 re-rank store (faiss IndexRefine(base, IndexScalarQuantizer(d, QT_8bit))): uint8 codes + [2, d] (vmin, vdiff)
static int sq8_input_check(const void* x, int x_dtype, int64_t n, int d, const float* sq) {
    if (x_dtype != RSB_DTYPE_F32 && x_dtype != RSB_DTYPE_F16)
        return fail(RSB_ERR_INVALID, "x_dtype must be RSB_DTYPE_F32 or RSB_DTYPE_F16, got %d", x_dtype);
    if (n < 0 || d <= 0) return fail(RSB_ERR_INVALID, "bad n = %lld / d = %d", (long long)n, d);
    if ((n > 0 && !x) || !sq) return fail(RSB_ERR_INVALID, "null argument");
    return RSB_OK;
}

extern "C" int rsb_sq8_train(const void* x, int x_dtype, int64_t n, int d, float* sq, rsb_stream_t stream) {
    RSB_TRY(sq8_input_check(x, x_dtype, n, d, sq));
    if (n == 0) return fail(RSB_ERR_INVALID, "the scalar quantizer needs at least one training row");
    const cudaError_t e = launch_sq8_train(x, x_dtype == RSB_DTYPE_F16, n, d, sq, (cudaStream_t)stream);
    if (e != cudaSuccess) return fail(RSB_ERR_CUDA, "sq8 train: %s", cudaGetErrorString(e));
    return RSB_OK;
}

extern "C" int rsb_sq8_encode(const void* x, int x_dtype, int64_t n, int d, const float* sq, uint8_t* codes,
                              rsb_stream_t stream) {
    RSB_TRY(sq8_input_check(x, x_dtype, n, d, sq));
    if (n == 0) return RSB_OK;
    if (!codes) return fail(RSB_ERR_INVALID, "null argument");
    const cudaError_t e = launch_sq8_encode(x, x_dtype == RSB_DTYPE_F16, n, d, sq, codes, (cudaStream_t)stream);
    if (e != cudaSuccess) return fail(RSB_ERR_CUDA, "sq8 encode: %s", cudaGetErrorString(e));
    return RSB_OK;
}

// ---- training steps (index.train) ---------------------------------------------------------------------------
extern "C" int rsb_kmeans_accumulate(const float* x, int64_t n, int d, const int32_t* assign, int k, float* sums,
                                     float* counts, rsb_stream_t stream) {
    if (!x || !assign || !sums || !counts || n < 0 || d <= 0 || k <= 0) return fail(RSB_ERR_INVALID, "bad argument");
    const cudaError_t e = launch_kmeans_accumulate(x, n, d, assign, k, sums, counts, (cudaStream_t)stream);
    if (e != cudaSuccess) return fail(e == cudaErrorMemoryAllocation ? RSB_ERR_OOM : RSB_ERR_CUDA, "%s", cudaGetErrorString(e));
    CHECK_LAUNCH();
    return RSB_OK;
}
extern "C" int rsb_pq_assign(const float* r, int64_t n, int d, int M, int ksub, const float* codebook, uint8_t* codes,
                             rsb_stream_t stream) {
    if (!r || !codebook || !codes || n < 0 || d <= 0 || M <= 0 || d % M) return fail(RSB_ERR_INVALID, "bad argument");
    if (ksub != 256 && ksub != 16) return fail(RSB_ERR_UNSUPPORTED, "ksub must be 256 or 16 (nbits 8 or 4), got %d", ksub);
    if (ksub == 16) launch_pq_encode4(r, n, d, nullptr, nullptr, codebook, M, false, codes, (cudaStream_t)stream);
    else launch_pq_encode(r, n, d, nullptr, nullptr, codebook, M, codes, (cudaStream_t)stream);
    CHECK_LAUNCH();
    return RSB_OK;
}
extern "C" int rsb_pq_accumulate(const float* r, int64_t n, int d, int M, int ksub, const uint8_t* codes, float* sums,
                                 float* counts, rsb_stream_t stream) {
    if (!r || !codes || !sums || !counts || n < 0 || d <= 0 || M <= 0 || d % M) return fail(RSB_ERR_INVALID, "bad argument");
    if (ksub != 256 && ksub != 16) return fail(RSB_ERR_UNSUPPORTED, "ksub must be 256 or 16 (nbits 8 or 4), got %d", ksub);
    const cudaError_t e = launch_pq_accumulate(r, n, d, M, ksub, codes, sums, counts, (cudaStream_t)stream);
    if (e != cudaSuccess) return fail(e == cudaErrorMemoryAllocation ? RSB_ERR_OOM : RSB_ERR_CUDA, "%s", cudaGetErrorString(e));
    CHECK_LAUNCH();
    return RSB_OK;
}

extern "C" int rsb_peer_broadcast(const void* src_dev, size_t bytes, void* const* dst_ptrs_dev, int npeers,
                                  size_t dst_offset_bytes, rsb_stream_t stream) {
    if (!src_dev || !dst_ptrs_dev || npeers <= 0) return fail(RSB_ERR_INVALID, "null argument");
    if ((bytes & 15) || (dst_offset_bytes & 15) || (reinterpret_cast<uintptr_t>(src_dev) & 15))
        return fail(RSB_ERR_INVALID, "rsb_peer_broadcast needs 16-byte aligned source, offset and size");
    launch_peer_broadcast(src_dev, bytes, dst_ptrs_dev, npeers, dst_offset_bytes, (cudaStream_t)stream);
    CHECK_LAUNCH();
    return RSB_OK;
}

// ---------------------------------------------------------------------------------------------------------
// merge / profiling / layout self-description
// ---------------------------------------------------------------------------------------------------------
extern "C" int rsb_merge_topk(const float* D_all, const int64_t* I_all, int nshards, int nq, int k, int k_out,
                              float* D, int64_t* I, rsb_stream_t stream) {
    if (nshards <= 0 || nq < 0 || k <= 0 || k_out <= 0) return fail(RSB_ERR_INVALID, "bad shape");
    if (nq == 0) return RSB_OK;
    if (!D_all || !I_all || !D || !I) return fail(RSB_ERR_INVALID, "null argument");
    if (launch_merge_shards(D_all, I_all, nshards, nq, k, k_out, D, I, (cudaStream_t)stream) != 0)
        return fail(RSB_ERR_UNSUPPORTED, "nshards * k = %d is too large for the merge kernel", nshards * k);
    CHECK_LAUNCH();
    return RSB_OK;
}

extern "C" int rsb_merge_topk_peers(const float* const* D_ptrs_dev, const int64_t* const* I_ptrs_dev, int nshards, int nq,
                                    int k, int k_out, float* D, int64_t* I, rsb_stream_t stream) {
    if (nshards <= 0 || nq < 0 || k <= 0 || k_out <= 0) return fail(RSB_ERR_INVALID, "bad shape");
    if (nq == 0) return RSB_OK;
    if (!D_ptrs_dev || !I_ptrs_dev || !D || !I) return fail(RSB_ERR_INVALID, "null argument");
    if (launch_merge_shards_peers(D_ptrs_dev, I_ptrs_dev, nshards, nq, k, k_out, D, I, (cudaStream_t)stream) != 0)
        return fail(RSB_ERR_UNSUPPORTED, "nshards * k = %d is too large for the merge kernel", nshards * k);
    CHECK_LAUNCH();
    return RSB_OK;
}

extern "C" int rsb_merge_topk_peers_scatter(const float* const* D_ptrs_dev, const int64_t* const* I_ptrs_dev, int nshards,
                                            int q0, int nq_slice, int k, int k_out, float* const* D_outs_dev,
                                            int64_t* const* I_outs_dev, int nout, rsb_stream_t stream) {
    if (nshards <= 0 || q0 < 0 || nq_slice < 0 || k <= 0 || k_out <= 0 || nout <= 0) return fail(RSB_ERR_INVALID, "bad shape");
    if (nq_slice == 0) return RSB_OK;
    if (!D_ptrs_dev || !I_ptrs_dev || !D_outs_dev || !I_outs_dev) return fail(RSB_ERR_INVALID, "null argument");
    if (launch_merge_shards_peers_scatter(D_ptrs_dev, I_ptrs_dev, nshards, q0, nq_slice, k, k_out, D_outs_dev, I_outs_dev,
                                          nout, (cudaStream_t)stream) != 0)
        return fail(RSB_ERR_UNSUPPORTED, "nshards * k = %d is too large for the merge kernel", nshards * k);
    CHECK_LAUNCH();
    return RSB_OK;
}

extern "C" int rsb_set_option(rsb_index_t* h, int option, int64_t value) {
    if (!h) return fail(RSB_ERR_INVALID, "null handle");
    switch (option) {
        case RSB_OPT_COARSE_TENSOR:
            if (value == 0 && h->kind == RSB_FLAT && h->dtype == RSB_DTYPE_F16)
                return fail(RSB_ERR_UNSUPPORTED, "an fp16 Flat index scores on tensor cores only (no CUDA-core fp16 path)");
            h->coarse_tensor = value != 0; h->flat_tensor = value != 0; return RSB_OK;
        case RSB_OPT_BY_RESIDUAL:
            if (!is_sq8_ivf(h)) return fail(RSB_ERR_INVALID, "RSB_OPT_BY_RESIDUAL applies to an IVFFLAT index with SQ8 storage only");
            if (h->ntotal || h->n_staged || h->ivf_reserved())
                return fail(RSB_ERR_STATE, "by_residual cannot change once vectors are added (or lists reserved)");
            h->by_residual = value != 0; return RSB_OK;
        case RSB_OPT_DEVICE_ROWS:
            if (h->kind != RSB_FLAT)
                return fail(RSB_ERR_INVALID, "RSB_OPT_DEVICE_ROWS applies to a Flat index with fp16 storage (RSB_DTYPE_F16) only");
            if (h->dtype != RSB_DTYPE_F16)
                return fail(RSB_ERR_INVALID, "a tiered Flat index stores fp16 rows: create it with RSB_DTYPE_F16 (an fp32 Flat "
                                             "index stays in device memory)");
            if (h->ntotal || h->n_staged) return fail(RSB_ERR_STATE, "device_rows cannot change once vectors are added");
            if (value < 0) return fail(RSB_ERR_INVALID, "device_rows must be >= 0, got %lld", (long long)value);
            RSB_TRY(ensure_copy_stream(h->tier));
            h->tier.dev_rows = value;
            return RSB_OK;
        case RSB_OPT_STAGING_BYTES:
            if (h->kind != RSB_FLAT || h->dtype != RSB_DTYPE_F16)
                return fail(RSB_ERR_INVALID, "RSB_OPT_STAGING_BYTES applies to a Flat index with fp16 storage (RSB_DTYPE_F16) only");
            if (value < (int64_t)h->row_bytes())
                return fail(RSB_ERR_INVALID, "a staging buffer must hold one row (%zu bytes), got %lld", h->row_bytes(),
                            (long long)value);
            h->tier.staging_bytes = (size_t)value;
            return RSB_OK;
        default: return fail(RSB_ERR_INVALID, "unknown option %d", option);
    }
}

extern "C" int rsb_set_profiling(rsb_index_t* h, int enable) {
    if (!h) return fail(RSB_ERR_INVALID, "null handle");
    h->prof = enable != 0;
    return RSB_OK;
}
extern "C" int rsb_get_profile(rsb_index_t* h, double* out, int n) {
    if (!h || !out || n < RSB_PROF_COUNT) return fail(RSB_ERR_INVALID, "need room for %d doubles", RSB_PROF_COUNT);
    for (int i = 0; i < RSB_PROF_COUNT; ++i) out[i] = 0.0;
    if (h->ev_done <= 0) return fail(RSB_ERR_STATE, "no profiled search on this handle (call rsb_set_profiling first)");
    // average over the searches profiled since the previous call (at most the last kProfSets of them)
    const int nsets = std::min(h->ev_done, (int)rsb_index::kProfSets);
    for (int s = 0; s < nsets; ++s) {
        cudaEvent_t* ev = h->evs[(h->ev_done - 1 - s) % rsb_index::kProfSets];
        CU(cudaEventSynchronize(ev[5]));
        for (int i = 0; i < 5; ++i) {
            float ms = 0.f;
            CU(cudaEventElapsedTime(&ms, ev[i], ev[i + 1]));
            out[i] += ms / nsets;
        }
    }
    h->ev_done = 0;
    unsigned long long host[4] = {0, 0, 0, 0};
    CU(cudaMemcpy(host, h->prof_dev, 32, cudaMemcpyDeviceToHost));
    out[RSB_PROF_SCAN_BYTES] = (double)host[0] * (double)h->row_bytes();
    out[RSB_PROF_PAIRS] = (double)(unsigned)(host[1] & 0xffffffffull);
    out[RSB_PROF_LAUNCHES] = (double)h->launches;
    out[RSB_PROF_SCAN_PATH] = (double)(unsigned)(host[2] & 0xffffffffull);
    out[RSB_PROF_RESCORED] = (double)host[3];
    return RSB_OK;
}

extern "C" int rsb_debug_smem_base(void) { return (int)probe_dynamic_smem_base(0); }

extern "C" int rsb_pq_lut_floats(rsb_index_t* h) {
    if (!h || h->kind != RSB_IVFPQ) return -1;
    return pq_interleaved_layout(h->Mb) ? kLutWords : h->Mb * 256;
}
extern "C" int rsb_pq_tables(rsb_index_t* h, const float* q, int nq, float* lut, rsb_stream_t stream) {
    if (!h || h->kind != RSB_IVFPQ) return fail(RSB_ERR_INVALID, "rsb_pq_tables needs an IVFPQ index");
    if (nq < 0 || (nq > 0 && (!q || !lut))) return fail(RSB_ERR_INVALID, "null argument");
    if (!h->has_codebook) return fail(RSB_ERR_STATE, "index has no PQ codebook");
    launch_pq_tables(h, q, nq, lut, (cudaStream_t)stream);
    CHECK_LAUNCH();
    return RSB_OK;
}

extern "C" int rsb_pq_layout_offset(int M, int v, int m) {
    if (v < 0 || v >= 32 || m < 0 || m >= M) return -1;
    if (pq_interleaved_layout(M)) return pq_byte_off(M, v, m);
    if ((M & 3) || M > 128 || M <= 0) return -1;
    return v * M + m;                               // generic M: natural order
}
extern "C" int rsb_pq_lut_index(int M, int j, int m) {
    if (j < 0 || j >= 256 || m < 0 || m >= M) return -1;
    if (pq_interleaved_layout(M)) return j * kLutRowWords + m;
    if ((M & 3) || M > 128 || M <= 0) return -1;
    return m * 256 + j;
}
