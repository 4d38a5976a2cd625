/*
 * rsb.h -- C-ABI of librsb (retrieval-scaling on H100): the drop-in boundary for the reference's
 * query -> top-k retrieval path.  Plain C types only: device pointers, sizes and a cudaStream_t passed
 * as void*.  No torch / C++ types cross this boundary.
 *
 * The reference (RulinShao/retrieval-scaling @ 9da3070) has no FFI of its own: its seam is the SWIG'd
 * `faiss` object protocol used by src/indicies/*.py.  Each entry point below names the reference call
 * site it replaces (paths relative to the reference root).  INTEGRATION.md shows the ctypes stub a
 * reference maintainer would add.
 *
 * Conventions
 *   - every function returns an int status: RSB_OK (0) or a negative RSB_ERR_* class; the message of the
 *     last error on the calling thread is available from rsb_last_error().  Nothing aborts the process and
 *     nothing falls back to the CPU.
 *   - all `*_dev` pointers are CUDA device pointers on the current device; they are owned by the caller.
 *     The library owns index storage behind the opaque handle (create/.../free).
 *   - work is enqueued on `stream`; results are valid after the stream is synchronised.  Functions that
 *     must read a size back (rsb_finalize) synchronise the stream themselves and say so.
 *   - search semantics are those of faiss 1.8.0 METRIC_INNER_PRODUCT indexes: scores float32, rows sorted
 *     by score descending, missing results padded with id -1 / score -FLT_MAX.
 */
#ifndef RSB_H_
#define RSB_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RSB_VERSION 301 /* 0.3.1 */

enum {
    RSB_OK = 0,
    RSB_ERR_INVALID = -1,     /* bad argument                         -> ValueError          */
    RSB_ERR_CUDA = -2,        /* CUDA runtime / launch failure        -> RuntimeError        */
    RSB_ERR_STATE = -3,       /* e.g. search before train             -> RuntimeError        */
    RSB_ERR_UNSUPPORTED = -4, /* e.g. nbits = 6                       -> NotImplementedError */
    RSB_ERR_OOM = -5          /* cudaMalloc failed / workspace small  -> MemoryError         */
};

enum { RSB_FLAT = 0, RSB_IVFFLAT = 1, RSB_IVFPQ = 2 };

typedef struct rsb_index rsb_index_t;
typedef void* rsb_stream_t; /* cudaStream_t */

int rsb_version(void);
const char* rsb_last_error(void);

/* ---- construction -------------------------------------------------------------------------------- */
/* dtype: storage dtype of the vectors (enum RSB_DTYPE_* below; anything else: RSB_ERR_INVALID).
 *   RSB_DTYPE_F32   fp32 rows.
 *   RSB_DTYPE_F16   every row as fp16 -- the embedding task writes fp16 passage embeddings (src/embed.py:137-138)
 *     and the reference upcasts them only on load (src/indicies/flat.py:86), so fp16 storage of them is lossless at
 *     half the bytes.  faiss equivalent: IndexScalarQuantizer / IndexIVFScalarQuantizer(QT_fp16, METRIC_INNER_PRODUCT,
 *     no residual).  Stored values are the fp16 rounding (to nearest even) of what is added; scores are exact fp32
 *     inner products of the fp32 query with the decoded rows.  d % 8 == 0 (16-byte rows), else RSB_ERR_INVALID. */
/* faiss.IndexFlatIP(d)                           <- src/indicies/flat.py:42, ric/conf/default.yaml `index_type: Flat`
 * fp16 rows are scored on wgmma tensor cores from the fp16 rows themselves (scaled fp16 hi/lo query split, then an
 * exact fp32 re-score) and need d % 64 == 0, else RSB_ERR_UNSUPPORTED.  Final scores equal the fp32 index's wherever
 * both return the same id. */
int rsb_flat_create(int d, int dtype, rsb_index_t** out);
/* faiss.IndexIVFFlat(IndexFlatIP(d), d, nlist, METRIC_INNER_PRODUCT)
 *                                                    <- src/indicies/ivf_flat.py:143-149, api/conf/ivf_flat.yaml
 * With fp16 rows the list scan reads 2 bytes per element and adds in the fp32 scan's order: ids and scores are
 * bit-identical to an fp32 index holding the same values.
 * dtype = RSB_DTYPE_SQ8: faiss.IndexIVFScalarQuantizer(IndexFlatIP(d), d, nlist, QT_8bit, METRIC_INNER_PRODUCT,
 *   by_residual), factory string "IVFn,SQ8": one uint8 code per element, d % 16 == 0 (else RSB_ERR_INVALID), with the
 *   train / encode / decode rules of the SQ8 re-rank store below.  The range [2, d] is set with rsb_set_sq_range before
 *   anything is added (rsb_add / rsb_add_codes / rsb_search before it: RSB_ERR_STATE).  RSB_OPT_BY_RESIDUAL (default 0)
 *   selects faiss' by_residual: rows are encoded as x - c_list (fp32 subtraction; fp16 rows widen exactly) and every
 *   score of list l is fl32(coarse_dis + s), coarse_dis = <q, c_l> added once after s = <q, decode(code)> is complete.
 *   The list scan loads one 4-byte word of codes per lane and step and decodes every element before the fp32 scan's
 *   fmaf sequence, so s (and, without residuals, ids and scores) is bit-identical to an fp32 index holding the decoded
 *   rows in the same lists. */
int rsb_ivfflat_create(int d, int nlist, int dtype, rsb_index_t** out);
/* faiss.IndexIVFPQ(IndexFlatIP(d), d, nlist, M, nbits, METRIC_INNER_PRODUCT)
 *                                                                    <- src/indicies/ivf_pq.py:146-152
 * M must divide d, else RSB_ERR_INVALID.  nbits other than 8 / 4 (codes crossing bytes, tables beyond shared memory)
 * returns RSB_ERR_UNSUPPORTED (-> NotImplementedError in Python).
 *   nbits = 8   tables of 256 entries, one byte per code.  M = 16, 32 or 64 run the tuned ADC scan (K = M/16 lanes of a
 *     warp cooperate on one vector with a bank-conflict-free look-up layout that exists for K in {1, 2, 4}:
 *     csrc/rsb_layout.h); any other multiple of 4 up to 128 (e.g. 24 / 48 / 96 on d = 768, which faiss and the
 *     reference's n_subquantizers key accept) runs a functionally complete generic path (natural code order, [m][256]
 *     tables, one thread per vector) -- correct, not tuned.  Other M: RSB_ERR_UNSUPPORTED.
 *   nbits = 4   codes are packed two per byte in faiss' order (PQEncoderGeneric, LSB first: byte b = c[2b] | c[2b+1] <<
 *     4), so a vector holds Mb = M / 2 code bytes, and the index is scanned as an 8-bit index of Mb byte sub-quantizers
 *     with the pair tables T'[b][j] = T[2b][j & 15] + T[2b+1][j >> 4]: M = 32 / 64 / 128 run the tuned scan (Mb = 16 /
 *     32 / 64), any other M with M % 8 == 0 and M / 2 <= 128 the generic one; other M: RSB_ERR_INVALID.  Scores differ
 *     from faiss' sequential sum over m by fp32 rounding only.  The codebook (rsb_set_pq_codebook /
 *     rsb_get_pq_codebook) is [M, 16, d/M], and codes (rsb_add_codes, rsb_export_lists) are [n, M / 2] packed bytes. */
int rsb_ivfpq_create(int d, int nlist, int M, int nbits, rsb_index_t** out);
int rsb_free(rsb_index_t* h);

/* ---- trained state (what index.train() produces; ivf_flat.py:166, ivf_pq.py:170) ------------------ */
/* coarse centroids [nlist, d] float32, copied */
int rsb_set_centroids(rsb_index_t* h, const float* centroids_dev, rsb_stream_t stream);
/* PQ codebook [M, 2^nbits, d/M] float32, copied */
int rsb_set_pq_codebook(rsb_index_t* h, const float* codebook_dev, rsb_stream_t stream);
int rsb_get_centroids(rsb_index_t* h, float* out_dev, rsb_stream_t stream);
int rsb_get_pq_codebook(rsb_index_t* h, float* out_dev, rsb_stream_t stream);

/* ---- population (index.add(x): flat.py:58, ivf_flat.py:180, ivf_pq.py:185) ------------------------- */
/* Rows x_dev [n, d] in x_dtype (RSB_DTYPE_F32 or RSB_DTYPE_F16, else RSB_ERR_INVALID), converted on the device to the
 * index's storage dtype: the embedding pickles' fp16 rows (src/indicies/flat.py:58-59, ivf_flat.py:180) cross PCIe once
 * at 2 bytes per element.  IVFPQ takes RSB_DTYPE_F32 only (RSB_ERR_UNSUPPORTED otherwise).  ids_dev may be NULL: ids
 * are then sequential from ntotal (faiss behaviour).  IVF: list = argmax_c <x,c> computed here in fp32 (fp16 rows are
 * assigned on their upcast, exact values, so the lists are those an fp32 index assigns); IVFPQ additionally encodes the
 * residual.  ws_dev/ws_bytes: see rsb_add_workspace_bytes. */
size_t rsb_add_workspace_bytes(rsb_index_t* h, int64_t n);
int rsb_add(rsb_index_t* h, const void* x_dev, int x_dtype, int64_t n, const int64_t* ids_dev, void* ws_dev,
            size_t ws_bytes, rsb_stream_t stream);
/* as rsb_add but the coarse assignment is supplied by the caller (int32 list id per row) */
int rsb_add_preassigned(rsb_index_t* h, const void* x_dev, int x_dtype, int64_t n, const int64_t* ids_dev,
                        const int32_t* list_dev, rsb_stream_t stream);
/* rows that are already codes (e.g. read from an existing index file): IVFPQ: PQ codes [n, M * nbits / 8] uint8;
 * IVFFLAT with SQ8 storage: SQ8 codes [n, d] uint8 of the index's range (encoded by residual when RSB_OPT_BY_RESIDUAL
 * is set).  Other indexes: RSB_ERR_INVALID. */
int rsb_add_codes(rsb_index_t* h, const uint8_t* codes_dev, int64_t n, const int64_t* ids_dev,
                  const int32_t* list_dev, rsb_stream_t stream);
/* Build the searchable layout (CSR inverted lists; PQ codes interleaved per 32 vectors).  Synchronises
 * `stream`.  rsb_search calls it implicitly when adds are pending.  No-op on an index with reserved lists. */
int rsb_finalize(rsb_index_t* h, rsb_stream_t stream);
/* Tiered IVFFLAT index (any storage dtype), for datastores larger than device memory: the list sizes are given up
 * front and the lists are split by id between device memory and page-locked host memory.
 *   sizes_host [nlist] int64 (host memory) fixes the CSR offsets.  L_dev = the largest list count whose rows fit
 *   device_rows: lists [0, L_dev) keep their rows in device memory (allocated once, here), lists [L_dev, nlist) in one
 *   page-locked block the handle owns, of exactly the bytes those lists need.  Ids, centroids, the SQ8 range and the
 *   list tables stay in device memory (8 bytes of ids per vector).  staging_bytes is the size of one of the two staging
 *   buffers a search copies host lists into (0: 256 MiB; raised to the largest host list, lowered to the host tier).
 *   Synchronises `stream`.
 * Refusals: an IVFPQ or FLAT handle, negative sizes or device_rows: RSB_ERR_INVALID; an untrained handle, a second
 * reservation, or rows already added: RSB_ERR_STATE.
 * After it, rsb_add / rsb_add_preassigned / rsb_add_codes place every row in its final slot: the batch is assigned (and
 * SQ8-encoded) on the device as before, stably sorted by list (insertion order inside a list is kept), device-tier rows
 * are scattered in place and host-tier rows copied device to host, one copy per run of consecutive slots; each add
 * synchronises `stream`.  A batch that would overflow a list's reservation is refused whole with RSB_ERR_STATE.
 * rsb_search, rsb_export_lists and rsb_export_rows before every reserved row has arrived return RSB_ERR_STATE (the
 * message gives both counts).  rsb_list_sizes reports the reserved sizes.
 * rsb_search / rsb_search_preassigned keep their signatures.  Per query batch: the coarse step; a kernel flags the host
 * lists the batch probes and the [nlist] flags are copied to the host; the device lists are scanned in place, enqueued
 * before the host waits for the flags (the one host synchronisation per batch: only the host can drive the copy
 * engine); then the probed host lists are packed in list order into chunks of at most one staging buffer, copied by a
 * copy stream the handle owns into two staging buffers of the workspace and scanned chunk by chunk.  Every (query,
 * list) pair is scanned once, by the all-device scan kernel on the same bytes; all pieces share the batch's top-k
 * thresholds and one merge gives the result, so ids and scores equal those of the all-device index of the same lists
 * (up to the order of exact score ties at the k-th place).  Shared thresholds (rsb_search_preassigned with
 * tau_local_dev) return RSB_ERR_UNSUPPORTED.
 * RSB_INFO_DEVICE_ROWS: the rows of lists [0, L_dev) (<= device_rows); RSB_INFO_HOST_BYTES: the host tier;
 * RSB_INFO_INDEX_BYTES: device bytes, as for every index.  Without a reservation nothing changes. */
int rsb_reserve_lists(rsb_index_t* h, const int64_t* sizes_host, int64_t device_rows, size_t staging_bytes,
                      rsb_stream_t stream);

/* ---- introspection --------------------------------------------------------------------------------- */
enum {
    RSB_INFO_KIND = 0, RSB_INFO_D = 1, RSB_INFO_NLIST = 2, RSB_INFO_M = 3, RSB_INFO_NBITS = 4,
    RSB_INFO_NTOTAL = 5,       /* index.ntotal     */
    RSB_INFO_IS_TRAINED = 6,   /* index.is_trained */
    RSB_INFO_MAX_LIST_LEN = 7,
    RSB_INFO_INDEX_BYTES = 8,  /* device bytes held by the searchable layout */
    RSB_INFO_DTYPE = 9,        /* storage dtype of the vectors: RSB_DTYPE_F32 / RSB_DTYPE_F16 / RSB_DTYPE_SQ8 (IVFPQ:
                                  RSB_DTYPE_F32) */
    RSB_INFO_BY_RESIDUAL = 10, /* 1 if an SQ8 IVFFLAT index encodes residuals (RSB_OPT_BY_RESIDUAL), else 0 */
    RSB_INFO_HOST_BYTES = 11,  /* page-locked host bytes held by the host tier of a tiered Flat index or of an IVFFLAT
                                  index with reserved lists (0 on other handles) */
    RSB_INFO_DEVICE_ROWS = 12  /* rows held in device memory: min(device_rows, ntotal) on a tiered Flat index, the rows of
                                  lists [0, L_dev) on an IVFFLAT index with reserved lists, else ntotal */
};
int rsb_info(rsb_index_t* h, int what, int64_t* out);
/* list sizes [nlist] int64 to a device buffer */
int rsb_list_sizes(rsb_index_t* h, int64_t* sizes_dev, rsb_stream_t stream);
/* Export the inverted lists in natural CSR order (insertion order inside each list), as the oracle and a
 * faiss file writer want them: offsets_dev [nlist+1] int64, payload_dev = uint8 codes [ntotal, M * nbits / 8] (IVFPQ)
 * or vectors [ntotal, d] in the storage dtype, float32 or fp16 (IVFFLAT / FLAT), or uint8 SQ8 codes [ntotal, d]
 * (IVFFLAT with SQ8 storage), ids_dev [ntotal] int64.  Any pointer may be NULL. */
int rsb_export_lists(rsb_index_t* h, int64_t* offsets_dev, void* payload_dev, int64_t* ids_dev,
                     rsb_stream_t stream);
/* Rows [r0, r0 + n) of a FLAT index, or CSR rows [r0, r0 + n) of an IVFFLAT index (the natural order of
 * rsb_export_lists), in the storage dtype ([n, d]; SQ8: uint8 codes), copied from whichever tier holds them to dst,
 * which may be device memory or host memory (pageable or pinned).  Lets a caller export a tiered index larger than
 * device memory one range at a time.  Pending adds are finalised first.  IVFPQ handles, or a range outside
 * [0, ntotal): RSB_ERR_INVALID; an IVFFLAT index whose reserved rows have not all arrived: RSB_ERR_STATE. */
int rsb_export_rows(rsb_index_t* h, int64_t r0, int64_t n, void* dst, rsb_stream_t stream);

/* ---- search (index.search(x, k) + index.nprobe: flat.py:139, ivf_flat.py:73,225, ivf_pq.py:76,230) --- */
/* covers the fp16 Flat index's scaled query split (2 x [nq, d] fp16 + [nq] fp32 per query batch), and on a tiered Flat
 * index two staging buffers of RSB_OPT_STAGING_BYTES each (fewer when the host tier is smaller), so a search allocates
 * nothing */
size_t rsb_workspace_bytes(rsb_index_t* h, int nq, int k, int nprobe);
/* q_dev [nq, d] float32; D_dev [nq, k] float32; I_dev [nq, k] int64.  nprobe ignored for FLAT. */
int rsb_search(rsb_index_t* h, const float* q_dev, int nq, int k, int nprobe,
               float* D_dev, int64_t* I_dev, void* ws_dev, size_t ws_bytes, rsb_stream_t stream);
/* faiss IndexIVF::search_preassigned: as rsb_search, but the probed lists list_dev [nq, nprobe] int64 (-1 =
 * skip) and their coarse scores coarse_dis_dev [nq, nprobe] float32 (<q, c_list>, added to every score of that list
 * by IVFPQ and by an SQ8 IVFFLAT index with RSB_OPT_BY_RESIDUAL; ignored by other IVFFLAT indexes) come from the
 * caller instead of the coarse quantizer.
 * Thresholds: tau_local_dev = NULL (with tau_peers_dev = NULL, npeers = 0) keeps the per-query running top-k
 * thresholds in the workspace.  Otherwise they are shared between GPUs (one process per GPU, datastore partitioned
 * across the GPUs; replaces the reference's one-process-per-shard search, src/search.py:282-296) in caller-owned
 * peer-mapped arrays: tau_local_dev [nq] uint32 is THIS GPU's array; tau_peers_dev is a DEVICE array of `npeers` base
 * pointers, one per GPU of the job (the own entry is recognised and skipped).  Whenever the scan raises a threshold it
 * also raises it on every peer (relaxed system-scope max reduction over NVLink), so every GPU filters with the best
 * bound found anywhere; results are unchanged (a bound is always the k-th best score of real candidates of that query).
 * The caller zeroes the arrays before the first search of a batch on ANY GPU and keeps the GPUs within one batch of
 * each other (a cross-GPU barrier per batch, which the top-k combine provides).  An inconsistent set (npeers < 0,
 * npeers > 0 without tau_peers_dev, or tau_peers_dev / npeers without tau_local_dev) returns RSB_ERR_INVALID before
 * any launch. */
int rsb_search_preassigned(rsb_index_t* h, const float* q_dev, int nq, int k, int nprobe,
                           const int64_t* list_dev, const float* coarse_dis_dev, float* D_dev, int64_t* I_dev,
                           void* ws_dev, size_t ws_bytes, uint32_t* tau_local_dev, uint32_t* const* tau_peers_dev,
                           int npeers, rsb_stream_t stream);
/* Copy `bytes` from src_dev to dst_ptrs_dev[p] + dst_offset_bytes for every p < npeers (peer-mapped destinations; P2P
 * stores over NVLink).  Used to publish a rank's slice of the coarse-quantizer tables to every GPU without NCCL.
 * 16-byte aligned pointers / sizes. */
int rsb_peer_broadcast(const void* src_dev, size_t bytes, void* const* dst_ptrs_dev, int npeers, size_t dst_offset_bytes,
                       rsb_stream_t stream);
/* coarse quantizer only: top-`nprobe` lists per query (the IndexFlatIP quantizer's search).
 * list_dev [nq, nprobe] int64, score_dev [nq, nprobe] float32 (may be NULL). */
int rsb_coarse(rsb_index_t* h, const float* q_dev, int nq, int nprobe, int64_t* list_dev, float* score_dev,
               void* ws_dev, size_t ws_bytes, rsb_stream_t stream);

/* ---- exact re-ranking (faiss IndexRefine / IndexRefineFlat::search; the reference's unused re-score path
 *      src/indicies/ivf_pq.py:119-123 `get_knn_scores` against `self.embeds`) ------------------------------------
 * The re-rank store is caller-owned, [ntotal, d], row i = the vector of index id i.  Scores are <q, x_id> accumulated
 * in fp32 from the decoded elements, in the same order for every store dtype (an fp16 store and an fp32 store of the
 * same fp16-representable values agree bit for bit).  Rows are sorted by score descending, ties by ascending id; fewer
 * than k valid candidates are padded with id -1 / score -FLT_MAX; candidate ids -1 (and ids outside [0, ntotal)) are
 * skipped.  k_base = k * k_factor <= 4096 (the scan's k limit); larger returns RSB_ERR_UNSUPPORTED.  ntotal <= 2^31.
 *
 * store_dtype (anything else: RSB_ERR_INVALID)
 *   RSB_DTYPE_F32, RSB_DTYPE_F16   fp32 / fp16 rows, d % 8 == 0 (16-byte rows); sq_dev is ignored.
 *   RSB_DTYPE_SQ8   faiss IndexRefine(base, IndexScalarQuantizer(d, QT_8bit)), factory string "...,Refine(SQ8)": one
 *     uint8 code per element, d % 16 == 0 (whole 16-byte rows).  Scalar quantizer QT_8bit, RS_minmax, one range per
 *     dimension; sq_dev (16-byte aligned) is [2, d] float32: vmin [d], then vdiff [d] (faiss' `sq.trained` layout).
 *     Every operation below is a separately rounded fp32 operation:
 *       train   vmin[j] = min over the rows of x[:, j], vdiff[j] = max - vmin[j]
 *       encode  xi = vdiff != 0 ? (x - vmin) / vdiff : 0, clamped to [0, 1]; code = (int)(255.f * xi)  (rows outside the
 *               trained range clamp; fp16 input is encoded from its exact fp32 value)
 *       decode  x = vmin + ((code + 0.5f) / 255.f) * vdiff
 *     The re-rank decodes every element and scores it as the fp32 store does (same lane order, same fmaf sequence), so
 *     ids and scores are bit-identical to an fp32 store holding the decoded rows.
 *
 * Tiers: rows [0, n_dev) are device memory (store_dev, 16-byte aligned), rows [n_dev, ntotal) page-locked host memory
 * mapped into the device address space (store_host points at row n_dev, not row 0; 16-byte aligned).  0 <= n_dev <=
 * ntotal, else RSB_ERR_INVALID.
 *   n_dev = ntotal   the all-device store: store_host and staging_bytes are ignored.
 *   n_dev < ntotal   the tiered store (n_dev = 0 keeps every row on the host).  Results are bit-identical to the
 *     all-device store holding the same values.  Queries are processed in chunks of floor(staging_bytes / (k_base * d *
 *     elem_bytes)) (staging_bytes must hold at least one query's worst case).  Within a chunk the host-tier candidates
 *     are de-duplicated on the device (radix sort by id), every distinct host row crosses PCIe once into a staging
 *     buffer inside the workspace, and the re-rank reads it from there; device-tier rows never cross PCIe.  Nothing
 *     synchronises the host.  host_rows_dev (device int64, may be NULL) is incremented by the number of distinct host
 *     rows gathered.  A host tier that is not page-locked and mapped (pageable memory, a device pointer) returns
 *     RSB_ERR_INVALID.
 * Every argument is checked before any launch.  The workspace queries return 0 for arguments the call would refuse;
 * they size the all-device store by nq, k_base and k alone, and the tiered store by its dtype and staging_bytes. */
/* RSB_DTYPE_SQ8: a re-rank store, or the storage of an IVFFLAT index (rsb_ivfflat_create); not a Flat index */
/* RSB_DTYPE_BF16: readers only (rsb_llm_create); every index and re-rank store creator refuses it (RSB_ERR_INVALID) */
enum { RSB_DTYPE_F32 = 0, RSB_DTYPE_F16 = 1, RSB_DTYPE_SQ8 = 2, RSB_DTYPE_BF16 = 3 };
int rsb_host_alloc(size_t bytes, void** out);   /* cudaHostAlloc(portable | mapped): exactly `bytes`, unlike torch's
                                                   pinned allocator, which rounds blocks up to a power of two */
int rsb_host_free(void* p);
size_t rsb_refine_workspace_bytes(int nq, int k_base, int k, int d, int store_dtype, int64_t n_dev, int64_t ntotal,
                                  size_t staging_bytes);
/* re-rank given candidates cand_dev [nq, k_base] int64 (e.g. a search result at k_base) -> D_dev/I_dev [nq, k] */
int rsb_refine(const float* q_dev, int nq, const void* store_dev, int64_t n_dev, const void* store_host,
               int store_dtype, const float* sq_dev, int d, int64_t ntotal, const int64_t* cand_dev, int k_base, int k,
               float* D_dev, int64_t* I_dev, void* ws_dev, size_t ws_bytes, size_t staging_bytes,
               int64_t* host_rows_dev, rsb_stream_t stream);
/* IndexRefine::search on an IVFPQ handle: rsb_search at k_base = k * k_factor into the workspace, then rsb_refine */
size_t rsb_search_refine_workspace_bytes(rsb_index_t* h, int nq, int k, int k_factor, int nprobe, int store_dtype,
                                         int64_t n_dev, int64_t ntotal, size_t staging_bytes);
int rsb_search_refine(rsb_index_t* h, const float* q_dev, int nq, int k, int k_factor, int nprobe,
                      const void* store_dev, int64_t n_dev, const void* store_host, int store_dtype,
                      const float* sq_dev, int64_t ntotal, float* D_dev, int64_t* I_dev, void* ws_dev,
                      size_t ws_bytes, size_t staging_bytes, int64_t* host_rows_dev, rsb_stream_t stream);
/* enable != 0: time the sort / gather / score stages of every later tiered chunk with CUDA events, on the device
 * current at the call (this waits for each chunk on the host: for measurement only).  ms_out (may be NULL) receives
 * the [3] milliseconds accumulated since the previous call, which resets them. */
int rsb_refine_tiered_profile(int enable, double* ms_out);
/* Train / encode an SQ8 store (rules above): x_dev [n, d] in x_dtype (RSB_DTYPE_F32 / RSB_DTYPE_F16); codes_dev [n, d]
 * uint8.  rsb_sq8_train needs n >= 1. */
int rsb_sq8_train(const void* x_dev, int x_dtype, int64_t n, int d, float* sq_dev, rsb_stream_t stream);
int rsb_sq8_encode(const void* x_dev, int x_dtype, int64_t n, int d, const float* sq_dev, uint8_t* codes_dev,
                   rsb_stream_t stream);
/* The range of an IVFFLAT index with SQ8 storage: sq_dev [2, d] float32 (vmin, then vdiff), copied.  Other handles:
 * RSB_ERR_INVALID.  rsb_set_sq_range on a populated index and rsb_get_sq_range before a range is set: RSB_ERR_STATE.
 * RSB_INFO_IS_TRAINED of such an index means centroids and range are both set. */
int rsb_set_sq_range(rsb_index_t* h, const float* sq_dev, rsb_stream_t stream);
int rsb_get_sq_range(rsb_index_t* h, float* out_dev, rsb_stream_t stream);

/* ---- shard merge (src/search.py:357-367; api/serve_main_node.py:130-163) ---------------------------- */
/* D_all_dev/I_all_dev [nshards, nq, k]: concat per query, sort by score desc (ties: lower shard, then lower
 * rank, i.e. Python's stable sort over shard order), keep k_out.  Entries with id < 0 are ignored. */
int rsb_merge_topk(const float* D_all_dev, const int64_t* I_all_dev, int nshards, int nq, int k, int k_out,
                   float* D_dev, int64_t* I_dev, rsb_stream_t stream);

/* Fused gather + merge for one box: D_ptrs_dev / I_ptrs_dev are DEVICE arrays of nshards pointers; entry s points
 * at shard s's [nq, k] scores / ids, which may live on another GPU (peer-mapped / symmetric memory).  The kernel
 * reads them in place with P2P loads over NVLink, so no all-gather buffer is materialised.  The caller orders the
 * producers before this call (cross-GPU barrier). */
int rsb_merge_topk_peers(const float* const* D_ptrs_dev, const int64_t* const* I_ptrs_dev, int nshards, int nq, int k,
                         int k_out, float* D_dev, int64_t* I_dev, rsb_stream_t stream);
/* Query-sliced form of the same merge (same reference semantics, src/search.py:357-367): this GPU merges only
 * queries [q0, q0 + nq_slice) from all shards and stores each merged row into every one of the `nout` result
 * buffers D_outs_dev[o] / I_outs_dev[o] (each [nq, k_out], peer-mapped), i.e. the gather of the inputs and the
 * broadcast of the outputs are both P2P traffic of this one kernel.  The caller provides a cross-GPU barrier before
 * (inputs complete) and after (outputs complete). */
int rsb_merge_topk_peers_scatter(const float* const* D_ptrs_dev, const int64_t* const* I_ptrs_dev, int nshards, int q0,
                                 int nq_slice, int k, int k_out, float* const* D_outs_dev, int64_t* const* I_outs_dev,
                                 int nout, rsb_stream_t stream);

/* ---- dense exact search without an index object (used for ground truth / k-means assignment) -------- */
size_t rsb_knn_workspace_bytes(int nq, int64_t n, int k);
int rsb_knn_ip(const float* q_dev, int nq, const float* x_dev, int64_t n, int d, int k, int64_t id_offset,
               float* D_dev, int64_t* I_dev, void* ws_dev, size_t ws_bytes, rsb_stream_t stream);

/* ---- training steps (index.train(x): src/indicies/ivf_flat.py:166, ivf_pq.py:170 -> faiss Clustering /
 *      ProductQuantizer::train).  Lloyd iterations are driven by the host (retrieval_scaling_b200/train.py); the
 *      arithmetic runs here.  Coarse assignment step = rsb_coarse(..., nprobe = 1) on a scratch handle holding the
 *      current centroids. ------------------------------------------------------------------------------------ */
/* sums_dev [k, d] += x[i], counts_dev [k] (float) += 1 for assign_dev[i] (int32, out-of-range ids are skipped) */
int rsb_kmeans_accumulate(const float* x_dev, int64_t n, int d, const int32_t* assign_dev, int k, float* sums_dev,
                          float* counts_dev, rsb_stream_t stream);
/* PQ k-means steps with ksub = 256 (nbits = 8) or ksub = 16 (nbits = 4) entries per sub-quantizer; other ksub ->
 * RSB_ERR_UNSUPPORTED.  codebook_dev [M, ksub, d/M]; codes_dev [n, M], one code per byte (not packed).
 * assignment: codes_dev[i, m] = argmin_j || r[i, m-th slice] - codebook[m][j] ||^2, the lowest j winning exact ties.
 * update: sums_dev [M, ksub, d/M] += slices, counts_dev [M, ksub] (float) += 1.  Member sums are added in a fixed
 * order, so training gives the same codebook on every run. */
int rsb_pq_assign(const float* r_dev, int64_t n, int d, int M, int ksub, const float* codebook_dev, uint8_t* codes_dev,
                  rsb_stream_t stream);
int rsb_pq_accumulate(const float* r_dev, int64_t n, int d, int M, int ksub, const uint8_t* codes_dev, float* sums_dev,
                      float* counts_dev, rsb_stream_t stream);

/* ---- options -------------------------------------------------------------------------------------------- */
enum {
    RSB_OPT_COARSE_TENSOR = 0,/* 1 (default): wgmma tensor-core candidates re-scored exactly in fp32 (coarse quantizer:
                                 fp16 hi/lo split of queries and centroids; fp32 Flat: 3xTF32); 0: CUDA-core fp32
                                 FMA tiles.  0 on an fp16 Flat index returns RSB_ERR_UNSUPPORTED: its rows are
                                 scored on tensor cores only */
    RSB_OPT_BY_RESIDUAL = 1,  /* SQ8 IVFFLAT only (RSB_ERR_INVALID on other handles), before anything is added
                                 (RSB_ERR_STATE after): 1 encodes x - c_list and adds the coarse score (faiss by_residual,
                                 the default of index_factory "IVFn,SQ8"); 0 (default) encodes x */
    RSB_OPT_DEVICE_ROWS = 2,  /* tiered Flat index, for datastores larger than device memory.  FLAT with RSB_DTYPE_F16 only
                                 (RSB_ERR_INVALID on other handles, fp32 Flat included), before anything is added
                                 (RSB_ERR_STATE after), value >= 0.  Rows [0, value) are kept in device memory (allocated
                                 once, at `value` rows, by the first add), rows from `value` on in page-locked host
                                 blocks the handle owns, one of exactly the bytes needed per add; no row is ever held
                                 twice.  rsb_add then also takes x in host memory (pageable or pinned): rows bound for
                                 the host tier are copied host to host (fp32 rows rounded to nearest even there), rows
                                 bound for the device tier cross PCIe once.
                                 rsb_search keeps its signature and semantics.  Per query batch a copy stream owned by
                                 the handle copies consecutive host chunks (RSB_OPT_STAGING_BYTES each) into two staging
                                 buffers of the workspace on the copy engine, while the device tier and then each
                                 resident chunk are scored: the fp16 candidate path of the all-device index over the
                                 piece's rows, the exact fp32 re-score of its candidates, and a merge into the running
                                 top-k (ties: the lower row).  Events order the reuse of the buffers and the copy stream
                                 is joined back to `stream`; nothing synchronises the host.  Scores are bit-equal to the
                                 all-device index wherever both return the same id.  While ntotal <= value the search is
                                 the all-device one. */
    RSB_OPT_STAGING_BYTES = 3 /* tiered Flat: bytes of one staging buffer (the search holds two), value >= d * 2 (one
                                 row); default 256 MiB.  FLAT with RSB_DTYPE_F16 only, at any time */
};
int rsb_set_option(rsb_index_t* h, int option, int64_t value);

/* ---- profiling: per-stage CUDA-event timings of the last rsb_search on this handle ------------------- */
enum {
    RSB_PROF_COARSE_MS = 0, /* centroid scan (sgemm + select)          */
    RSB_PROF_SETUP_MS = 1,  /* (query,list) work-list construction      */
    RSB_PROF_LUT_MS = 2,    /* PQ look-up-table build                   */
    RSB_PROF_SCAN_MS = 3,   /* inverted-list scan kernel (the hot one)  */
    RSB_PROF_MERGE_MS = 4,  /* per-query top-k merge                    */
    RSB_PROF_SCAN_BYTES = 5,/* algorithmic bytes of the scan: sum over probed (q,list) pairs of len*row_bytes
                               (IVF-Flat row_bytes = d * 4, d * 2 with fp16 storage, d with SQ8 storage) */
    RSB_PROF_PAIRS = 6,     /* number of valid (q,list) pairs            */
    RSB_PROF_LAUNCHES = 7,  /* kernels launched by the last search       */
    RSB_PROF_SCAN_PATH = 8, /* IVFPQ scan: 1 = literal-offset shared-memory look-ups, 2 = generic addressing */
    RSB_PROF_RESCORED = 9,  /* IVFPQ paired scan: vectors re-scored exactly after the quantised-table filter */
    RSB_PROF_COUNT = 10
};
int rsb_set_profiling(rsb_index_t* h, int enable);
/* synchronises the events of the last search; out[RSB_PROF_COUNT] doubles */
int rsb_get_profile(rsb_index_t* h, double* out, int n);

/* ---- query encoder: BERT-base forward in fp16 on wgmma tensor cores ------------------------------------
 * Replaces `model(**encoded_batch)` (src/search.py:92) for `Contriever(BertModel)` (contriever/src/contriever.py:
 * 11-55) and plain HF BERT checkpoints with CLS pooling (src/search.py:93-94).  Token streams are un-padded:
 * input_ids / token_type_ids are [T] int32 (padding removed), cu_seqlens [B+1] int32 prefix sums. */
typedef struct rsb_bert rsb_bert_t;
const char* rsb_bert_last_error(void);
int rsb_bert_create(int hidden, int layers, int heads, int intermediate, int vocab, int max_pos, int type_vocab,
                    float ln_eps, rsb_bert_t** out);
/* A T5 encoder behind the same handle: the transformer of a sentence-transformers model such as GTR-T5
 * (`SentenceTransformer(name).encode(...)`, src/search.py:49-61 and :244-246, src/embed.py:25-40 and :130).  HF
 * T5EncoderModel in fp16: d_model 768, 12 heads of 64 (d_kv 64), feed_forward_proj "relu" with d_ff % 128 == 0, any
 * layer count, vocabulary and bucket count; anything else is RSB_ERR_UNSUPPORTED.  max_distance is the config's
 * relative_attention_max_distance: the buckets themselves are uploaded as a table (rsb_bert_load).  The clamp of HF
 * T5Block in fp16 is restated with the condition taken over the real tokens of the batch (HF's covers pad positions
 * too).  Free with rsb_bert_free. */
int rsb_t5_create(int layers, int d_ff, int vocab, int num_buckets, int max_distance, float eps, rsb_bert_t** out);
/* A RoBERTa encoder behind the same handle: HF RobertaModel as `AutoModel.from_pretrained(name)` builds it for the
 * DRAGON-RoBERTa query and context encoders, with the CLS row taken (src/search.py:241-243 and :93-94, src/embed.py:
 * 123-126 and :74-78).  BERT-base layers (hidden 768, 12 heads, erf GELU; intermediate % 128 == 0, RSB_ERR_UNSUPPORTED
 * otherwise) with RoBERTa's positions: a token with id padding_idx gets position padding_idx, every other token
 * padding_idx + the number of ids != padding_idx from the start of its sequence up to and including itself
 * (modeling_roberta.py create_position_ids_from_input_ids), so a pad id inside a sequence is not counted.
 * padding_idx must leave at least one position below max_pos (RSB_ERR_INVALID); type_vocab 1 or 2
 * (RSB_ERR_UNSUPPORTED otherwise).  The handle then takes rsb_bert_load with HF RobertaModel keys, which are
 * BertModel's ("embeddings.token_type_embeddings.weight" is [type_vocab, 768]; pooler.* is not loaded), and runs
 * rsb_bert_forward / rsb_bert_attention.  rsb_bert_forward on it returns RSB_ERR_UNSUPPORTED before any launch when
 * padding_idx + max_seqlen >= max_pos (a position would pass the table; with roberta-base's 514 rows and padding_idx 1
 * every sequence of <= 512 tokens fits), and RSB_ERR_INVALID when token_type_ids_dev holds a value outside
 * [0, type_vocab) (it reads them back to the host to check; NULL means all zero).  Free with rsb_bert_free. */
int rsb_roberta_create(int layers, int intermediate, int vocab, int max_pos, int type_vocab, float ln_eps,
                       int padding_idx, rsb_bert_t** out);
int rsb_bert_free(rsb_bert_t* h);
/* name = HF BertModel state_dict key (e.g. "encoder.layer.3.attention.self.query.weight"); data fp16, copied.
 * T5 handles take HF T5EncoderModel keys instead: "shared.weight" or "encoder.embed_tokens.weight" (tied),
 * "encoder.block.N.layer.0.SelfAttention.{q,k,v,o}.weight", "encoder.block.N.layer.{0,1}.layer_norm.weight",
 * "encoder.block.N.layer.1.DenseReluDense.{wi,wo}.weight", "encoder.final_layer_norm.weight",
 * "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight" ([num_buckets, 12], serves every layer) and
 * "relative_position_bucket": int32 [1023], the bucket of relative position r = key - query = -511..511 at index
 * r + 511, from HF's `_relative_position_bucket` (bidirectional) on the host; every entry must lie in
 * [0, num_buckets) (RSB_ERR_INVALID otherwise).  Both architectures take the sentence-transformers Dense head
 * "dense.weight" [768, 768] and "dense.bias" [768] (zero unless loaded). */
int rsb_bert_load(rsb_bert_t* h, const char* name, const void* f16_dev, int64_t n_elements, rsb_stream_t stream);
size_t rsb_bert_workspace_bytes(rsb_bert_t* h, int total_tokens);
/* pooling: RSB_POOL_MEAN (0) = mean over tokens (Contriever), RSB_POOL_CLS (1) = CLS row, optionally OR-ed with the
 * sentence-transformers head bits: RSB_POOL_DENSE (fp16 Linear 768 -> 768 on the pooled rows; RSB_ERR_STATE if
 * dense.weight was not loaded) and RSB_POOL_NORMALIZE (x / max(||x||_2, 1e-12), after the Dense layer).  A T5 handle
 * returns RSB_ERR_STATE until both of its bias tables are loaded.  out_f16_dev [B, 768] fp16.
 * Diagnostic, not used on the product path: RSB_POOL_TOKENS (alone; with any other bit RSB_ERR_INVALID) skips the
 * pooling and writes the final hidden states [T, 768] fp16 to out_f16_dev (BERT: after the last LayerNorm; T5: after
 * final_layer_norm), so that tests can compare every token row with a reference. */
enum { RSB_POOL_MEAN = 0, RSB_POOL_CLS = 1, RSB_POOL_DENSE = 2, RSB_POOL_NORMALIZE = 4, RSB_POOL_TOKENS = 8 };
int rsb_bert_forward(rsb_bert_t* h, const int32_t* input_ids_dev, const int32_t* token_type_ids_dev,
                     const int32_t* cu_seqlens_dev, int B, int T, int max_seqlen, int pooling, void* out_f16_dev,
                     void* ws_dev, size_t ws_bytes, rsb_stream_t stream);
int64_t rsb_bert_launches(rsb_bert_t* h);
/* Diagnostic, not used on the product path: one attention step of rsb_bert_forward on a caller's tensors, through
 * the forward's own dispatch (the list of sequences longer than 32 tokens, the flash kernel on the handle's side
 * stream, the kernel for sequences of <= 32 tokens on `stream`, the join).  qkv_dev [T, 2304] fp16 holds each token's
 * Q | K | V (12 heads of 64 each), ctx_dev [T, 768] fp16 receives softmax(scores) V per sequence and head; rows of
 * zero-length sequences and rows past cu_seqlens[B] are not written.  BERT handles score q.k / 8; T5 handles score
 * fp16(fp16(q.k) + bias[key - query]) from the loaded bias tables (RSB_ERR_STATE until both are loaded).
 * max_seqlen > 512 or above the handle's max_pos: RSB_ERR_UNSUPPORTED. */
int rsb_bert_attention(rsb_bert_t* h, const void* qkv_dev, const int32_t* cu_seqlens_dev, int B, int T, int max_seqlen,
                       void* ctx_dev, rsb_stream_t stream);
/* the encoder's tensor-core GEMM on its own: C[M,N] = A[M,K] . W[N,K]^T + bias (epilogue 0), GELU (1),
 * + residual (2) or ReLU (3); all fp16 row-major device pointers, N % 128 == 0, K % 64 == 0.  OR-ing
 * RSB_GEMM_REVERSED into the epilogue visits the 128-row tiles last-to-first, the order of the forward's FFN2.
 * C_dev may be residual_dev itself (the residual add in place, as the reader's o_proj and down_proj run it): each
 * element's residual is loaded by the thread that stores that element, before the store.  A_dev and W_dev must not
 * overlap C_dev. */
enum { RSB_GEMM_REVERSED = 256 };
int rsb_gemm_f16(const void* A_dev, const void* W_dev, const void* bias_dev, const void* residual_dev, void* C_dev,
                 int M, int N, int K, int epilogue, rsb_stream_t stream);

/* ---- reader LM for perplexity evaluation: HF causal LMs, prefill only, fp16 or bf16 ---------------------------------
 * Replaces the reader of the reference's perplexity loop (src/evaluate_perplexity.py:98-108 loads it, :126-134 runs
 * `lm(input_ids, labels=labels)` one window at a time).  Errors of these entries are reported by rsb_llm_last_error().
 * rsb_llm_create makes a reader of one family.  Every refusal below comes before any CUDA call, and the error names the
 * field.  For every family: family not one of RSB_LLM_*, or dtype neither RSB_DTYPE_F16 nor RSB_DTYPE_BF16,
 * RSB_ERR_INVALID; non-positive layers, vocab, max_pos, rope_theta or eps, or tied not 0 / 1, RSB_ERR_INVALID; clip_qkv
 * negative, infinite or NaN, or non-zero for any family but RSB_LLM_OLMO, RSB_ERR_INVALID; intermediate % 128 != 0
 * RSB_ERR_UNSUPPORTED.  Any vocabulary size: the LM head is padded to a multiple of 128 rows that never enter the
 * log-sum-exp.  tied = 1 (tie_word_embeddings): the LM head is the embedding; an untied "lm_head.weight" is accepted
 * and ignored.  inv_freq = 1 / rope_theta ** (2i / rotary_dims) in fp32.
 *   RSB_LLM_LLAMA, HF LlamaForCausalLM: head_dim 128 (hidden == 128 * heads), heads % kv_heads == 0 (else
 *     RSB_ERR_UNSUPPORTED), rotary_dims = 128 (else RSB_ERR_INVALID), eps = rms_norm_eps.  SiLU MLP, no biases,
 *     LlamaRMSNorm, default RoPE.  Weights: "model.embed_tokens.weight", "model.norm.weight", "lm_head.weight" and
 *     "model.layers.N.{self_attn.{q,k,v,o}_proj, mlp.{gate,up,down}_proj, input_layernorm,
 *     post_attention_layernorm}.weight".
 *   RSB_LLM_NEOX, HF GPTNeoXForCausalLM (Pythia): kv_heads == heads and tied = 0 (else RSB_ERR_UNSUPPORTED); hidden,
 *     heads and intermediate positive (else RSB_ERR_INVALID); head_dim = hidden / heads in {64, 80, 128, 256} (else
 *     RSB_ERR_UNSUPPORTED naming head_dim); hidden <= 8192 (the LayerNorm kernel's widest row, else RSB_ERR_UNSUPPORTED
 *     naming hidden; Pythia-12B has 5120); rotary_dims = HF's rotary_ndims, even and in [2, head_dim] (rotary_dims <= 0
 *     or > head_dim RSB_ERR_INVALID, odd RSB_ERR_UNSUPPORTED); rope_theta = rotary_emb_base, eps = layer_norm_eps.
 *     The forward is HF's: LayerNorm (fp32 mean and biased variance, one rounding) with bias, query_key_value with
 *     bias, partial rotary on dims [0, rotary_dims) of each Q / K head, causal attention scaled by head_dim^-0.5, dense
 *     with bias, dense_h_to_4h -> GELU -> dense_4h_to_h with biases, the parallel residual x = fp16(fp16(mlp(ln2(x)) +
 *     attn(ln1(x))) + x), final_layer_norm and a bias-free embed_out.  Weights: "gpt_neox.embed_in.weight",
 *     "embed_out.weight", "gpt_neox.final_layer_norm.{weight,bias}" and "gpt_neox.layers.N.{input_layernorm,
 *     post_attention_layernorm, attention.query_key_value, attention.dense, mlp.dense_h_to_4h,
 *     mlp.dense_4h_to_h}.{weight,bias}".  query_key_value's per-head interleaved rows (q_h | k_h | v_h for each head h)
 *     are stored as [Q heads | K heads | V heads].
 *   RSB_LLM_OLMO (HF OlmoForCausalLM: OLMo-1B/7B-hf, OLMo-1.7) and RSB_LLM_OLMO2 (Olmo2ForCausalLM): the Llama rules
 *     (head_dim 128, heads % kv_heads == 0, rotary_dims = 128), and OLMo with hidden > 8192 (the LayerNorm kernel's
 *     widest row) RSB_ERR_UNSUPPORTED.  The forward is a Llama layer (SwiGLU, no biases, causal GQA attention scaled by
 *     128^-0.5) except:
 *     RoPE keeps cos / sin in fp32: x * cos + rotate_half(x) * sin is evaluated in fp32 and rounded to half once;
 *     OLMo: both pre-norms and the final norm are OlmoLayerNorm, without weight or bias: fp16 of the fp32 (x - mean) *
 *       rsqrt(biased var + eps), one rounding; eps is 1e-5 in HF (no config field).  clip_qkv > 0 clamps every q, k and
 *       v projection element to [-clip_qkv, clip_qkv] before RoPE; 0 = none (HF clip_qkv null);
 *     OLMo-2: no pre-norms.  x = fp16(x + post_attention_layernorm(o_proj(attn(x)))), then x = fp16(x +
 *       post_feedforward_layernorm(mlp(x))).  Every norm is Olmo2RMSNorm, fp16(w * (x * rsqrt(mean(x^2) + eps))) with the
 *       weight multiply in fp32 and one rounding; q_norm normalises the whole q projection (hidden wide) and k_norm the
 *       whole k projection (kv_heads * 128 wide), before RoPE; the final model.norm is one too.  eps = rms_norm_eps.
 *     Weights: "model.embed_tokens.weight", "lm_head.weight" and "model.layers.N.{self_attn.{q,k,v,o}_proj,
 *     mlp.{gate,up,down}_proj}.weight"; OLMo-2 also "model.norm.weight" and "model.layers.N.{self_attn.q_norm,
 *     self_attn.k_norm, post_attention_layernorm, post_feedforward_layernorm}.weight".  OLMo has no norm weights: a
 *     norm name is an unknown weight (RSB_ERR_INVALID).
 * dtype is the element type of the handle's weights and activations: RSB_DTYPE_F16, or RSB_DTYPE_BF16, the reference's
 * reader dtype.  In bf16 the forward is HF's bf16 forward: every point where the fp16 forward rounds to fp16 (each GEMM
 * output, norm output, RoPE product and sum, attention's P before P V, SwiGLU / GELU output, residual add, the logits)
 * rounds to bf16 instead, with the same fp32 arithmetic in between; OLMo's fp32 cos / sin RoPE rounds once, to bf16, and
 * clip_qkv acts as the bf16 clamp (the clamped value is the bound rounded to bf16).  The NLL is the fp32 log-sum-exp of
 * the bf16 logits, as transformers' logits.float() after a bf16 lm_head.  rsb_llm_load, rsb_llm_attention and
 * rsb_llm_hidden_states take and return the handle's dtype. */
typedef struct rsb_llm rsb_llm_t;
enum { RSB_LLM_LLAMA = 0, RSB_LLM_NEOX = 1, RSB_LLM_OLMO = 2, RSB_LLM_OLMO2 = 3 };
const char* rsb_llm_last_error(void);
int rsb_llm_create(int family, int dtype, int layers, int hidden, int heads, int kv_heads, int intermediate, int vocab,
                   int max_pos, int rotary_dims, float rope_theta, float eps, float clip_qkv, int tied, rsb_llm_t** out);
/* name = an HF state-dict key of the handle's family (above), data on the device in the handle's dtype, copied; any
 * other name RSB_ERR_INVALID ("unknown weight name"). */
int rsb_llm_load(rsb_llm_t* h, const char* name, const void* f16_dev, int64_t n_elements, rsb_stream_t stream);
size_t rsb_llm_workspace_bytes(rsb_llm_t* h, int total_tokens, int label_tokens);
/* B packed sequences: ids_dev / labels_dev [T] int32 (label -100 = ignored), cu_seqlens_dev [B+1] int32 (0 .. T), every
 * sequence <= max_seqlen <= max_pos tokens (RSB_ERR_UNSUPPORTED past max_pos).  Positions restart at 0 in every
 * sequence.  nll_out_dev [T] fp32: at position t that is not the first of its sequence and whose label is not -100,
 * logsumexp(logits of t - 1) - logit[labels[t]] (HF's shifted causal-LM loss per token), 0 elsewhere.  label_tokens of
 * rsb_llm_workspace_bytes counts those positions.  Ids outside [0, vocab), labels that are neither -100 nor an id and
 * malformed offsets are RSB_ERR_INVALID before any launch; RSB_ERR_STATE until every weight is loaded. */
int rsb_llm_nll(rsb_llm_t* h, const int32_t* ids_dev, const int32_t* cu_seqlens_dev, int B, int T, int max_seqlen,
                const int32_t* labels_dev, float* nll_out_dev, void* ws_dev, size_t ws_bytes, rsb_stream_t stream);
int rsb_llm_free(rsb_llm_t* h);
/* Diagnostic, not used on the product path: one attention step of rsb_llm_nll on a caller's tensors, with the forward's
 * own work list.  qkv_dev [T, (heads + 2 kv_heads) head_dim] in the handle's dtype (fp16 or bf16) holds each token's
 * Q | K | V heads (GPT-NeoX: the permuted [Q heads | K heads | V heads] layout rsb_llm_load stores); RoPE is applied to
 * its Q and K heads in place (positions restart at 0 in every window; GPT-NeoX rotates the first rotary_dims of each
 * head and leaves the other dims bit-identical), then ctx_dev [T, heads head_dim] in the same dtype receives causal
 * softmax(q k^T / sqrt(head_dim)) v per window and query head h, which reads KV head h / (heads / kv_heads).  OLMo and
 * OLMo-2 run layer 0's prologue in place of RoPE: the clip_qkv clamp of q, k and v (OLMo), or q_norm / k_norm (OLMo-2;
 * RSB_ERR_STATE until layer 0's q_norm and k_norm are loaded), then the fp32-cos / sin RoPE.  Windows may be empty and
 * cu_seqlens_dev [B+1] may end below T: rows of empty windows and rows at or past cu_seqlens[B] are neither rotated nor
 * written.  The offset refusals of rsb_llm_nll apply (RSB_ERR_INVALID / RSB_ERR_UNSUPPORTED before any launch); no
 * other weight needs to be loaded. */
int rsb_llm_attention(rsb_llm_t* h, void* qkv_dev, const int32_t* cu_seqlens_dev, int B, int T, int max_seqlen,
                      void* ctx_dev, rsb_stream_t stream);
/* Diagnostic, not used on the product path: the residual stream after the last decoder layer of rsb_llm_nll's forward,
 * before the final norm, out_dev [T, hidden] in the handle's dtype.  The refusals of rsb_llm_nll apply; the workspace is
 * rsb_llm_workspace_bytes(h, T, 0). */
int rsb_llm_hidden_states(rsb_llm_t* h, const int32_t* ids_dev, const int32_t* cu_seqlens_dev, int B, int T,
                          int max_seqlen, void* out_dev, void* ws_dev, size_t ws_bytes, rsb_stream_t stream);
/* Diagnostic, not used on the product path: the GPT-NeoX LayerNorm step of rsb_llm_nll's forward on a caller's fp16 rows
 * of `hidden` elements.  Output row i reads input row r = rows_dev ? rows_dev[i] : i of x_dev, i < n_rows.
 *   add_dev != NULL: first x[r] = fp16(x[r] + add[r]) (the parallel residual's last sum), written back to x_dev.
 *   w1_dev != NULL: out1[i] = fp16((x[r] - mean) * rsqrt(var + eps) * w1 + b1), mean and biased variance in fp32, one
 *   rounding (torch's fp16 LayerNorm); w2_dev != NULL (only with w1_dev): out2[i] likewise with w2 / b2, from the same
 *   statistics.  Neither: only the add.
 * hidden must be a multiple of 8 and at most 8192 (RSB_ERR_UNSUPPORTED, also the largest GPT-NeoX hidden rsb_llm_create
 * accepts); a missing bias or output RSB_ERR_INVALID; both before any launch.  No handle is needed. */
int rsb_llm_layernorm(int hidden, float eps, void* x_dev, const void* add_dev, const int32_t* rows_dev, int n_rows,
                      const void* w1_dev, const void* b1_dev, const void* w2_dev, const void* b2_dev, void* out1_dev,
                      void* out2_dev, rsb_stream_t stream);
/* Diagnostic, not used on the product path: the OLMo-2 norm step of rsb_llm_nll's forward on a caller's fp16 rows of
 * `hidden` elements, with Olmo2RMSNorm norm(v) = fp16(w * (v * rsqrt(mean(v^2) + eps))) (fp32 statistics, the weight
 * multiply in fp32, one rounding).  Row i reads row r = rows_dev ? rows_dev[i] : i, i < n_rows.
 *   a_dev != NULL: x[r] = fp16(x[r] + norm(a[r])) in place (the post-norm residual add); out_dev is not written.
 *   a_dev == NULL: out[i] = norm(x[r]) (the final norm); x_dev is read only.
 * A null x_dev or w_dev, or a null out_dev without a_dev, RSB_ERR_INVALID; hidden not a positive multiple of 8
 * RSB_ERR_UNSUPPORTED; both before any launch.  No handle is needed. (OLMo's LayerNorm is rsb_llm_layernorm with unit
 * w1 and zero b1.) */
int rsb_llm_olmo2_norm(int hidden, float eps, void* x_dev, const void* a_dev, const int32_t* rows_dev, int n_rows,
                       const void* w_dev, void* out_dev, rsb_stream_t stream);

/* ---- MinHash de-duplication of retrieved passages ----------------------------------------------------------------
 * Replaces utils/deduplication.py's `remove_duplicates_with_minhash` (datasketch MinHash(num_perm=128) and
 * MinHashLSH(threshold=0.8)) run by src/search.py:471-479 on the merged multi-source results.  Errors of these entries
 * are reported by rsb_dedup_last_error().
 * rsb_minhash_signatures: texts are the UTF-8 slices text_dev[text_off_dev[t] .. text_off_dev[t+1]) of one buffer of
 * total_bytes < 2^31 bytes, each valid UTF-8 on its own.  Words are split on the code points of Python's str.isspace()
 * (`text.split()`); shingle i of a text is words i..i+12 joined by single spaces, hashed as datasketch's sha1_hash32
 * (first 4 bytes of SHA-1, little-endian).  sig_dev [n_texts, 128] uint32 receives, per permutation j, the minimum over
 * the shingles of ((h * a_j + b_j) mod 2^64) mod (2^61 - 1) & 0xffffffff (2^32 - 1 without shingles); perm_a_dev /
 * perm_b_dev uint64 [128] are MinHash.permutations.  n_words_dev [n_texts] int32 receives the word counts.  ws_dev holds
 * rsb_minhash_workspace_bytes(total_bytes) bytes. */
const char* rsb_dedup_last_error(void);
size_t rsb_minhash_workspace_bytes(int64_t total_bytes);
int rsb_minhash_signatures(const uint8_t* text_dev, const int64_t* text_off_dev, int n_texts, int64_t total_bytes,
                           const uint64_t* perm_a_dev, const uint64_t* perm_b_dev, uint32_t* sig_dev, int32_t* n_words_dev,
                           void* ws_dev, size_t ws_bytes, rsb_stream_t stream);
/* rsb_minhash_dedup: the slots of group g are rows group_off_dev[g] .. group_off_dev[g+1]) of sig_dev [*, 128] (16-byte
 * aligned) and n_words_dev.  keep_dev[s] = 1 unless slot s has fewer than 13 words, or some earlier slot of its group
 * shares all `rows` values of one of the `bands` bands [k * rows, (k + 1) * rows) with it and more than max_equal of
 * the 128 values (MinHashLSH candidate with jaccard > threshold; 0.8 -> bands 9, rows 13, max_equal 102).
 * bands * rows <= 128. */
int rsb_minhash_dedup(const uint32_t* sig_dev, const int32_t* n_words_dev, const int32_t* group_off_dev, int n_groups,
                      int bands, int rows, int max_equal, uint8_t* keep_dev, rsb_stream_t stream);
/* host function, no GPU: mask[q] = 1 iff byte q of the valid UTF-8 bytes[0, n) belongs to a character on which the
 * signatures' word split splits (lets host-side tests pin the whitespace set against Python's str.isspace()) */
int rsb_utf8_space_mask(const uint8_t* bytes, int64_t n, uint8_t* mask);

/* ---- BM25 search (the reference's sparse retriever) ----------------------------------------------------------------
 * Replaces src/search.py:763-807's pyserini LuceneSearcher.search (Lucene 9 BM25Similarity, k1 = 0.9, b = 0.4) over
 * a term-major posting index; retrieval_scaling_b200/bm25.py builds the index and analyzes the queries.  Stateless:
 * the caller owns every array.  Errors of these entries are reported by rsb_bm25_last_error().
 * rsb_bm25_search: the postings of term t are post_dev[term_off_dev[t] .. term_off_dev[t+1]), each an 8-byte pair
 * (int32 document number, fp32 x = 1f + (float) tf * cache[norm(doc)]) sorted by document, post_dev 8-byte aligned.
 * Query q's clauses are q_off_dev[q] .. q_off_dev[q+1]) of q_term_dev (term ids, strictly ascending, each < the number
 * of terms) and q_w_dev (fp32 clause weights count * idf).  Score of document d = the fp32 sum, in ascending term id,
 * of w - w / x over the clauses whose term has a posting for d, each operation rounded on its own.  D_dev [nq, k]
 * fp32 and I_dev [nq, k] int64 receive the hits (score > 0) best first, ties to the lower document number, then
 * -FLT_MAX and -1.  ws_dev holds rsb_bm25_workspace_bytes(n_docs, nq, k) bytes.  n_docs < 2^31; k > 4096
 * RSB_ERR_UNSUPPORTED; both before any launch.  q_term_dev / q_w_dev may be null when no query has a clause, and
 * post_dev when no term has a posting (zero-length arrays); term_off_dev and q_off_dev are always read. */
const char* rsb_bm25_last_error(void);
size_t rsb_bm25_workspace_bytes(int64_t n_docs, int nq, int k);
int rsb_bm25_search(const int64_t* term_off_dev, const int32_t* post_dev, int64_t n_docs, const int32_t* q_off_dev,
                    const int32_t* q_term_dev, const float* q_w_dev, int nq, int k, float* D_dev, int64_t* I_dev,
                    void* ws_dev, size_t ws_bytes, rsb_stream_t stream);

/* diagnostic: shared-window address at which dynamic shared memory starts (the scan kernel folds it into LDS) */
int rsb_debug_smem_base(void);
/* diagnostic: the fp32 look-up tables an IVFPQ search builds for queries q_dev [nq, d], as the scan reads them:
 * lut_dev [nq, rsb_pq_lut_floats(h)], entry (j, b) of byte sub-quantizer b at rsb_pq_lut_index(Mb, j, b) (Mb = M * nbits
 * / 8; with nbits = 4 the entry is the pair sum T[2b][j & 15] + T[2b+1][j >> 4]).  rsb_pq_lut_floats: -1 if h is not
 * IVFPQ. */
int rsb_pq_lut_floats(rsb_index_t* h);
int rsb_pq_tables(rsb_index_t* h, const float* q_dev, int nq, float* lut_dev, rsb_stream_t stream);

/* ---- layout self-description (lets host-side tests pin the interleaved PQ layout without a GPU) ------- */
/* M here counts code bytes per vector (M * nbits / 8; with 4-bit codes, byte b holds sub-quantizers 2b and 2b+1) */
/* byte offset, inside a 32-vector block of M*32 bytes, of sub-quantizer m of block-local vector v */
int rsb_pq_layout_offset(int M, int v, int m);
/* float index, inside one 256x64 look-up-table row block, where entry (j, m) lives (first replica) */
int rsb_pq_lut_index(int M, int j, int m);

#ifdef __cplusplus
}
#endif
#endif /* RSB_H_ */
