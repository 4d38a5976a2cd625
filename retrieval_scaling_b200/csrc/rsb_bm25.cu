// rsb_bm25.cu -- BM25 top-k over a term-major posting index (the reference's pyserini LuceneSearcher.search with
// Lucene 9 BM25Similarity, k1 = 0.9, b = 0.4), term at a time:
//   bm25_tile_kernel         one CTA per (document tile, query): fp32 accumulators for BM25_TILE documents in shared
//                            memory; for each query term in ascending term id, the term's postings inside the tile add
//                            w - w / x to their document's accumulator; then the tile's top min(k, hits) documents
//                            with score > 0 as one item's key list
//   merge_items_flat_kernel  (rsb_dense.cu) merges the tiles of a query, tiles as items, in document order
// A term has at most one posting per document, so the threads of a term never write the same accumulator: no atomics,
// and every document's sum runs in the same order (ascending term id), whatever the launch: the result is
// deterministic.
#include "../../include/rsb.h"
#include "rsb_common.cuh"
#include "rsb_internal.h"

#include <cfloat>
#include <cstdarg>
#include <cstdio>
#include <string>

using namespace rsb;

static thread_local std::string g_bmerr;
static int bfail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_bmerr = buf;
    return code;
}
#define BCU(expr)                                                                                                   \
    do {                                                                                                            \
        cudaError_t e__ = (expr);                                                                                   \
        if (e__ != cudaSuccess)                                                                                     \
            return bfail(e__ == cudaErrorMemoryAllocation ? RSB_ERR_OOM : RSB_ERR_CUDA, "%s: %s (%s:%d)", #expr,    \
                         cudaGetErrorString(e__), __FILE__, __LINE__);                                              \
    } while (0)

extern "C" const char* rsb_bm25_last_error(void) { return g_bmerr.c_str(); }

namespace {

constexpr int BM25_THREADS = 512;
constexpr int BM25_TILE = 16384;      // documents per CTA: 64 KB of fp32 accumulators
constexpr int BM25_TERMS = 256;       // query terms whose tile bounds are resolved at once
constexpr int BM25_MAX_K = 4096;      // the select limit of the other searches

__host__ __device__ __forceinline__ int tile_k(int k) { return k < BM25_TILE ? k : BM25_TILE; }
__host__ __device__ __forceinline__ int tile_cap(int k) { return next_pow2(tile_k(k) + BM25_THREADS); }

size_t tile_smem(int k) {
    const size_t bounds = (size_t)BM25_TERMS * (sizeof(int64_t) + sizeof(int) + sizeof(float));
    const size_t keys = (size_t)tile_cap(k) * sizeof(u64);
    return (size_t)BM25_TILE * sizeof(float) + (bounds > keys ? bounds : keys);
}

// first position in post[lo, hi) whose document is >= doc (the postings of a term are sorted by document)
__device__ __forceinline__ int64_t lower_doc(const int2* __restrict__ post, int64_t lo, int64_t hi, int doc) {
    while (lo < hi) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(&post[mid].x) < doc) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// One posting: acc[doc] += w - w / x, each operation rounded on its own (Lucene's float arithmetic, no fma).
__device__ __forceinline__ void add_posting(float* acc, int2 v, int d0, float w) {
    float& a = acc[v.x - d0];
    a = __fadd_rn(a, __fsub_rn(w, __fdiv_rn(w, __int_as_float(v.y))));
}

// blockIdx.x = tile * nq + q: the CTAs resident at one time score the same tile for different queries, so the
// postings of the terms the queries share are read from HBM once and from L2 after that.
__global__ void __launch_bounds__(BM25_THREADS) bm25_tile_kernel(
    const int64_t* __restrict__ term_off, const int2* __restrict__ post, int n_docs, const int* __restrict__ q_off,
    const int* __restrict__ q_term, const float* __restrict__ q_w, int nq, int ntiles, int k_tile, int cap,
    u64* __restrict__ out_keys, int* __restrict__ out_cnt) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float* acc = reinterpret_cast<float*>(smem_raw);                          // [BM25_TILE]
    unsigned char* scratch = smem_raw + (size_t)BM25_TILE * sizeof(float);
    int64_t* s_lo = reinterpret_cast<int64_t*>(scratch);                       // scoring: [BM25_TERMS] bounds, ...
    int* s_n = reinterpret_cast<int*>(s_lo + BM25_TERMS);
    float* s_w = reinterpret_cast<float*>(s_n + BM25_TERMS);
    u64* keys = reinterpret_cast<u64*>(scratch);                               // selection: [cap] (same bytes)
    __shared__ int s_count;
    const int tid = threadIdx.x;
    const int q = blockIdx.x % nq, tile = blockIdx.x / nq;
    const int d0 = tile * BM25_TILE, nd = min(BM25_TILE, n_docs - d0);
    for (int i = tid; i < BM25_TILE; i += BM25_THREADS) acc[i] = 0.f;
    const int t0 = q_off[q], nt = q_off[q + 1] - t0;

    for (int c0 = 0; c0 < nt; c0 += BM25_TERMS) {
        const int nc = min(BM25_TERMS, nt - c0);
        __syncthreads();                          // the previous chunk's bounds are consumed (first: acc is zeroed)
        if (tid < nc) {
            const int t = q_term[t0 + c0 + tid];
            const int64_t b = term_off[t], e = term_off[t + 1];
            const int64_t lo = lower_doc(post, b, e, d0);
            s_lo[tid] = lo;
            s_n[tid] = (int)(lower_doc(post, lo, e, d0 + nd) - lo);
            s_w[tid] = q_w[t0 + c0 + tid];
        }
        __syncthreads();
        for (int j = 0; j < nc; ++j) {
            const int n = s_n[j];
            if (n == 0) continue;                 // block-uniform: a term without postings here writes nothing
            const int2* p = post + s_lo[j];
            const float w = s_w[j];
            int i = tid;
            for (; i + 3 * BM25_THREADS < n; i += 4 * BM25_THREADS) {      // four loads in flight per thread
                const int2 v0 = __ldg(p + i), v1 = __ldg(p + i + BM25_THREADS);
                const int2 v2 = __ldg(p + i + 2 * BM25_THREADS), v3 = __ldg(p + i + 3 * BM25_THREADS);
                add_posting(acc, v0, d0, w);
                add_posting(acc, v1, d0, w);
                add_posting(acc, v2, d0, w);
                add_posting(acc, v3, d0, w);
            }
            for (; i < n; i += BM25_THREADS) add_posting(acc, __ldg(p + i), d0, w);
            __syncthreads();                      // the next term may add to the same documents from other threads
        }
    }

    // the tile's top k_tile documents with score > 0, ties to the lower document (make_key's slot order)
    __syncthreads();                              // every thread is past its last read of s_lo / s_n / s_w
    if (tid == 0) s_count = 0;
    __syncthreads();
    unsigned tau = 0u;
    for (int i0 = 0; i0 < nd; i0 += BM25_THREADS) {
        const int i = i0 + tid;
        const float s = i < nd ? acc[i] : 0.f;
        const unsigned o = ord_f32(s);
        warp_append(keys, &s_count, s > 0.f && o > tau, make_key(o, (unsigned)(d0 + i)));
        tau = block_maybe_compact(keys, &s_count, k_tile, cap, BM25_THREADS, tau);
    }
    block_compact(keys, &s_count, k_tile, cap, tau);
    const int n = min(s_count, k_tile);
    const size_t item = (size_t)q * ntiles + tile;
    for (int i = tid; i < n; i += BM25_THREADS) out_keys[item * k_tile + i] = keys[i];
    if (tid == 0) out_cnt[item] = n;
}

int64_t num_tiles(int64_t n_docs) { return (n_docs + BM25_TILE - 1) / BM25_TILE; }

}  // namespace

extern "C" size_t rsb_bm25_workspace_bytes(int64_t n_docs, int nq, int k) {
    if (n_docs < 0 || nq < 0 || k < 1) return 0;
    return (size_t)nq * (size_t)num_tiles(n_docs) * ((size_t)tile_k(k) * sizeof(u64) + sizeof(int));
}

extern "C" int rsb_bm25_search(const int64_t* term_off_dev, const int32_t* post_dev, int64_t n_docs,
                               const int32_t* q_off_dev, const int32_t* q_term_dev, const float* q_w_dev, int nq, int k,
                               float* D_dev, int64_t* I_dev, void* ws_dev, size_t ws_bytes, rsb_stream_t stream) {
    if (n_docs < 0 || n_docs >= ((int64_t)1 << 31) || nq < 0)
        return bfail(RSB_ERR_INVALID, "bad shape n_docs=%lld nq=%d (fewer than 2^31 documents)", (long long)n_docs, nq);
    if (k < 1) return bfail(RSB_ERR_INVALID, "k=%d: k must be positive", k);
    if (k > BM25_MAX_K) return bfail(RSB_ERR_UNSUPPORTED, "k=%d: at most %d results per query", k, BM25_MAX_K);
    const int64_t ntiles = num_tiles(n_docs);
    if (ntiles * nq >= ((int64_t)1 << 31))
        return bfail(RSB_ERR_INVALID, "nq=%d x %lld document tiles: fewer than 2^31 per call", nq, (long long)ntiles);
    if (nq == 0) return RSB_OK;
    // q_term / q_w are read only for clauses and post only inside a term's postings: a batch without clauses (every
    // query empty or unknown) passes zero-length, possibly null, arrays, and so does an index without postings
    if (!q_off_dev || !D_dev || !I_dev || (ntiles && (!term_off_dev || !ws_dev)))
        return bfail(RSB_ERR_INVALID, "null argument");
    if ((uintptr_t)post_dev & 7) return bfail(RSB_ERR_INVALID, "postings must be 8-byte aligned");
    const size_t need = rsb_bm25_workspace_bytes(n_docs, nq, k);
    if (ws_bytes < need) return bfail(RSB_ERR_OOM, "workspace too small: need %zu bytes, got %zu", need, ws_bytes);
    cudaStream_t st = (cudaStream_t)stream;
    const int kt = tile_k(k);
    u64* keys = static_cast<u64*>(ws_dev);
    int* cnt = reinterpret_cast<int*>(static_cast<unsigned char*>(ws_dev) + (size_t)nq * ntiles * kt * sizeof(u64));
    if (ntiles) {
        const size_t smem = tile_smem(k);
        static PerDeviceSize configured;
        if (configured.raise(smem))
            BCU(cudaFuncSetAttribute(bm25_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        bm25_tile_kernel<<<(unsigned)(ntiles * nq), BM25_THREADS, smem, st>>>(
            term_off_dev, reinterpret_cast<const int2*>(post_dev), (int)n_docs, q_off_dev, q_term_dev, q_w_dev, nq,
            (int)ntiles, kt, tile_cap(k), keys, cnt);
        BCU(cudaPeekAtLastError());
    }
    launch_merge_items(keys, cnt, nq, (int)ntiles, kt, k, nullptr, 0, D_dev, I_dev, st);
    BCU(cudaPeekAtLastError());
    return RSB_OK;
}
