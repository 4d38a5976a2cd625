// rsb_dedup.cu -- MinHash near-duplicate removal of retrieved passages (the reference's utils/deduplication.py over
// datasketch MinHash / MinHashLSH), for one batch of queries at a time:
//   minhash_split_hash_kernel   one block per text: word boundaries by Python's str.split() whitespace over UTF-8,
//                               then SHA-1 of every 13-word shingle "w_i w_i+1 ... w_i+12" (single spaces), read
//                               straight from the word byte ranges, first 4 digest bytes little-endian
//   minhash_signature_kernel    one block per text, one thread per permutation: min over the shingles of
//                               ((h * a + b) mod 2^64) mod (2^61 - 1) & 0xffffffff
//   minhash_dedup_kernel        one block per group (query): slot j is dropped when an earlier slot shares a whole
//                               LSH band with it and more than max_equal of the 128 values are equal, or when it has
//                               no shingle (fewer than 13 words)
#include "../../include/rsb.h"
#include "rsb_internal.h"

#include <cub/block/block_scan.cuh>

#include <cstdarg>
#include <cstdio>
#include <string>

using namespace rsb;

static thread_local std::string g_derr;
static int dfail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_derr = buf;
    return code;
}
#define DCU(expr)                                                                                                   \
    do {                                                                                                            \
        cudaError_t e__ = (expr);                                                                                   \
        if (e__ != cudaSuccess)                                                                                     \
            return dfail(e__ == cudaErrorMemoryAllocation ? RSB_ERR_OOM : RSB_ERR_CUDA, "%s: %s (%s:%d)", #expr,    \
                         cudaGetErrorString(e__), __FILE__, __LINE__);                                              \
    } while (0)

extern "C" const char* rsb_dedup_last_error(void) { return g_derr.c_str(); }

namespace {

constexpr int NPERM = 128;        // MinHash(num_perm=128)
constexpr int SHINGLE = 13;       // shingle_document(text, shingle_size=13)
constexpr int HT = 128;           // threads of the split / hash block
constexpr int DT = 256;           // threads (slots in flight) of the dedup block
constexpr int LEAD_TILE_WORDS = 8192;
constexpr u64 MERSENNE = (1ull << 61) - 1;

// Length in bytes of the whitespace character starting at p (0 if none): exactly the code points for which Python's
// str.isspace() holds, which is what str.split() without arguments splits on.  p holds `avail` valid UTF-8 bytes.
__host__ __device__ __forceinline__ int space_len(const uint8_t* p, int64_t avail) {
    const unsigned c = p[0];
    if (c < 0x80) return (c == 0x20 || (c >= 0x09 && c <= 0x0d) || (c >= 0x1c && c <= 0x1f)) ? 1 : 0;
    if (c == 0xc2) return (avail >= 2 && (p[1] == 0x85 || p[1] == 0xa0)) ? 2 : 0;       // U+0085, U+00A0
    if (avail < 3) return 0;
    const unsigned c1 = p[1], c2 = p[2];
    if (c == 0xe1) return (c1 == 0x9a && c2 == 0x80) ? 3 : 0;                            // U+1680
    if (c == 0xe2) {
        if (c1 == 0x80) return ((c2 >= 0x80 && c2 <= 0x8a) || c2 == 0xa8 || c2 == 0xa9 || c2 == 0xaf) ? 3 : 0;
        return (c1 == 0x81 && c2 == 0x9f) ? 3 : 0;                                       // U+2000-200A/2028/2029/202F, U+205F
    }
    if (c == 0xe3) return (c1 == 0x80 && c2 == 0x80) ? 3 : 0;                            // U+3000
    return 0;
}

// byte q of s[0, n) belongs to a whitespace character (one of at most 3 bytes, starting at q, q-1 or q-2)
__host__ __device__ __forceinline__ bool in_space(const uint8_t* s, int64_t n, int64_t q) {
    for (int k = 0; k < 3 && k <= q; ++k)
        if (space_len(s + q - k, n - (q - k)) > k) return true;
    return false;
}

__device__ __forceinline__ uint32_t rotl(uint32_t x, int k) { return __funnelshift_l(x, x, k); }

// one SHA-1 compression of the 16 big-endian words col[0], col[HT], ..., col[15 * HT]
__device__ __forceinline__ void sha1_block(uint32_t h[5], const uint32_t* col) {
    uint32_t w[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) w[k] = col[k * HT];
    uint32_t a = h[0], b = h[1], c = h[2], d = h[3], e = h[4];
#pragma unroll
    for (int i = 0; i < 80; ++i) {
        uint32_t wi;
        if (i < 16) {
            wi = w[i];
        } else {
            wi = rotl(w[(i - 3) & 15] ^ w[(i - 8) & 15] ^ w[(i - 14) & 15] ^ w[i & 15], 1);
            w[i & 15] = wi;
        }
        uint32_t f, k;
        if (i < 20)      { f = (b & c) | (~b & d);          k = 0x5A827999u; }
        else if (i < 40) { f = b ^ c ^ d;                   k = 0x6ED9EBA1u; }
        else if (i < 60) { f = (b & c) | (b & d) | (c & d); k = 0x8F1BBCDCu; }
        else             { f = b ^ c ^ d;                   k = 0xCA62C1D6u; }
        const uint32_t t = rotl(a, 5) + f + e + k + wi;
        e = d; d = c; c = rotl(b, 30); b = a; a = t;
    }
    h[0] += a; h[1] += b; h[2] += c; h[3] += d; h[4] += e;
}

__global__ void __launch_bounds__(HT) minhash_split_hash_kernel(const uint8_t* __restrict__ text,
                                                                const int64_t* __restrict__ text_off,
                                                                int32_t* __restrict__ word_start, int32_t* __restrict__ word_end,
                                                                uint32_t* __restrict__ shingle_hash, int32_t* __restrict__ n_words) {
    using Scan = cub::BlockScan<int, HT>;
    __shared__ typename Scan::TempStorage scan_tmp;
    __shared__ uint32_t msg[16 * HT];           // the current 64-byte block of every thread, word k of thread t at [k][t]
    const int t = blockIdx.x;
    const int64_t o0 = text_off[t], n = text_off[t + 1] - o0;
    const uint8_t* s = text + o0;
    int32_t* ws = word_start + o0;              // a text of n bytes has at most n words: its slices start at o0
    int32_t* we = word_end + o0;

    // 1. word boundaries: the k-th word start and the k-th word end of the text, by a block scan over 128-byte chunks
    int nstart = 0, nend = 0;
    for (int64_t c = 0; c < n; c += HT) {
        const int64_t q = c + threadIdx.x;
        int st = 0, en = 0;
        if (q < n && !in_space(s, n, q)) {
            st = q == 0 || in_space(s, n, q - 1);
            en = q == n - 1 || in_space(s, n, q + 1);
        }
        int excl, agg;
        Scan(scan_tmp).ExclusiveSum(st | (en << 16), excl, agg);
        if (st) ws[nstart + (excl & 0xffff)] = (int32_t)q;
        if (en) we[nend + (excl >> 16)] = (int32_t)q + 1;
        nstart += agg & 0xffff;
        nend += agg >> 16;
        __syncthreads();                        // scan_tmp is reused
    }
    if (threadIdx.x == 0) n_words[t] = nstart;

    // 2. SHA-1 of each shingle, the message built byte by byte from the word ranges, with the standard padding
    uint32_t* col = msg + threadIdx.x;
    for (int i = threadIdx.x; i + SHINGLE <= nstart; i += HT) {
        uint32_t msg_len = SHINGLE - 1;
#pragma unroll 1
        for (int w = 0; w < SHINGLE; ++w) msg_len += (uint32_t)(we[i + w] - ws[i + w]);
        const uint32_t total = ((msg_len + 8) / 64 + 1) * 64;     // 0x80, zeros, 8-byte bit length: a multiple of 64
        const u64 bits = (u64)msg_len * 8;
        uint32_t h[5] = {0x67452301u, 0xEFCDAB89u, 0x98BADCFEu, 0x10325476u, 0xC3D2E1F0u};
        int w = 0;
        int32_t q = ws[i], qe = we[i];
        uint32_t cur = 0;
#pragma unroll 1
        for (uint32_t pos = 0; pos < total; ++pos) {
            uint32_t byte;
            if (pos < msg_len) {
                if (q < qe) {
                    byte = __ldg(s + q++);
                } else {                        // end of word w: the joining space, then word w + 1
                    byte = ' ';
                    ++w;
                    q = ws[i + w];
                    qe = we[i + w];
                }
            } else if (pos == msg_len) {
                byte = 0x80;
            } else if (pos >= total - 8) {
                byte = (uint32_t)(bits >> (8 * (total - 1 - pos))) & 0xff;
            } else {
                byte = 0;
            }
            cur = (cur << 8) | byte;
            if ((pos & 3) == 3) {
                col[((pos >> 2) & 15) * HT] = cur;
                if ((pos & 63) == 63) sha1_block(h, col);
            }
        }
        shingle_hash[o0 + i] = __byte_perm(h[0], 0, 0x0123);     // digest bytes 0..3 read little-endian
    }
}

__global__ void __launch_bounds__(NPERM) minhash_signature_kernel(const int64_t* __restrict__ text_off,
                                                                  const int32_t* __restrict__ n_words,
                                                                  const uint32_t* __restrict__ shingle_hash,
                                                                  const u64* __restrict__ perm_a, const u64* __restrict__ perm_b,
                                                                  uint32_t* __restrict__ sig) {
    const int t = blockIdx.x, j = threadIdx.x;
    const u64 a = perm_a[j], b = perm_b[j];
    const int nsh = max(0, n_words[t] - (SHINGLE - 1));
    const uint32_t* hs = shingle_hash + text_off[t];
    uint32_t m = 0xffffffffu;
#pragma unroll 4
    for (int i = 0; i < nsh; ++i) {
        u64 x = (u64)hs[i] * a + b;                             // wraps mod 2^64, as numpy's uint64 product does
        x = (x & MERSENNE) + (x >> 61);                         // mod 2^61 - 1: at most 2^61 + 6 here
        if (x >= MERSENNE) x -= MERSENNE;
        m = min(m, (uint32_t)x);
    }
    sig[(int64_t)t * NPERM + j] = m;
}

// slot j of a group is a duplicate when some earlier slot i shares all `rows` values of some band with it (the
// MinHashLSH candidate test) and more than max_equal of the 128 values are equal (jaccard > threshold).  The first value
// of every band ("lead") of a tile of earlier slots sits in shared memory; a lead match is confirmed from global memory.
__global__ void __launch_bounds__(DT, 2) minhash_dedup_kernel(const uint32_t* __restrict__ sig, const int32_t* __restrict__ n_words,
                                                           const int32_t* __restrict__ group_off, int bands, int rows,
                                                           int max_equal, int tile, uint8_t* __restrict__ keep) {
    extern __shared__ uint32_t lead_smem[];
    uint32_t* lead = lead_smem;                 // [tile][bands]
    uint32_t* mine = lead_smem + tile * bands;  // [bands][DT]: the leads of this thread's slot
    const int s0 = group_off[blockIdx.x], n = group_off[blockIdx.x + 1] - s0;
    for (int jb = 0; jb < n; jb += DT) {
        const int j = jb + threadIdx.x;
        const bool live = j < n && n_words[s0 + j] >= SHINGLE;
        const uint32_t* sj = sig + (int64_t)(s0 + j) * NPERM;
        if (live)
            for (int k = 0; k < bands; ++k) mine[k * DT + threadIdx.x] = sj[k * rows];
        bool dup = false;
        const int jend = min(n, jb + DT);
        for (int i0 = 0; i0 < jend - 1; i0 += tile) {
            const int cnt = min(tile, jend - 1 - i0);
            __syncthreads();
            for (int e = threadIdx.x; e < cnt * bands; e += DT) {
                const int ii = e / bands, k = e - ii * bands;
                lead[e] = sig[(int64_t)(s0 + i0 + ii) * NPERM + k * rows];
            }
            __syncthreads();
            if (!live || dup) continue;
            const int iend = min(cnt, j - i0);
            for (int ii = 0; ii < iend && !dup; ++ii) {
                for (int k = 0; k < bands; ++k) {
                    if (lead[ii * bands + k] != mine[k * DT + threadIdx.x]) continue;
                    const uint32_t* si = sig + (int64_t)(s0 + i0 + ii) * NPERM;
                    bool band = true;
                    for (int rr = 1; rr < rows && band; ++rr) band = si[k * rows + rr] == sj[k * rows + rr];
                    if (!band) continue;
                    int eq = 0;
                    for (int p = 0; p < NPERM; p += 4) {
                        const uint4 x = *reinterpret_cast<const uint4*>(si + p);
                        const uint4 y = *reinterpret_cast<const uint4*>(sj + p);
                        eq += (x.x == y.x) + (x.y == y.y) + (x.z == y.z) + (x.w == y.w);
                    }
                    dup = eq > max_equal;
                    break;                      // a candidate is judged once, whichever band made it one
                }
            }
        }
        if (j < n) keep[s0 + j] = live && !dup;
        __syncthreads();                        // `mine` is rewritten by the next round
    }
}

}  // namespace

extern "C" size_t rsb_minhash_workspace_bytes(int64_t total_bytes) {
    return total_bytes < 0 ? 0 : (size_t)total_bytes * 3 * sizeof(int32_t);
}

extern "C" int rsb_minhash_signatures(const uint8_t* text_dev, const int64_t* text_off_dev, int n_texts, int64_t total_bytes,
                                      const uint64_t* perm_a_dev, const uint64_t* perm_b_dev, uint32_t* sig_dev,
                                      int32_t* n_words_dev, void* ws_dev, size_t ws_bytes, rsb_stream_t stream) {
    if (n_texts < 0 || total_bytes < 0 || total_bytes >= ((int64_t)1 << 31))
        return dfail(RSB_ERR_INVALID, "bad shape n_texts=%d total_bytes=%lld (a batch holds fewer than 2^31 bytes)",
                     n_texts, (long long)total_bytes);
    if (n_texts == 0) return RSB_OK;
    if (!text_off_dev || !perm_a_dev || !perm_b_dev || !sig_dev || !n_words_dev || (total_bytes && (!text_dev || !ws_dev)))
        return dfail(RSB_ERR_INVALID, "null argument");
    const size_t need = rsb_minhash_workspace_bytes(total_bytes);
    if (ws_bytes < need) return dfail(RSB_ERR_OOM, "workspace too small: need %zu bytes, got %zu", need, ws_bytes);
    cudaStream_t st = (cudaStream_t)stream;
    int32_t* word_start = (int32_t*)ws_dev;
    int32_t* word_end = word_start + total_bytes;
    uint32_t* shingle_hash = (uint32_t*)(word_end + total_bytes);
    minhash_split_hash_kernel<<<n_texts, HT, 0, st>>>(text_dev, text_off_dev, word_start, word_end, shingle_hash, n_words_dev);
    DCU(cudaPeekAtLastError());
    minhash_signature_kernel<<<n_texts, NPERM, 0, st>>>(text_off_dev, n_words_dev, shingle_hash, (const u64*)perm_a_dev,
                                                        (const u64*)perm_b_dev, sig_dev);
    DCU(cudaPeekAtLastError());
    return RSB_OK;
}

extern "C" int rsb_minhash_dedup(const uint32_t* sig_dev, const int32_t* n_words_dev, const int32_t* group_off_dev,
                                 int n_groups, int bands, int rows, int max_equal, uint8_t* keep_dev, rsb_stream_t stream) {
    if (n_groups < 0 || bands < 1 || rows < 1 || bands * rows > NPERM || max_equal < 0 || max_equal > NPERM)
        return dfail(RSB_ERR_INVALID, "bad arguments n_groups=%d bands=%d rows=%d max_equal=%d (bands * rows <= %d)",
                     n_groups, bands, rows, max_equal, NPERM);
    if (n_groups == 0) return RSB_OK;
    if (!sig_dev || !n_words_dev || !group_off_dev || !keep_dev) return dfail(RSB_ERR_INVALID, "null argument");
    if ((uintptr_t)sig_dev & 15) return dfail(RSB_ERR_INVALID, "signatures must be 16-byte aligned");
    const int tile = LEAD_TILE_WORDS / bands;
    const size_t smem = (size_t)(tile + DT) * bands * sizeof(uint32_t);
    static PerDeviceSize configured;
    if (smem > 48 * 1024 && configured.raise(smem))
        DCU(cudaFuncSetAttribute(minhash_dedup_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    minhash_dedup_kernel<<<n_groups, DT, smem, (cudaStream_t)stream>>>(sig_dev, n_words_dev, group_off_dev, bands, rows,
                                                                       max_equal, tile, keep_dev);
    DCU(cudaPeekAtLastError());
    return RSB_OK;
}

extern "C" int rsb_utf8_space_mask(const uint8_t* bytes, int64_t n, uint8_t* mask) {
    if (n < 0 || (n && (!bytes || !mask))) return dfail(RSB_ERR_INVALID, "bad arguments");
    for (int64_t q = 0; q < n; ++q) mask[q] = in_space(bytes, n, q);
    return RSB_OK;
}
