// rsb_llm.cu -- reader-LM forward for perplexity evaluation: HF LlamaForCausalLM (Llama-2 MHA, Llama-3 GQA),
// GPTNeoXForCausalLM (Pythia) and OlmoForCausalLM / Olmo2ForCausalLM, chosen by rsb_llm_create's family, in fp16 or
// bf16 (every kernel is a template on its element type and rounds to it where HF's forward in that dtype rounds),
// over packed un-padded sequences: a prefill ending in the per-token negative log-likelihood of the labels, which
// replaces the reader call of the reference's perplexity loop (src/evaluate_perplexity.py:126-134: `lm(input_ids,
// labels=labels)` one window at a time, HF in bf16), and greedy generation with a KV cache (rsb_llm_generate).
//
//   embed_rows_kernel        X[t] = embed_tokens[ids[t]]
//   rms_rows_kernel          LlamaRMSNorm (the weight multiply in half) or Olmo2RMSNorm (in fp32), optionally fused with
//                            OLMo-2's post-norm residual add; the final norm runs on the gathered label rows only
//   rsb_gemm_f16             every linear layer on the encoder's TMA + wgmma kernel (gemm_tn_kernel, rsb_bert.cu): fused
//                            q|k|v and gate|up weights, residual adds through its residual epilogue with a zero bias
//   rope_kernel              HF rotate_half RoPE on the first rotary_dims of each Q and K head of the fused QKV rows (all
//                            128 for Llama); positions restart at 0 in every packed sequence
//   ln_rows_kernel           GPT-NeoX: torch's fp16 LayerNorm, with the parallel residual's last add and both norms fused
//   olmo_qkv_kernel          OLMo / OLMo-2: clip_qkv clamp or whole-projection QK RMSNorm, then RoPE with fp32 cos / sin
//   attention_causal_kernel  causal flash attention, head_dim 64 / 80 / 128 / 256, GQA, mma.sync.m16n8k16 with fp32 running max / sum;
//                            key blocks above the diagonal are never visited
//   swiglu_kernel            act = fp16(fp16(silu(gate)) * up), HF LlamaMLP's order
//   nll_rows_kernel          fp32 logsumexp over the real vocabulary (pad rows of the LM head excluded) - logit[label]
// Generation adds:
//   kv_store_kernel          K (after RoPE) and V of each row into the KV cache, in the prefill and in every decode step
//   decode_attention_kernel  split-KV attention of one query row per sequence over its cache, all query heads of a KV
//                            head in one mma tile; decode_combine_kernel merges the chunks
//   greedy_rows_kernel       fp32 argmax over the real vocabulary (lowest id on ties) and its log-softmax
// Multiple-choice scoring (rsb_llm_loglikelihood) adds:
//   choice_rows_kernel       the same pass over each scored row, then the log-softmax and greedy flag of its targets
#include "../../include/rsb.h"

#include "rsb_internal.h"

#include "rsb_dtype.cuh"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <map>
#include <set>
#include <string>
#include <type_traits>
#include <vector>

namespace {

using namespace rsbdt;

constexpr int HD = 128;                      // head_dim of every Llama reader
constexpr int AQ = 64, AK = 64;              // attention: 64 queries per block (16 per warp), key blocks of 64
constexpr size_t LOGIT_BYTES = 256u << 20;   // bound of the logits workspace of one LM-head chunk

__device__ __forceinline__ float block_sum(float v, float* red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float s = 0.f;
    for (int i = 0; i < nw; ++i) s += red[i];
    return s;
}

// one block per token; hidden % 8 == 0
template <typename T>
__global__ void embed_rows_kernel(const int* __restrict__ ids, const T* __restrict__ embed, int hidden,
                                  T* __restrict__ X) {
    const int t = blockIdx.x;
    const uint4* src = reinterpret_cast<const uint4*>(embed + (size_t)ids[t] * hidden);
    uint4* dst = reinterpret_cast<uint4*>(X + (size_t)t * hidden);
    for (int i = threadIdx.x; i < hidden / 8; i += blockDim.x) dst[i] = src[i];
}

// RMSNorm with fp32 statistics, rstd = rsqrt(mean(v^2) + eps), in one of HF's two rounding orders.  One block per
// output row i, input row r = rows ? rows[i] : i.
//   OLMO2 = false, LlamaRMSNorm (modeling_llama.py): weight * fp16(v * rstd), the weight multiply in half.
//   OLMO2 = true, Olmo2RMSNorm: fp16(w * (v * rstd)), the weight multiply in fp32 and one rounding.
//   A != nullptr: X[r] = fp16(X[r] + norm(A[r])), OLMo-2's post-norm residual add, in place; out is not written.
//   A == nullptr: out[i] = norm(X[r]).
template <typename T, bool OLMO2>
__global__ __launch_bounds__(256)
void rms_rows_kernel(T* __restrict__ X, const T* __restrict__ A, const int* __restrict__ rows, int hidden,
                     const T* __restrict__ w, float eps, T* __restrict__ out) {
    __shared__ float red[8];
    const int i = blockIdx.x;
    const int r = rows ? rows[i] : i;
    const uint4* a = reinterpret_cast<const uint4*>((A ? A : X) + (size_t)r * hidden);
    float s = 0.f;
    for (int c = threadIdx.x; c < hidden / 8; c += blockDim.x) {
        const uint4 v = a[c];
        const pair_t<T>* h2 = reinterpret_cast<const pair_t<T>*>(&v);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = to_f2(h2[e]);
            s = fmaf(f.x, f.x, s);
            s = fmaf(f.y, f.y, s);
        }
    }
    const float rstd = rsqrtf(block_sum(s, red) / (float)hidden + eps);
    const uint4* wv = reinterpret_cast<const uint4*>(w);
    uint4* x = reinterpret_cast<uint4*>(X + (size_t)r * hidden);
    uint4* o = reinterpret_cast<uint4*>(out + (size_t)i * hidden);
    for (int c = threadIdx.x; c < hidden / 8; c += blockDim.x) {
        const uint4 v = a[c], g = wv[c];
        const pair_t<T>* h2 = reinterpret_cast<const pair_t<T>*>(&v);
        const pair_t<T>* g2 = reinterpret_cast<const pair_t<T>*>(&g);
        uint4 nv;
        pair_t<T>* n2 = reinterpret_cast<pair_t<T>*>(&nv);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 f = to_f2(h2[e]);
            if constexpr (OLMO2) {
                const float2 gf = to_f2(g2[e]);
                n2[e] = from_f2<T>(__fmul_rn(gf.x, __fmul_rn(f.x, rstd)), __fmul_rn(gf.y, __fmul_rn(f.y, rstd)));
            } else {
                n2[e] = __hmul2(g2[e], from_f2<T>(f.x * rstd, f.y * rstd));
            }
        }
        if (A) {
            uint4 xv = x[c];
            pair_t<T>* x2 = reinterpret_cast<pair_t<T>*>(&xv);
#pragma unroll
            for (int e = 0; e < 4; ++e) x2[e] = __hadd2(x2[e], n2[e]);
            x[c] = xv;
        } else {
            o[c] = nv;
        }
    }
}

// The packed sequence b of token t: cu[b] <= t < cu[b+1].
__device__ __forceinline__ int seq_index(const int* __restrict__ cu_seqlens, int B, int t) {
    int lo = 0, hi = B;
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (cu_seqlens[mid] <= t) lo = mid; else hi = mid;
    }
    return lo;
}

// Position of row t: pos[t] when the caller gives explicit positions (a decode step, one row per sequence), else its
// position in its packed sequence, t - cu[b].
__device__ __forceinline__ int seq_position(const int* __restrict__ cu_seqlens, int B, const int* __restrict__ pos, int t) {
    return pos ? pos[t] : t - cu_seqlens[seq_index(cu_seqlens, B, t)];
}

// HF apply_rotary_pos_emb (modeling_llama.py, modeling_gpt_neox.py): rotate_half on dims [0, rot) of every Q and K
// head (head_dim hd apart, Q heads then K heads at the start of each QKV row, ld halves apart); dims [rot, hd) are
// neither read nor written (GPT-NeoX partial rotary; Llama has rot = hd = 128).  x_embed = x * cos + rotate_half(x) *
// sin in fp16, cos / sin = fp16(cos / sin(fp32(inv_freq[i] * pos))).  Each fp16 product and sum is one fp32 operation
// rounded to half, as torch computes half tensors.  One block per token; positions as seq_position.
template <typename T>
__global__ void rope_kernel(T* __restrict__ qkv, const int* __restrict__ cu_seqlens, int B, const int* __restrict__ positions,
                            int ld, int rot_heads, int hd, int rot, const float* __restrict__ inv_freq) {
    const int t = blockIdx.x;
    const float pos = (float)seq_position(cu_seqlens, B, positions, t);
    const int half_rot = rot >> 1;
    T* row = qkv + (size_t)t * ld;
    // pair p = head hh, dim i: advanced by blockDim.x pairs per step without a division in the loop
    const int dh = blockDim.x / half_rot, di = blockDim.x % half_rot;
    int hh = threadIdx.x / half_rot, i = threadIdx.x % half_rot;
    for (int p = threadIdx.x; p < rot_heads * half_rot; p += blockDim.x, hh += dh, i += di) {
        if (i >= half_rot) { i -= half_rot; ++hh; }
        T* x = row + hh * hd;
        const float f = inv_freq[i] * pos;
        const float c = to_f(from_f<T>(cosf(f))), s = to_f(from_f<T>(sinf(f)));
        const float x1 = to_f(x[i]), x2 = to_f(x[i + half_rot]);
        const float a1 = to_f(from_f<T>(x1 * c)), b1 = to_f(from_f<T>(-x2 * s));
        const float a2 = to_f(from_f<T>(x2 * c)), b2 = to_f(from_f<T>(x1 * s));
        x[i] = from_f<T>(a1 + b1);
        x[i + half_rot] = from_f<T>(a2 + b2);
    }
}

// torch's fp16 nn.LayerNorm, once or twice on the same row: mean and biased variance in fp32 (two passes over the row
// held in registers), y = fp16((x - mean) * rsqrt(var + eps) * w + b) with one rounding.  One block of 256 threads per
// output row i, input row r = rows ? rows[i] : i; hidden % 8 == 0 and hidden <= 8192.
//   add != nullptr: first X[r] = fp16(X[r] + add[r]) (the parallel residual's last sum, HF's order), written back.
//   w1 != nullptr: out1[i] = LN(X[r]; w1, b1); w2 != nullptr: out2[i] = LN(X[r]; w2, b2) from the same statistics.
constexpr int LN_THREADS = 256, LN_VEC = 4;   // up to 4 x 8 halves per thread
constexpr int LN_MAX_HIDDEN = LN_THREADS * LN_VEC * 8;   // 8192: the widest row ln_rows_kernel holds
template <typename T>
__global__ __launch_bounds__(LN_THREADS)
void ln_rows_kernel(T* __restrict__ X, const T* __restrict__ add, const int* __restrict__ rows, int hidden,
                    const T* __restrict__ w1, const T* __restrict__ b1, const T* __restrict__ w2,
                    const T* __restrict__ b2, float eps, T* __restrict__ out1, T* __restrict__ out2) {
    __shared__ float red[LN_THREADS / 32];
    const int i = blockIdx.x;
    const int r = rows ? rows[i] : i;
    const int n8 = hidden / 8;
    uint4* x = reinterpret_cast<uint4*>(X + (size_t)r * hidden);
    uint4 v[LN_VEC];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < LN_VEC; ++k) {
        const int c = threadIdx.x + k * LN_THREADS;
        v[k] = make_uint4(0, 0, 0, 0);
        if (c < n8) {
            v[k] = x[c];
            if (add) {
                const uint4 a = reinterpret_cast<const uint4*>(add + (size_t)r * hidden)[c];
                pair_t<T>* h2 = reinterpret_cast<pair_t<T>*>(&v[k]);
                const pair_t<T>* a2 = reinterpret_cast<const pair_t<T>*>(&a);
#pragma unroll
                for (int e = 0; e < 4; ++e) h2[e] = __hadd2(h2[e], a2[e]);
                x[c] = v[k];
            }
            const pair_t<T>* h2 = reinterpret_cast<const pair_t<T>*>(&v[k]);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 f = to_f2(h2[e]);
                s += f.x + f.y;
            }
        }
    }
    if (!w1 && !w2) return;
    const float mean = block_sum(s, red) / (float)hidden;
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < LN_VEC; ++k) {
        if (threadIdx.x + k * LN_THREADS < n8) {
            const pair_t<T>* h2 = reinterpret_cast<const pair_t<T>*>(&v[k]);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 f = to_f2(h2[e]);
                const float d0 = f.x - mean, d1 = f.y - mean;
                q = fmaf(d0, d0, q);
                q = fmaf(d1, d1, q);
            }
        }
    }
    const float rstd = rsqrtf(block_sum(q, red) / (float)hidden + eps);
    for (int n = 0; n < 2; ++n) {
        const T* w = n ? w2 : w1;
        const T* b = n ? b2 : b1;
        if (!w) continue;
        uint4* o = reinterpret_cast<uint4*>((n ? out2 : out1) + (size_t)i * hidden);
#pragma unroll
        for (int k = 0; k < LN_VEC; ++k) {
            const int c = threadIdx.x + k * LN_THREADS;
            if (c >= n8) continue;
            const uint4 g = reinterpret_cast<const uint4*>(w)[c], bb = reinterpret_cast<const uint4*>(b)[c];
            const pair_t<T>* h2 = reinterpret_cast<const pair_t<T>*>(&v[k]);
            const pair_t<T>* g2 = reinterpret_cast<const pair_t<T>*>(&g);
            const pair_t<T>* bb2 = reinterpret_cast<const pair_t<T>*>(&bb);
            uint4 ov;
            pair_t<T>* o2 = reinterpret_cast<pair_t<T>*>(&ov);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 f = to_f2(h2[e]), gf = to_f2(g2[e]), bf = to_f2(bb2[e]);
                o2[e] = from_f2<T>(fmaf((f.x - mean) * rstd, gf.x, bf.x), fmaf((f.y - mean) * rstd, gf.y, bf.y));
            }
            o[c] = ov;
        }
    }
}

// OLMo / OLMo-2 attention prologue on the fused QKV rows ([Q heads | K heads | V heads], 128 wide), HF's order.  One
// block per token; positions as seq_position (restarting at 0 in every packed sequence, or explicit).
//   clip > 0 (OLMo clip_qkv): every Q, K and V element is clamped to [-clip, clip] (in fp32, rounded to half).
//   qn != nullptr (OLMo-2 q_norm / k_norm): Q = fp16(qn * (Q * rsqrt(mean(Q^2) + eps))) over the whole Q projection
//   (heads x 128 wide, not per head), K likewise with kn over kv_heads x 128: fp32 statistics, the weight multiply in
//   fp32, one rounding, which RoPE then reads.
//   RoPE: OlmoRotaryEmbedding / Olmo2RotaryEmbedding keep cos / sin in fp32, so x * cos + rotate_half(x) * sin is
//   evaluated in fp32 (each product and the sum one fp32 rounding, as torch promotes) and rounded to half once.
template <typename T>
__global__ __launch_bounds__(256)
void olmo_qkv_kernel(T* __restrict__ qkv, const int* __restrict__ cu_seqlens, int B, const int* __restrict__ positions,
                     int heads, int kv_heads, const float* __restrict__ inv_freq, float clip, const T* __restrict__ qn,
                     const T* __restrict__ kn, float eps) {
    __shared__ float red[8];
    const int t = blockIdx.x;
    const float pos = (float)seq_position(cu_seqlens, B, positions, t);
    const int nq = heads * HD, nk = kv_heads * HD;
    T* row = qkv + (size_t)t * (nq + 2 * nk);
    float rq = 1.f, rk = 1.f;
    if (qn) {
        float sq = 0.f, sk = 0.f;
        const uint4* v = reinterpret_cast<const uint4*>(row);
        for (int c = threadIdx.x; c < (nq + nk) / 8; c += blockDim.x) {
            const uint4 u = v[c];
            const pair_t<T>* h2 = reinterpret_cast<const pair_t<T>*>(&u);
            float s = 0.f;
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 f = to_f2(h2[e]);
                s = fmaf(f.x, f.x, s);
                s = fmaf(f.y, f.y, s);
            }
            if (c < nq / 8) sq += s; else sk += s;
        }
        rq = rsqrtf(block_sum(sq, red) / (float)nq + eps);   // every read of the row precedes block_sum's barriers
        rk = rsqrtf(block_sum(sk, red) / (float)nk + eps);
    }
    auto clamped = [clip](float x) { return to_f(from_f<T>(fminf(fmaxf(x, -clip), clip))); };
    for (int p = threadIdx.x; p < (heads + kv_heads) * (HD / 2); p += blockDim.x) {
        const int hh = p / (HD / 2), i = p % (HD / 2);
        T* x = row + hh * HD;
        float x1 = to_f(x[i]), x2 = to_f(x[i + HD / 2]);
        if (clip > 0.f) { x1 = clamped(x1); x2 = clamped(x2); }
        if (qn) {
            const bool q = hh < heads;
            const T* w = q ? qn + hh * HD : kn + (hh - heads) * HD;
            const float r = q ? rq : rk;
            x1 = to_f(from_f<T>(__fmul_rn(to_f(w[i]), __fmul_rn(x1, r))));
            x2 = to_f(from_f<T>(__fmul_rn(to_f(w[i + HD / 2]), __fmul_rn(x2, r))));
        }
        const float f = inv_freq[i] * pos;
        const float c = cosf(f), s = sinf(f);
        x[i] = from_f<T>(__fadd_rn(__fmul_rn(x1, c), __fmul_rn(-x2, s)));
        x[i + HD / 2] = from_f<T>(__fadd_rn(__fmul_rn(x2, c), __fmul_rn(x1, s)));
    }
    if (clip > 0.f)
        for (int e = threadIdx.x; e < nk; e += blockDim.x) row[nq + nk + e] = from_f<T>(clamped(to_f(row[nq + nk + e])));
}

template <typename T>
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
    if constexpr (std::is_same<T, __half>::value)
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
    else
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                     : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                     : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
template <typename T>
__device__ __forceinline__ uint32_t ld32(const T* p) { return *reinterpret_cast<const uint32_t*>(p); }

// Row of 16-byte element idx >= 0 of a tile with n such elements per row: a shift when n is a power of two.
template <int n>
__device__ __forceinline__ int tile_row(int idx) {
    if constexpr ((n & (n - 1)) == 0) return idx >> (31 - __builtin_clz(n));
    else return (int)((unsigned)idx / n);
}

// Shared tile `which` (0 = K, 1 = V, 2 = Q) of 64 rows of D halves, padded by 8 halves per row against bank conflicts.
template <int D, int which, typename T>
__device__ __forceinline__ T (&attention_tile())[AK][D + 8] {
    if constexpr (D > 128) {
        extern __shared__ __align__(16) unsigned char attn_dyn[];
        return *reinterpret_cast<T (*)[AK][D + 8]>(attn_dyn + which * sizeof(T[AK][D + 8]));
    } else {
        __shared__ __align__(16) T tile[AK][D + 8];
        return tile;
    }
}

// Causal attention of one (sequence, query block of 64, head) at head_dim D: blockIdx.x = item (b, qb) from the host's
// list, heaviest query blocks first; blockIdx.y = query head h, which reads KV head h / (heads / kv_heads).  4 warps,
// 16 query rows each; key blocks 0..qb (every later one is fully masked) are staged in shared memory by the whole block.
// S = Q K^T and O += P V on mma.sync.m16n8k16 with fp32 accumulators; online softmax in the log2 domain with fp32
// running maximum and sum, P rounded to half for the P V product.  Inside the diagonal block a warp skips the key tiles
// of 8 that lie entirely above its last row.
// D <= 128: Q fragments in registers, K / V tiles in static shared memory (34.8 KB at D = 128).  D = 256: the 16 x 256
// fp32 output alone is 128 registers per thread, so Q is staged once in shared memory and its fragments are loaded
// with ldmatrix per 16-column step; Q, K and V tiles (3 x 33.8 KB) are dynamic shared memory.
template <int D, typename T>
__global__ __launch_bounds__(128)
void attention_causal_kernel(const T* __restrict__ qkv, const int* __restrict__ cu_seqlens,
                             const int2* __restrict__ items, T* __restrict__ ctx, int heads, int kv_heads,
                             float scale_log2) {
    constexpr int PAD = D + 8, KS = D / 16, NT = D / 8;
    constexpr bool QSMEM = D > 128;
    constexpr int KT = QSMEM ? 32 : AK, NKT = KT / 8;   // keys per softmax step; its key tiles of 8
    auto& Ks = attention_tile<D, 0, T>();
    auto& Vs = attention_tile<D, 1, T>();
    auto& Qs = attention_tile<D, 2, T>();           // D > 128 only
    const int2 it = items[blockIdx.x];
    const int b = it.x, qb = it.y, h = blockIdx.y, kvh = h / (heads / kv_heads);
    const int hid = heads * D, ld = hid + 2 * kv_heads * D;
    const int t0 = cu_seqlens[b], S = cu_seqlens[b + 1] - t0;
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const int qw = qb * AQ + wib * 16;           // first query row of this warp
    const bool active = qw < S;                  // warp-uniform; idle warps still stage K / V and meet the barriers
    const T* qbase = qkv + (size_t)t0 * ld + h * D;
    const T* kbase = qkv + (size_t)t0 * ld + hid + kvh * D;
    const T* vbase = kbase + kv_heads * D;
    const int r0 = qw + g, r1 = r0 + 8;

    uint32_t qa[QSMEM ? 1 : KS][4];
    if constexpr (QSMEM) {
#pragma unroll
        for (int i = 0; i < AQ * NT / 128; ++i) {   // 64 query rows, zero past the window (read by the first barrier)
            const int idx = threadIdx.x + 128 * i, j = tile_row<NT>(idx), c = idx - j * NT;
            const int q = qb * AQ + j;
            *reinterpret_cast<uint4*>(&Qs[j][c * 8]) =
                q < S ? *reinterpret_cast<const uint4*>(qbase + (size_t)q * ld + c * 8) : make_uint4(0, 0, 0, 0);
        }
    } else {
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            const int c = ks * 16 + 2 * t;
            qa[ks][0] = r0 < S ? ld32(qbase + (size_t)r0 * ld + c) : 0u;
            qa[ks][1] = r1 < S ? ld32(qbase + (size_t)r1 * ld + c) : 0u;
            qa[ks][2] = r0 < S ? ld32(qbase + (size_t)r0 * ld + c + 8) : 0u;
            qa[ks][3] = r1 < S ? ld32(qbase + (size_t)r1 * ld + c + 8) : 0u;
        }
    }
    float o[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) o[nt][e] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // l_run: per-lane partial sums

    for (int kb = 0; kb <= qb; ++kb) {
        __syncthreads();                         // the previous key block has been consumed by every warp
#pragma unroll
        for (int i = 0; i < AK * NT / 128; ++i) {   // 64 rows x D / 8 uint4 of K and of V
            const int idx = threadIdx.x + 128 * i, j = tile_row<NT>(idx), c = idx - j * NT;
            const int key = kb * AK + j;
            uint4 kv = make_uint4(0, 0, 0, 0), vv = kv;
            if (key < S) {
                kv = *reinterpret_cast<const uint4*>(kbase + (size_t)key * ld + c * 8);
                vv = *reinterpret_cast<const uint4*>(vbase + (size_t)key * ld + c * 8);
            }
            *reinterpret_cast<uint4*>(&Ks[j][c * 8]) = kv;
            *reinterpret_cast<uint4*>(&Vs[j][c * 8]) = vv;
        }
        __syncthreads();
        if (!active) continue;
#pragma unroll
        for (int sb = 0; sb < AK / KT; ++sb) {   // key steps of KT within the staged block
        const int k0 = kb * AK + sb * KT;        // first key of this step
        // key tiles of 8 holding at least one key <= this warp's last row (all of them below the diagonal block)
        int nvt;
        if constexpr (KT == AK) {
            nvt = kb < qb ? 8 : min(8, (qw + 15 - k0) / 8 + 1);
        } else {
            nvt = kb < qb ? NKT : (qw + 15 < k0 ? 0 : min(NKT, (qw + 15 - k0) / 8 + 1));
            if (nvt == 0) continue;              // warp-uniform: every key of the step is above this warp's rows
        }
        float sacc[NKT][4];
#pragma unroll
        for (int nt = 0; nt < NKT; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) sacc[nt][e] = 0.f;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            if constexpr (QSMEM) {
                const uint32_t addr = (uint32_t)__cvta_generic_to_shared(&Qs[wib * 16 + (lane & 15)][ks * 16 + (lane >> 4) * 8]);
                asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                             : "=r"(qa[0][0]), "=r"(qa[0][1]), "=r"(qa[0][2]), "=r"(qa[0][3]) : "r"(addr));
            }
#pragma unroll
            for (int nt = 0; nt < NKT; ++nt) {
                if (nt < nvt) {
                    const int j = sb * KT + nt * 8 + g, c = ks * 16 + 2 * t;
                    const uint32_t kf[2] = {ld32(&Ks[j][c]), ld32(&Ks[j][c + 8])};
                    mma16816<T>(sacc[nt], qa[QSMEM ? 0 : ks], kf);
                }
            }
        }
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int nt = 0; nt < NKT; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = k0 + nt * 8 + 2 * t + (e & 1), row = (e < 2) ? r0 : r1;
                const float sv = (nt < nvt && key <= row && key < S) ? sacc[nt][e] * scale_log2 : -INFINITY;
                sacc[nt][e] = sv;
                mx[e >> 1] = fmaxf(mx[e >> 1], sv);
            }
        float corr[2], mref[2];
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 1));
            mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 2));
            const float mn = fmaxf(m_run[hr], mx[hr]);
            mref[hr] = mn == -INFINITY ? 0.f : mn;   // a row without any valid key so far keeps probability 0
            corr[hr] = exp2f(m_run[hr] - mref[hr]);
            m_run[hr] = mn;
        }
        float sum[2] = {0.f, 0.f};
#pragma unroll
        for (int nt = 0; nt < NKT; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float p = exp2f(sacc[nt][e] - mref[e >> 1]);   // 2^-inf = 0
                sacc[nt][e] = p;
                sum[e >> 1] += p;
            }
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) l_run[hr] = l_run[hr] * corr[hr] + sum[hr];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            o[nt][0] *= corr[0]; o[nt][1] *= corr[0];
            o[nt][2] *= corr[1]; o[nt][3] *= corr[1];
        }
        uint32_t pa[NKT / 2][4];
#pragma unroll
        for (int kk = 0; kk < NKT / 2; ++kk) {
            pa[kk][0] = pair_bits<T>(sacc[2 * kk][0], sacc[2 * kk][1]);
            pa[kk][1] = pair_bits<T>(sacc[2 * kk][2], sacc[2 * kk][3]);
            pa[kk][2] = pair_bits<T>(sacc[2 * kk + 1][0], sacc[2 * kk + 1][1]);
            pa[kk][3] = pair_bits<T>(sacc[2 * kk + 1][2], sacc[2 * kk + 1][3]);
        }
#pragma unroll
        for (int kk = 0; kk < NKT / 2; ++kk) {
            if (kk * 2 < nvt) {                  // a 16-key step whose keys are all masked adds nothing
#pragma unroll
                for (int nt = 0; nt < NT; ++nt) {
                    uint32_t vb[2];
                    const uint32_t addr = (uint32_t)__cvta_generic_to_shared(&Vs[sb * KT + kk * 16 + (lane & 15)][nt * 8]);
                    asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];"
                                 : "=r"(vb[0]), "=r"(vb[1]) : "r"(addr));
                    mma16816<T>(o[nt], pa[kk], vb);
                }
            }
        }
        }
    }
    if (!active) return;
    float inv[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        float l = l_run[hr];
        l += __shfl_xor_sync(0xffffffffu, l, 1);
        l += __shfl_xor_sync(0xffffffffu, l, 2);
        inv[hr] = l > 0.f ? 1.f / l : 0.f;
    }
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        const int col = h * D + nt * 8 + 2 * t;
        if (r0 < S) *reinterpret_cast<pair_t<T>*>(ctx + (size_t)(t0 + r0) * hid + col) = from_f2<T>(o[nt][0] * inv[0], o[nt][1] * inv[0]);
        if (r1 < S) *reinterpret_cast<pair_t<T>*>(ctx + (size_t)(t0 + r1) * hid + col) = from_f2<T>(o[nt][2] * inv[1], o[nt][3] * inv[1]);
    }
}
constexpr size_t attention_dyn_smem(int D) { return D > 128 ? 3 * (size_t)AK * (D + 8) * sizeof(__half) : 0; }   // 2-byte elements in both dtypes

// KV cache of a generate call, per layer [slots][kv_heads][cap][head_dim] for K and again for V: one (sequence, KV head)
// is a contiguous run of positions.  Row t of the fused QKV rows goes to slot b, position p: in a prefill (slot ==
// nullptr) b is its packed sequence and p its position there, in a decode step b = slot[t] and p = pos[t].  K is stored
// after RoPE (OLMo: after clip_qkv and QK-norm), the values the attention kernels read.  One block per row.
template <typename T>
__global__ void kv_store_kernel(const T* __restrict__ qkv, const int* __restrict__ cu_seqlens, int B,
                                const int* __restrict__ slot, const int* __restrict__ pos, int heads, int kv_heads,
                                int hd, int cap, T* __restrict__ kc, T* __restrict__ vc) {
    const int t = blockIdx.x;
    const int b = slot ? slot[t] : seq_index(cu_seqlens, B, t);
    const int p = seq_position(cu_seqlens, B, pos, t);
    const int ld = (heads + 2 * kv_heads) * hd, n8 = hd / 8;
    const uint4* k = reinterpret_cast<const uint4*>(qkv + (size_t)t * ld + heads * hd);
    const uint4* v = k + kv_heads * n8;
    for (int e = threadIdx.x; e < kv_heads * n8; e += blockDim.x) {
        const int kvh = e / n8, c = e - kvh * n8;
        const size_t dst = (((size_t)b * kv_heads + kvh) * cap + p) * n8 + c;
        reinterpret_cast<uint4*>(kc)[dst] = k[e];
        reinterpret_cast<uint4*>(vc)[dst] = v[e];
    }
}

// Split-KV decode attention (flash-decoding).  Row i (one query token per live sequence) attends to positions
// [0, pos[i]] of its cache slot.  The positions are cut into chunks of DCH; warp w of block (x, y, i) takes chunk c =
// 4x + w and, as the rows of one 16-row mma tile, query heads 16 gt .. 16 gt + 15 of the G = heads / kv_heads that read
// KV head kvh, with y = kvh * ceil(G / 16) + gt.  For G <= 16 (every GQA reader released so far) one tile holds the
// whole group, so every cached byte is read once per step; a larger group (multi-query attention) reads it once per
// tile.  Chunk boundaries depend on the position only, never on the batch, so a
// sequence's result is the same in any batch.  Per chunk the warp stages Q (once) and 16 keys of K and V at a time in
// its own shared memory, computes S = Q K^T and O += P V on mma.sync.m16n8k16 with fp32 accumulators, online softmax
// in the log2 domain with fp32 running max and sum, P rounded to the dtype for P V (the prefill kernel's numerics).
// It writes the unnormalised O [D] and (max, sum) of every query head to part; decode_combine_kernel merges them.
constexpr int DCH = 64;                          // positions per chunk
constexpr int DEC_WARPS = 4;
template <int D> constexpr size_t decode_smem() { return (size_t)DEC_WARPS * 3 * 16 * (D + 8) * sizeof(__half); }

template <int D, typename T>
__global__ __launch_bounds__(32 * DEC_WARPS)
void decode_attention_kernel(const T* __restrict__ qkv, const T* __restrict__ kc, const T* __restrict__ vc,
                             const int* __restrict__ slot, const int* __restrict__ pos, int heads, int kv_heads, int cap,
                             int chunks, float scale_log2, float* __restrict__ part_o, float2* __restrict__ part_ml) {
    constexpr int PAD = D + 8, KS = D / 16, NT = D / 8, N8 = D / 8;
    extern __shared__ __align__(16) unsigned char dec_smem[];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const int G = heads / kv_heads, gtiles = (G + 15) / 16, ld = (heads + 2 * kv_heads) * D;
    const int c = blockIdx.x * DEC_WARPS + w, kvh = blockIdx.y / gtiles, g0 = (blockIdx.y - kvh * gtiles) * 16;
    const int i = blockIdx.z, nq = min(16, G - g0);   // query heads kvh * G + g0 .. + nq - 1
    const int L = pos[i] + 1, k_begin = c * DCH;
    if (k_begin >= L) return;                    // warp-uniform; no block-wide barrier below
    T (*Qs)[PAD] = reinterpret_cast<T (*)[PAD]>(dec_smem + (size_t)w * 3 * 16 * PAD * sizeof(T));
    T (*Ks)[PAD] = Qs + 16;
    T (*Vs)[PAD] = Qs + 32;
    const T* q = qkv + (size_t)i * ld + ((size_t)kvh * G + g0) * D;
    const size_t base = ((size_t)slot[i] * kv_heads + kvh) * cap * D;
    const T* kb = kc + base;
    const T* vb = vc + base;
    for (int e = lane; e < 16 * N8; e += 32) {   // the tile's query heads; rows >= nq are zero
        const int r = e / N8, cc = e - r * N8;
        *reinterpret_cast<uint4*>(&Qs[r][cc * 8]) =
            r < nq ? reinterpret_cast<const uint4*>(q + (size_t)r * D)[cc] : make_uint4(0, 0, 0, 0);
    }
    float o[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e) o[nt][e] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
    const int k_end = min(L, k_begin + DCH);
    for (int k0 = k_begin; k0 < k_end; k0 += 16) {
        __syncwarp();                            // the previous step's tiles (and the Q rows) are in place / consumed
        for (int e = lane; e < 16 * N8; e += 32) {   // keys past the row's length are zero, never stale cache
            const int r = e / N8, cc = e - r * N8, key = k0 + r;
            uint4 kv = make_uint4(0, 0, 0, 0), vv = kv;
            if (key < k_end) {
                kv = reinterpret_cast<const uint4*>(kb + (size_t)key * D)[cc];
                vv = reinterpret_cast<const uint4*>(vb + (size_t)key * D)[cc];
            }
            *reinterpret_cast<uint4*>(&Ks[r][cc * 8]) = kv;
            *reinterpret_cast<uint4*>(&Vs[r][cc * 8]) = vv;
        }
        __syncwarp();
        float sacc[2][4];
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) sacc[nt][e] = 0.f;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
            uint32_t qa[4];
            const uint32_t addr = (uint32_t)__cvta_generic_to_shared(&Qs[lane & 15][ks * 16 + (lane >> 4) * 8]);
            asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
                         : "=r"(qa[0]), "=r"(qa[1]), "=r"(qa[2]), "=r"(qa[3]) : "r"(addr));
#pragma unroll
            for (int nt = 0; nt < 2; ++nt) {
                const int j = nt * 8 + g, cc = ks * 16 + 2 * t;
                const uint32_t kf[2] = {ld32(&Ks[j][cc]), ld32(&Ks[j][cc + 8])};
                mma16816<T>(sacc[nt], qa, kf);
            }
        }
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const int key = k0 + nt * 8 + 2 * t + (e & 1);
                const float sv = key < k_end ? sacc[nt][e] * scale_log2 : -INFINITY;
                sacc[nt][e] = sv;
                mx[e >> 1] = fmaxf(mx[e >> 1], sv);
            }
        float corr[2], mref[2];
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
            mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 1));
            mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 2));
            const float mn = fmaxf(m_run[hr], mx[hr]);   // finite: key k0 < k_end is valid in every step
            mref[hr] = mn;
            corr[hr] = exp2f(m_run[hr] - mref[hr]);
            m_run[hr] = mn;
        }
        float sum[2] = {0.f, 0.f};
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float p = exp2f(sacc[nt][e] - mref[e >> 1]);
                sacc[nt][e] = p;
                sum[e >> 1] += p;
            }
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) l_run[hr] = l_run[hr] * corr[hr] + sum[hr];
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            o[nt][0] *= corr[0]; o[nt][1] *= corr[0];
            o[nt][2] *= corr[1]; o[nt][3] *= corr[1];
        }
        const uint32_t pa[4] = {pair_bits<T>(sacc[0][0], sacc[0][1]), pair_bits<T>(sacc[0][2], sacc[0][3]),
                                pair_bits<T>(sacc[1][0], sacc[1][1]), pair_bits<T>(sacc[1][2], sacc[1][3])};
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            uint32_t vf[2];
            const uint32_t addr = (uint32_t)__cvta_generic_to_shared(&Vs[lane & 15][nt * 8]);
            asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];" : "=r"(vf[0]), "=r"(vf[1]) : "r"(addr));
            mma16816<T>(o[nt], pa, vf);
        }
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        l_run[hr] += __shfl_xor_sync(0xffffffffu, l_run[hr], 1);
        l_run[hr] += __shfl_xor_sync(0xffffffffu, l_run[hr], 2);
    }
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
        const int r = g + 8 * hr;                // query head kvh * G + g0 + r
        if (r >= nq) continue;
        const size_t idx = ((size_t)i * heads + kvh * G + g0 + r) * chunks + c;
        float* po = part_o + idx * D;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt)
            *reinterpret_cast<float2*>(po + nt * 8 + 2 * t) = make_float2(o[nt][2 * hr], o[nt][2 * hr + 1]);
        if (t == 0) part_ml[idx] = make_float2(m_run[hr], l_run[hr]);
    }
}

// ctx[i, h] = sum_c 2^(m_c - M) O_c / sum_c 2^(m_c - M) l_c over the chunks of row i in chunk order, rounded to the
// dtype once.  Block (h, i), one thread per element of the head.
template <typename T>
__global__ void decode_combine_kernel(const float* __restrict__ part_o, const float2* __restrict__ part_ml,
                                      const int* __restrict__ pos, int heads, int D, int chunks, T* __restrict__ ctx) {
    const int h = blockIdx.x, i = blockIdx.y, d = threadIdx.x;
    const int n = (pos[i] + DCH) / DCH;          // chunks holding positions 0 .. pos[i]
    const size_t base = ((size_t)i * heads + h) * chunks;
    float M = -INFINITY;
    for (int c = 0; c < n; ++c) M = fmaxf(M, part_ml[base + c].x);
    float num = 0.f, den = 0.f;
    for (int c = 0; c < n; ++c) {
        const float2 ml = part_ml[base + c];
        const float s = exp2f(ml.x - M);
        num = fmaf(s, part_o[(base + c) * D + d], num);
        den = fmaf(s, ml.y, den);
    }
    ctx[((size_t)i * heads + h) * D + d] = from_f<T>(num / den);
}

// act[t, j] = fp16(fp16(silu(gate[t, j])) * up[t, j]) with gu = [gate | up] rows of 2 * inter; silu as torch computes it
// on half, x / (1 + exp(-x)) in fp32 rounded to half.  8 elements per thread.
template <typename T>
__global__ void swiglu_kernel(const T* __restrict__ gu, long long n8, int inter, T* __restrict__ act) {
    const int per_row = inter / 8;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8; i += (long long)gridDim.x * blockDim.x) {
        const long long t = i / per_row;
        const int c = (int)(i % per_row) * 8;
        const uint4 gv = *reinterpret_cast<const uint4*>(gu + t * 2 * inter + c);
        const uint4 uv = *reinterpret_cast<const uint4*>(gu + t * 2 * inter + inter + c);
        const pair_t<T>* g2 = reinterpret_cast<const pair_t<T>*>(&gv);
        const pair_t<T>* u2 = reinterpret_cast<const pair_t<T>*>(&uv);
        uint4 ov;
        pair_t<T>* o2 = reinterpret_cast<pair_t<T>*>(&ov);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const float2 x = to_f2(g2[e]);
            const pair_t<T> s = from_f2<T>(__fdiv_rn(x.x, 1.f + expf(-x.x)), __fdiv_rn(x.y, 1.f + expf(-x.y)));
            const float2 sf = to_f2(s), uf = to_f2(u2[e]);
            o2[e] = from_f2<T>(sf.x * uf.x, sf.y * uf.y);
        }
        *reinterpret_cast<uint4*>(act + t * inter + c) = ov;
    }
}

__device__ __forceinline__ void lse_merge(float& m, float& s, float m2, float s2) {
    const float mn = fmaxf(m, m2);
    if (mn == -INFINITY) return;
    s = s * expf(m - mn) + s2 * expf(m2 - mn);
    m = mn;
}

// nll_out[out_idx[i]] = logsumexp(logits[i, 0:vocab]) - logits[i, label[i]] in fp32; columns vocab..ld-1 are the LM
// head's pad rows and never enter the sum.  One block per row, one pass with a running (max, sum) per thread.
template <typename T>
__global__ __launch_bounds__(256)
void nll_rows_kernel(const T* __restrict__ logits, int vocab, int ld, const int* __restrict__ labels,
                     const int* __restrict__ out_idx, float* __restrict__ nll_out) {
    __shared__ float rm[8], rs[8];
    const int i = blockIdx.x;
    const T* row = logits + (size_t)i * ld;
    float m = -INFINITY, s = 0.f;
    for (int c = threadIdx.x * 8; c < vocab; c += blockDim.x * 8) {
        const uint4 v = *reinterpret_cast<const uint4*>(row + c);
        const T* hv = reinterpret_cast<const T*>(&v);
        float x[8], mx = -INFINITY;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            x[e] = c + e < vocab ? to_f(hv[e]) : -INFINITY;
            mx = fmaxf(mx, x[e]);
        }
        const float mn = fmaxf(m, mx);
        if (mn == -INFINITY) continue;           // every logit so far -inf: nothing to add, and -inf - -inf is NaN
        float acc = s * expf(m - mn);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc += expf(x[e] - mn);
        m = mn;
        s = acc;
    }
    for (int off = 16; off > 0; off >>= 1)
        lse_merge(m, s, __shfl_xor_sync(0xffffffffu, m, off), __shfl_xor_sync(0xffffffffu, s, off));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { rm[warp] = m; rs[warp] = s; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float M = rm[0], Sm = rs[0];
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w) lse_merge(M, Sm, rm[w], rs[w]);
        nll_out[out_idx[i]] = (M + logf(Sm)) - to_f(row[labels[i]]);
    }
}

// One block's single pass over row[0:vocab]: the fp32 logsumexp (nll_rows_kernel's sum) and the argmax compared in fp32,
// the lowest index on ties (torch.argmax); the LM head's pad columns vocab.. never compete.  The results are valid in
// thread 0 only.  blockDim.x <= 256.
template <typename T>
__device__ __forceinline__ void row_lse_argmax(const T* __restrict__ row, int vocab, float& lse, float& best, int& arg) {
    __shared__ float rm[8], rs[8], rv[8];
    __shared__ int ri[8];
    float m = -INFINITY, s = 0.f, bv = -INFINITY;
    int bi = INT_MAX;
    for (int c = threadIdx.x * 8; c < vocab; c += blockDim.x * 8) {
        const uint4 v = *reinterpret_cast<const uint4*>(row + c);
        const T* hv = reinterpret_cast<const T*>(&v);
        float x[8], mx = -INFINITY;
#pragma unroll
        for (int e = 0; e < 8; ++e) {
            x[e] = c + e < vocab ? to_f(hv[e]) : -INFINITY;
            mx = fmaxf(mx, x[e]);
            if (c + e < vocab && (x[e] > bv || (x[e] == bv && c + e < bi))) { bv = x[e]; bi = c + e; }
        }
        const float mn = fmaxf(m, mx);
        if (mn == -INFINITY) continue;           // every logit so far -inf: nothing to add, and -inf - -inf is NaN
        float acc = s * expf(m - mn);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc += expf(x[e] - mn);
        m = mn;
        s = acc;
    }
    auto better = [](float v, int k, float bv, int bk) { return v > bv || (v == bv && k < bk); };
    for (int off = 16; off > 0; off >>= 1) {
        lse_merge(m, s, __shfl_xor_sync(0xffffffffu, m, off), __shfl_xor_sync(0xffffffffu, s, off));
        const float ov = __shfl_xor_sync(0xffffffffu, bv, off);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
        if (better(ov, oi, bv, bi)) { bv = ov; bi = oi; }
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { rm[warp] = m; rs[warp] = s; rv[warp] = bv; ri[warp] = bi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float M = rm[0], Sm = rs[0], V = rv[0];
        int I = ri[0];
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w) {
            lse_merge(M, Sm, rm[w], rs[w]);
            if (better(rv[w], ri[w], V, I)) { V = rv[w]; I = ri[w]; }
        }
        if (I >= vocab) I = 0;                   // every logit NaN: the log-probability is NaN as well
        lse = M + logf(Sm);
        best = V;
        arg = I;
    }
}

// Greedy choice of row i (row_lse_argmax).  Writes the id to next[i] and out_tokens[s, step], and its fp32 log-softmax
// logit - logsumexp to out_lp[s, step] when out_lp is given, with s = slot ? slot[i] : base + i.  One block per row.
template <typename T>
__global__ __launch_bounds__(256)
void greedy_rows_kernel(const T* __restrict__ logits, int vocab, int ld, const int* __restrict__ slot, int base,
                        int step, int max_new, int* __restrict__ next, int* __restrict__ out_tokens,
                        float* __restrict__ out_lp) {
    const int i = blockIdx.x;
    float lse, V;
    int I;
    row_lse_argmax(logits + (size_t)i * ld, vocab, lse, V, I);
    if (threadIdx.x == 0) {
        const size_t o = (size_t)(slot ? slot[i] : base + i) * max_new + step;
        next[i] = I;
        out_tokens[o] = I;
        if (out_lp) out_lp[o] = V - lse;
    }
}

// Scored choices of row i (row_lse_argmax): for each of its targets j in [ptr[i], ptr[i+1]), out_lp[out[j]] = fp32
// logit[tok[j]] - logsumexp, bit for bit -nll_rows_kernel of the same (row, label), and out_greedy[out[j]] = 1 when
// tok[j] is the row's argmax, else 0.  One block per distinct row; the targets are spread over the block.
template <typename T>
__global__ __launch_bounds__(256)
void choice_rows_kernel(const T* __restrict__ logits, int vocab, int ld, const int* __restrict__ ptr,
                        const int* __restrict__ tok, const int* __restrict__ out, float* __restrict__ out_lp,
                        int* __restrict__ out_greedy) {
    __shared__ float s_lse;
    __shared__ int s_arg;
    const int i = blockIdx.x;
    const T* row = logits + (size_t)i * ld;
    float lse, V;
    int I;
    row_lse_argmax(row, vocab, lse, V, I);
    if (threadIdx.x == 0) { s_lse = lse; s_arg = I; }
    __syncthreads();
    for (int j = ptr[i] + threadIdx.x; j < ptr[i + 1]; j += blockDim.x) {
        const int t = tok[j];
        out_lp[out[j]] = to_f(row[t]) - s_lse;
        out_greedy[out[j]] = t == s_arg;
    }
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
thread_local std::string g_lerr;
int lfail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_lerr = buf;
    return code;
}

// Llama: wgu = gate | up, no biases.  GPT-NeoX: wgu = dense_h_to_4h, wdown = dense_4h_to_h, wqkv = query_key_value
// with its rows permuted to [Q heads | K heads | V heads], and the biases and LayerNorm biases below.  OLMo-2: ln1 / ln2
// = post_attention_layernorm / post_feedforward_layernorm, qn / kn = self_attn.q_norm / k_norm.
struct LlmLayer {
    __half *wqkv = nullptr, *wo = nullptr, *wgu = nullptr, *wdown = nullptr, *ln1 = nullptr, *ln2 = nullptr;
    __half *bqkv = nullptr, *bo = nullptr, *bgu = nullptr, *bdown = nullptr, *ln1b = nullptr, *ln2b = nullptr;
    __half *qn = nullptr, *kn = nullptr;
};

// How rsb_llm_load copies a weight to its destination.
enum class Copy {
    plain,
    neox_qkv,    // GPT-NeoX query_key_value weight or bias: per-head q_h | k_h | v_h rows to [Q heads | K heads | V heads]
    tied,        // the embedding of a tied handle: embed and lm_head
};

// Destination of one HF state-dict name.
struct Weight {
    __half* dst;
    int64_t n;                                   // elements
    Copy copy;
    bool counted;                                // required; a tied handle's lm_head.weight is accepted, copied, not counted
};

}  // namespace

struct rsb_llm {
    int family = RSB_LLM_LLAMA, dtype = RSB_DTYPE_F16;   // dtype: element type of weights and activations
    int layers = 0, hidden = 0, heads = 0, kv_heads = 0, inter = 0, vocab = 0, vocab_pad = 0, max_pos = 0;
    int head_dim = HD, rot = HD;                 // rot: rotated dims of each Q / K head (GPT-NeoX rotary_ndims)
    float eps = 0.f, clip = 0.f;                 // clip: OLMo clip_qkv, 0 = none
    bool tied = false;
    // Device buffers of 2-byte elements, fp16 or bf16 by the handle's dtype; every zero fill means 0 in both.
    // OLMo: final_g holds ones, the unit scale with which ln_rows_kernel (and zero_bias as its shift) is OlmoLayerNorm
    __half *embed = nullptr, *lm_head = nullptr, *final_g = nullptr, *final_b = nullptr, *zero_bias = nullptr;
    float* inv_freq = nullptr;
    std::vector<LlmLayer> L;
    // The only place the C side knows HF weight names: every name rsb_llm_load takes, with its destination.
    std::map<std::string, Weight> weights;
    std::vector<void*> owned;                    // every device allocation of the handle
    std::set<std::string> loaded;                // required weights loaded so far
    int qkv_n() const { return (heads + 2 * kv_heads) * head_dim; }
    size_t required() const {
        return std::count_if(weights.begin(), weights.end(), [](const auto& w) { return w.second.counted; });
    }
    int chunk_rows() const { return (int)std::max<size_t>(128, LOGIT_BYTES / ((size_t)vocab_pad * 2) / 128 * 128); }
};

namespace {

// A weight or bias buffer of the handle as element type E (the buffers are allocated as __half, 2 bytes either way).
template <typename E> const E* as(const __half* p) { return reinterpret_cast<const E*>(p); }

// f(E()) for the handle's element type E
template <class F> int with_dtype(const rsb_llm* h, F&& f) {
    return h->dtype == RSB_DTYPE_BF16 ? f(__nv_bfloat16()) : f(__half());
}

template <typename E> using same_t = typename std::common_type<E>::type;   // E, not deduced from this argument

template <typename E>
int gemm(const E* A, int M, const __half* W, int N, int K, const __half* bias, const same_t<E>* residual, same_t<E>* C,
         int epi, cudaStream_t st) {
    const int rc = std::is_same<E, __half>::value ? rsb_gemm_f16(A, W, bias, residual, C, M, N, K, epi, st)
                                                  : rsb::gemm_bf16(A, W, bias, residual, C, M, N, K, epi, st);
    return rc == RSB_OK ? RSB_OK : lfail(rc, "linear layer (%s)", rsb_bert_last_error());
}

// workspace: X, normed rows, QKV, attention output, gate|up, SwiGLU output, one chunk of logits, the label tables and
// the attention work list.  Label tables: logit row, label and output index per scored token.  GPT-NeoX: slot 1 holds
// both normed rows (ln1 | ln2), slot 4 the dense_h_to_4h output and slot 5 the attention block's output, to which the
// MLP output is added in place.
size_t llm_ws_layout(const rsb_llm* h, size_t T, size_t nl, size_t off[10]) {
    auto al = [](size_t x) { return (x + 1023) / 1024 * 1024; };
    const bool neox = h->family == RSB_LLM_NEOX;
    const size_t chunk = std::min<size_t>(std::max<size_t>(nl, 1), (size_t)h->chunk_rows());
    size_t o = 0;
    off[0] = o; o += al(T * h->hidden * 2);                 // X (residual stream)
    off[1] = o; o += al((neox ? 2 : 1) * T * h->hidden * 2);           // normed rows
    off[2] = o; o += al(T * (size_t)h->qkv_n() * 2);        // QKV
    off[3] = o; o += al(T * h->hidden * 2);                 // attention output
    off[4] = o; o += al((neox ? 1 : 2) * T * (size_t)h->inter * 2);    // gate | up
    off[5] = o; o += al(T * (size_t)(neox ? h->hidden : h->inter) * 2);   // SwiGLU output
    off[6] = o; o += al(chunk * (size_t)h->vocab_pad * 2);  // logits of one chunk of label rows
    off[7] = o; o += al(3 * std::max<size_t>(nl, 1) * sizeof(int));   // rows | labels | out_idx
    off[8] = o; o += al(T * sizeof(int2));                  // attention items (b, query block)
    off[9] = o;
    return o;
}

// Allocates a handle's device buffers and registers weight names against them; ok turns false on a failed cudaMalloc.
struct WeightTable {
    rsb_llm* h;
    bool ok = true;
    template <typename P = __half>
    P* alloc(size_t n) {
        void* p = nullptr;
        if (cudaMalloc(&p, n * sizeof(P)) != cudaSuccess) { ok = false; return nullptr; }
        h->owned.push_back(p);
        return static_cast<P*>(p);
    }
    void add(const std::string& name, __half* dst, int64_t n, Copy copy = Copy::plain, bool counted = true) {
        h->weights[name] = Weight{dst, n, copy, counted};
    }
    __half* weight(const std::string& name, int64_t n, Copy copy = Copy::plain) {   // a buffer of its own
        __half* p = alloc(n);
        add(name, p, n, copy);
        return p;
    }
};

// LlamaForCausalLM, OlmoForCausalLM and Olmo2ForCausalLM names; q|k|v and gate|up land in one fused weight each.
// Llama: input_layernorm / post_attention_layernorm are ln1 / ln2.  OLMo: no norm weights (OlmoLayerNorm has none).
// OLMo-2: post_attention_layernorm / post_feedforward_layernorm are ln1 / ln2, and q_norm / k_norm.
void llama_weights(WeightTable& t) {
    rsb_llm* h = t.h;
    const int64_t H = h->hidden, KV = (int64_t)h->kv_heads * HD, I = h->inter, V = h->vocab;
    t.add("model.embed_tokens.weight", h->embed, V * H, h->tied ? Copy::tied : Copy::plain);
    t.add("lm_head.weight", h->lm_head, V * H, Copy::plain, !h->tied);
    if (h->family != RSB_LLM_OLMO) t.add("model.norm.weight", h->final_g, H);
    for (int li = 0; li < h->layers; ++li) {
        LlmLayer& l = h->L[li];
        const std::string p = "model.layers." + std::to_string(li) + ".";
        l.wqkv = t.alloc((H + 2 * KV) * H);
        t.add(p + "self_attn.q_proj.weight", l.wqkv, H * H);
        t.add(p + "self_attn.k_proj.weight", l.wqkv + H * H, KV * H);
        t.add(p + "self_attn.v_proj.weight", l.wqkv + (H + KV) * H, KV * H);
        l.wo = t.weight(p + "self_attn.o_proj.weight", H * H);
        l.wgu = t.alloc(2 * I * H);
        t.add(p + "mlp.gate_proj.weight", l.wgu, I * H);
        t.add(p + "mlp.up_proj.weight", l.wgu + I * H, I * H);
        l.wdown = t.weight(p + "mlp.down_proj.weight", I * H);
        if (h->family == RSB_LLM_LLAMA) {
            l.ln1 = t.weight(p + "input_layernorm.weight", H);
            l.ln2 = t.weight(p + "post_attention_layernorm.weight", H);
        } else if (h->family == RSB_LLM_OLMO2) {
            l.ln1 = t.weight(p + "post_attention_layernorm.weight", H);
            l.ln2 = t.weight(p + "post_feedforward_layernorm.weight", H);
            l.qn = t.weight(p + "self_attn.q_norm.weight", H);
            l.kn = t.weight(p + "self_attn.k_norm.weight", KV);
        }
    }
}

// GPTNeoXForCausalLM names.  query_key_value's rows are [heads, 3, head_dim] (q_h | k_h | v_h per head); they land as
// [Q heads | K heads | V heads], so the forward reads the Llama layout.
void neox_weights(WeightTable& t) {
    rsb_llm* h = t.h;
    const int64_t H = h->hidden, I = h->inter, V = h->vocab;
    t.add("gpt_neox.embed_in.weight", h->embed, V * H);
    t.add("embed_out.weight", h->lm_head, V * H);
    t.add("gpt_neox.final_layer_norm.weight", h->final_g, H);
    h->final_b = t.weight("gpt_neox.final_layer_norm.bias", H);
    for (int li = 0; li < h->layers; ++li) {
        LlmLayer& l = h->L[li];
        const std::string p = "gpt_neox.layers." + std::to_string(li) + ".";
        l.ln1 = t.weight(p + "input_layernorm.weight", H);
        l.ln1b = t.weight(p + "input_layernorm.bias", H);
        l.ln2 = t.weight(p + "post_attention_layernorm.weight", H);
        l.ln2b = t.weight(p + "post_attention_layernorm.bias", H);
        l.wqkv = t.weight(p + "attention.query_key_value.weight", 3 * H * H, Copy::neox_qkv);
        l.bqkv = t.weight(p + "attention.query_key_value.bias", 3 * H, Copy::neox_qkv);
        l.wo = t.weight(p + "attention.dense.weight", H * H);
        l.bo = t.weight(p + "attention.dense.bias", H);
        l.wgu = t.weight(p + "mlp.dense_h_to_4h.weight", I * H);
        l.bgu = t.weight(p + "mlp.dense_h_to_4h.bias", I);
        l.wdown = t.weight(p + "mlp.dense_4h_to_h.weight", H * I);
        l.bdown = t.weight(p + "mlp.dense_4h_to_h.bias", H);
    }
}

// The refusals of rsb_llm_create (rsb.h), before any CUDA call.
int check_create(int family, int dtype, int layers, int hidden, int heads, int kv_heads, int intermediate, int vocab,
                 int max_pos, int rotary_dims, float rope_theta, float eps, float clip_qkv, int tied) {
    if (family < RSB_LLM_LLAMA || family > RSB_LLM_OLMO2)
        return lfail(RSB_ERR_INVALID, "family %ld is none of RSB_LLM_LLAMA, _NEOX, _OLMO and _OLMO2", (long)family);
    if (dtype != RSB_DTYPE_F16 && dtype != RSB_DTYPE_BF16)
        return lfail(RSB_ERR_INVALID, "dtype %ld is neither RSB_DTYPE_F16 nor RSB_DTYPE_BF16", (long)dtype);
    const bool neox = family == RSB_LLM_NEOX;
    if (layers <= 0 || vocab <= 0 || max_pos <= 0 || !(rope_theta > 0.f) || !(eps > 0.f) || (tied != 0 && tied != 1) ||
        (neox && (hidden <= 0 || heads <= 0 || intermediate <= 0)))
        return lfail(RSB_ERR_INVALID, "layers, vocab, max_pos, rope_theta (GPT-NeoX rotary_base), eps (rms_eps, ln_eps) "
                     "and, for GPT-NeoX, hidden, heads and intermediate must be positive, tied 0 or 1");
    if (!(clip_qkv >= 0.f) || std::isinf(clip_qkv) || (family != RSB_LLM_OLMO && clip_qkv != 0.f))
        return lfail(RSB_ERR_INVALID, "clip_qkv must be finite and >= 0 (0 = none), and 0 for every family but OLMo");
    if (neox) {
        if (kv_heads != heads)
            return lfail(RSB_ERR_UNSUPPORTED, "kv_heads %ld != heads %ld: GPT-NeoX has no grouped KV heads",
                         (long)kv_heads, (long)heads);
        if (tied) return lfail(RSB_ERR_UNSUPPORTED, "tied: GPT-NeoX readers have an untied embed_out");
        const int hd = hidden / heads;
        if (hidden % heads || (hd != 64 && hd != 80 && hd != 128 && hd != 256))
            return lfail(RSB_ERR_UNSUPPORTED, "head_dim %ld (hidden %ld / heads %ld): only head_dim 64, 80, 128 and 256 "
                         "are implemented", (long)(hidden % heads ? -1 : hd), (long)hidden, (long)heads);
        if (rotary_dims <= 0 || rotary_dims > hd)
            return lfail(RSB_ERR_INVALID, "rotary_dims %ld is not in [1, head_dim %ld]", (long)rotary_dims, (long)hd);
        if (rotary_dims % 2) return lfail(RSB_ERR_UNSUPPORTED, "rotary_dims %ld is odd", (long)rotary_dims);
    } else {
        if (heads <= 0 || hidden != heads * HD)
            return lfail(RSB_ERR_UNSUPPORTED, "only head_dim 128 is implemented (hidden %ld != 128 x heads)", (long)hidden);
        if (kv_heads <= 0 || heads % kv_heads)
            return lfail(RSB_ERR_UNSUPPORTED, "num_attention_heads must be a multiple of num_key_value_heads (got %ld kv "
                         "heads)", (long)kv_heads);
        if (rotary_dims != HD)
            return lfail(RSB_ERR_INVALID, "rotary_dims %ld: only GPT-NeoX rotates part of a head (rotary_dims = head_dim "
                         "128)", (long)rotary_dims);
    }
    if ((neox || family == RSB_LLM_OLMO) && hidden > LN_MAX_HIDDEN)
        return lfail(RSB_ERR_UNSUPPORTED, "hidden %ld: the LayerNorm kernel holds rows of at most %ld", (long)hidden,
                     (long)LN_MAX_HIDDEN);
    if (intermediate <= 0 || intermediate % 128)
        return lfail(RSB_ERR_UNSUPPORTED, "intermediate_size %ld is not a multiple of 128", (long)intermediate);
    return RSB_OK;
}

}  // namespace

extern "C" const char* rsb_llm_last_error(void) { return g_lerr.c_str(); }

// Replaces `AutoModelForCausalLM.from_pretrained(cfg.model.lm_model, torch_dtype=torch.bfloat16)`
// (src/evaluate_perplexity.py:98-108).  Every refusal comes before any CUDA call.
extern "C" int rsb_llm_create(int family, int dtype, int layers, int hidden, int heads, int kv_heads, int intermediate,
                              int vocab, int max_pos, int rotary_dims, float rope_theta, float eps, float clip_qkv,
                              int tied, rsb_llm_t** out) {
    if (!out) return lfail(RSB_ERR_INVALID, "out is NULL");
    *out = nullptr;
    const int rc = check_create(family, dtype, layers, hidden, heads, kv_heads, intermediate, vocab, max_pos,
                                rotary_dims, rope_theta, eps, clip_qkv, tied);
    if (rc != RSB_OK) return rc;
    rsb_llm* h = new rsb_llm();
    h->family = family; h->dtype = dtype;
    h->layers = layers; h->hidden = hidden; h->heads = heads; h->kv_heads = kv_heads; h->inter = intermediate;
    h->head_dim = hidden / heads; h->rot = rotary_dims;
    h->vocab = vocab; h->vocab_pad = (vocab + 127) / 128 * 128; h->max_pos = max_pos;
    h->eps = eps; h->clip = clip_qkv; h->tied = tied != 0;
    const size_t H = hidden, V = h->vocab_pad;
    const size_t zb = std::max({(size_t)h->qkv_n(), 2 * (size_t)intermediate, V, H});
    WeightTable t{h};
    h->embed = t.alloc((size_t)vocab * H);
    h->lm_head = t.alloc(V * H);
    h->final_g = t.alloc(H);
    h->zero_bias = t.alloc(zb);
    h->inv_freq = t.alloc<float>(rotary_dims / 2);
    h->L.resize(layers);
    if (family == RSB_LLM_NEOX) neox_weights(t); else llama_weights(t);
    if (!t.ok) { rsb_llm_free(h); return lfail(RSB_ERR_OOM, "allocating reader weights failed"); }
    // LlamaRotaryEmbedding / GPTNeoXRotaryEmbedding: inv_freq = 1 / theta ** (arange(0, rot, 2).float() / rot), in fp32
    std::vector<float> inv(rotary_dims / 2);
    for (int i = 0; i < rotary_dims / 2; ++i) inv[i] = 1.f / powf(rope_theta, (float)(2 * i) / (float)rotary_dims);
    bool ok = cudaMemcpy(h->inv_freq, inv.data(), inv.size() * sizeof(float), cudaMemcpyHostToDevice) == cudaSuccess;
    ok &= cudaMemset(h->zero_bias, 0, zb * 2) == cudaSuccess;
    ok &= cudaMemset(h->lm_head, 0, V * H * 2) == cudaSuccess;   // pad rows stay zero (and outside the sum)
    if (family == RSB_LLM_OLMO) {
        const std::vector<uint16_t> ones(H, dtype == RSB_DTYPE_BF16 ? 0x3F80 : 0x3C00);   // 1.0 in bf16 / fp16
        ok &= cudaMemcpy(h->final_g, ones.data(), H * 2, cudaMemcpyHostToDevice) == cudaSuccess;
    }
    if (!ok) { rsb_llm_free(h); return lfail(RSB_ERR_CUDA, "initialising the reader failed"); }
    *out = h;
    return RSB_OK;
}

extern "C" int rsb_llm_free(rsb_llm_t* h) {
    if (!h) return RSB_OK;
    for (void* p : h->owned) cudaFree(p);
    delete h;
    return RSB_OK;
}

// name = an HF state-dict key of the handle's family (rsb.h), data on the device in the handle's dtype, copied
// (src/evaluate_perplexity.py:98-108 loads the same checkpoint).
extern "C" int rsb_llm_load(rsb_llm_t* h, const char* name, const void* f16_dev, int64_t n, rsb_stream_t stream) {
    if (!h || !name || !f16_dev) return lfail(RSB_ERR_INVALID, "null argument");
    const auto it = h->weights.find(name);
    if (it == h->weights.end()) return lfail(RSB_ERR_INVALID, "unknown weight name %s", name);
    const Weight& w = it->second;
    if (n != w.n) return lfail(RSB_ERR_INVALID, "weight %s has the wrong size (%ld elements)", name, (long)n);
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e;
    if (w.copy == Copy::neox_qkv) {              // one strided copy per part
        const int64_t H = h->hidden, per_row = n / (3 * H);   // H (weight) or 1 (bias)
        const size_t part = (size_t)h->head_dim * per_row * 2;     // bytes of one head's q (or k or v) rows
        e = cudaSuccess;
        for (int p = 0; p < 3 && e == cudaSuccess; ++p)
            e = cudaMemcpy2DAsync(w.dst + p * H * per_row, part, static_cast<const char*>(f16_dev) + p * part, 3 * part,
                                  part, h->heads, cudaMemcpyDeviceToDevice, st);
    } else {
        e = cudaMemcpyAsync(w.dst, f16_dev, (size_t)n * 2, cudaMemcpyDeviceToDevice, st);
        if (e == cudaSuccess && w.copy == Copy::tied)
            e = cudaMemcpyAsync(h->lm_head, f16_dev, (size_t)n * 2, cudaMemcpyDeviceToDevice, st);
    }
    if (e != cudaSuccess) return lfail(RSB_ERR_CUDA, "copy of %s failed", name);
    if (w.counted) h->loaded.insert(name);
    return RSB_OK;
}

extern "C" size_t rsb_llm_workspace_bytes(rsb_llm_t* h, int total_tokens, int label_tokens) {
    if (!h || total_tokens < 0 || label_tokens < 0) return 0;
    size_t off[10];
    return llm_ws_layout(h, (size_t)std::max(total_tokens, 1), (size_t)label_tokens, off);
}

namespace {

// Checks offsets read back from the device: 0 = cu[0] <= cu[1] <= ... <= cu[B] <= T, every window <= max_seqlen tokens.
int check_offsets(const std::vector<int32_t>& cu, int B, int T, int max_seqlen) {
    if (cu[0] != 0 || cu[B] > T) return lfail(RSB_ERR_INVALID, "cu_seqlens must run from 0 to at most T (T = %ld)", (long)T);
    for (int b = 0; b < B; ++b) {
        const int S = cu[b + 1] - cu[b];
        if (S < 0) return lfail(RSB_ERR_INVALID, "cu_seqlens decreases at sequence %ld", (long)b);
        if (S > max_seqlen) return lfail(RSB_ERR_INVALID, "a sequence of %ld tokens is longer than max_seqlen", (long)S);
    }
    return RSB_OK;
}

// The attention work list: one item (sequence b, query block q) per 64 queries of every window, heaviest query blocks
// first (block q of a sequence visits q + 1 key blocks), uploaded to d_items (room for cu[B] items).
int upload_attention_items(const std::vector<int32_t>& cu, int B, int2* d_items, cudaStream_t st, int* n_items) {
    std::vector<int2> items;
    for (int b = 0; b < B; ++b)
        for (int q = 0; q * AQ < cu[b + 1] - cu[b]; ++q) items.push_back(make_int2(b, q));
    std::stable_sort(items.begin(), items.end(), [](const int2& a, const int2& b) { return a.y > b.y; });
    *n_items = (int)items.size();
    if (!items.empty() &&
        cudaMemcpyAsync(d_items, items.data(), items.size() * sizeof(int2), cudaMemcpyHostToDevice, st) != cudaSuccess)
        return lfail(RSB_ERR_CUDA, "uploading the attention work list failed");
    return RSB_OK;
}

// The KV cache of a generate call (kv_store_kernel's layout) and, in a decode step, where each row goes.
template <typename E>
struct KvCache {
    E *k, *v;                                    // [layers][slots][kv_heads][cap][head_dim] each
    int slots, cap;
    const int *slot = nullptr, *pos = nullptr;   // decode step: cache slot and position of each row; prefill: nullptr
    float* part_o = nullptr;                     // decode step: split-KV partials of decode_attention_kernel
    float2* part_ml = nullptr;
    int chunks = 0;                              // decode step: DCH-position chunks of the longest row
    size_t layer_elems(const rsb_llm* h) const { return (size_t)slots * h->kv_heads * cap * h->head_dim; }
};

template <int D, typename E>
void launch_decode_attention(const rsb_llm* h, const E* QKV, const E* kc, const E* vc, const KvCache<E>& kv, int n_rows,
                             float scale_log2, cudaStream_t st) {
    constexpr size_t smem = decode_smem<D>();
    static rsb::PerDeviceFlag configured;        // attributes are per (function, device)
    if (configured.first())
        cudaFuncSetAttribute(decode_attention_kernel<D, E>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    const int gtiles = (h->heads / h->kv_heads + 15) / 16;   // 16-row query-head tiles per KV head
    const dim3 grid((unsigned)((kv.chunks + DEC_WARPS - 1) / DEC_WARPS), h->kv_heads * gtiles, n_rows);
    decode_attention_kernel<D, E><<<grid, 32 * DEC_WARPS, smem, st>>>(QKV, kc, vc, kv.slot, kv.pos, h->heads, h->kv_heads,
                                                                      kv.cap, kv.chunks, scale_log2, kv.part_o, kv.part_ml);
}

// One attention step of layer li on the fused QKV rows [n_tok, qkv_n]: RoPE on the Q and K heads in place (OLMo: the
// clip / QK-norm prologue and fp32 RoPE), then attention into CTX [n_tok, hidden].
//   kv == nullptr or a prefill (kv->pos == nullptr): rows are the packed windows of cu_seqlens, n_tok = cu[B], with
//   positions restarting at 0 in each; causal attention.  With kv, K and V also go to the cache, slot b for window b.
//   A decode step (kv->pos): row i is one token of cache slot kv->slot[i] at position kv->pos[i]; its K and V are
//   appended there and it attends to positions 0 .. pos[i] of the slot (split-KV).
template <typename E>
void attention_step(const rsb_llm* h, int li, E* QKV, const int32_t* cu_seqlens, int B, int n_tok,
                    const int2* d_items, int n_items, E* CTX, const KvCache<E>* kv, cudaStream_t st) {
    const bool decode = kv && kv->pos;
    if (n_tok == 0 || (!decode && n_items == 0)) return;
    const LlmLayer& l = h->L[li];
    const int* pos = decode ? kv->pos : nullptr;
    const float scale_log2 = 1.4426950408889634f / sqrtf((float)h->head_dim);   // 1/sqrt(head_dim) in the log2 domain
    if (h->family == RSB_LLM_OLMO || h->family == RSB_LLM_OLMO2)
        olmo_qkv_kernel<E><<<n_tok, 256, 0, st>>>(QKV, cu_seqlens, B, pos, h->heads, h->kv_heads, h->inv_freq, h->clip,
                                                  as<E>(l.qn), as<E>(l.kn), h->eps);
    else
        rope_kernel<E><<<n_tok, 256, 0, st>>>(QKV, cu_seqlens, B, pos, h->qkv_n(), h->heads + h->kv_heads, h->head_dim,
                                              h->rot, h->inv_freq);
    if (kv) {
        E* kc = kv->k + (size_t)li * kv->layer_elems(h);
        E* vc = kv->v + (size_t)li * kv->layer_elems(h);
        kv_store_kernel<E><<<n_tok, 128, 0, st>>>(QKV, cu_seqlens, B, kv->slot, pos, h->heads, h->kv_heads, h->head_dim,
                                                  kv->cap, kc, vc);
        if (decode) {
            switch (h->head_dim) {
                case 64: launch_decode_attention<64>(h, QKV, kc, vc, *kv, n_tok, scale_log2, st); break;
                case 80: launch_decode_attention<80>(h, QKV, kc, vc, *kv, n_tok, scale_log2, st); break;
                case 128: launch_decode_attention<128>(h, QKV, kc, vc, *kv, n_tok, scale_log2, st); break;
                default: launch_decode_attention<256>(h, QKV, kc, vc, *kv, n_tok, scale_log2, st);
            }
            decode_combine_kernel<E><<<dim3(h->heads, n_tok), h->head_dim, 0, st>>>(kv->part_o, kv->part_ml, pos, h->heads,
                                                                                  h->head_dim, kv->chunks, CTX);
            return;
        }
    }
    const dim3 grid((unsigned)n_items, h->heads);
    switch (h->head_dim) {
        case 64: attention_causal_kernel<64, E><<<grid, 128, 0, st>>>(QKV, cu_seqlens, d_items, CTX, h->heads, h->kv_heads, scale_log2); break;
        case 80: attention_causal_kernel<80, E><<<grid, 128, 0, st>>>(QKV, cu_seqlens, d_items, CTX, h->heads, h->kv_heads, scale_log2); break;
        case 128: attention_causal_kernel<128, E><<<grid, 128, 0, st>>>(QKV, cu_seqlens, d_items, CTX, h->heads, h->kv_heads, scale_log2); break;
        default: {
            constexpr size_t smem = attention_dyn_smem(256);
            static rsb::PerDeviceFlag configured;            // attributes are per (function, device)
            if (configured.first())
                cudaFuncSetAttribute(attention_causal_kernel<256, E>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            attention_causal_kernel<256, E><<<grid, 128, smem, st>>>(QKV, cu_seqlens, d_items, CTX, h->heads, h->kv_heads, scale_log2);
        }
    }
}

// Refusals shared by rsb_llm_nll and rsb_llm_hidden_states, then the read-back of the offsets and ids (and labels).
int check_forward(rsb_llm* h, const int32_t* ids, const int32_t* cu_seqlens, const int32_t* labels, int B, int T,
                  int max_seqlen, cudaStream_t st, std::vector<int32_t>& cu, std::vector<int32_t>& lab) {
    if (B <= 0 || T <= 0) return lfail(RSB_ERR_INVALID, "empty batch");
    if (max_seqlen > h->max_pos)
        return lfail(RSB_ERR_UNSUPPORTED, "sequence longer than max_position_embeddings (%ld)", (long)h->max_pos);
    if (h->loaded.size() != h->required())
        return lfail(RSB_ERR_STATE, "%ld reader weights are not loaded", (long)(h->required() - h->loaded.size()));
    std::vector<int32_t> hid(T);
    cu.assign(B + 1, 0);
    lab.assign(labels ? T : 0, 0);
    if (cudaMemcpyAsync(cu.data(), cu_seqlens, cu.size() * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaMemcpyAsync(hid.data(), ids, (size_t)T * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        (labels && cudaMemcpyAsync(lab.data(), labels, (size_t)T * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess) ||
        cudaStreamSynchronize(st) != cudaSuccess)
        return lfail(RSB_ERR_CUDA, "reading back the batch failed");
    if (cu[0] != 0 || cu[B] != T) return lfail(RSB_ERR_INVALID, "cu_seqlens must run from 0 to T (T = %ld)", (long)T);
    const int rc = check_offsets(cu, B, T, max_seqlen);
    if (rc != RSB_OK) return rc;
    for (int t = 0; t < T; ++t) {
        if (hid[t] < 0 || hid[t] >= h->vocab) return lfail(RSB_ERR_INVALID, "token id %ld is outside the vocabulary", (long)hid[t]);
        if (labels && lab[t] != -100 && (lab[t] < 0 || lab[t] >= h->vocab))
            return lfail(RSB_ERR_INVALID, "label %ld is neither -100 nor a token id", (long)lab[t]);
    }
    return RSB_OK;
}

// Workspace slots of one forward (llm_ws_layout), its attention work list and, in rsb_llm_generate, the KV cache.
template <typename E>
struct Fwd {
    E *X, *Hn, *QKV, *CTX, *GU, *ACT;
    const int32_t* cu_seqlens;
    int B, T, n_items;
    const int2* d_items;
    const KvCache<E>* kv = nullptr;
};

// The sequential-residual decoder layers, x layers.  LlamaDecoderLayer: x += o_proj(attn(rms1(x))); x +=
// down(swiglu(gate|up(rms2(x)))).  OlmoDecoderLayer: the same with OlmoLayerNorm (ln_rows_kernel with unit scale and
// zero shift) as both pre-norms.  Olmo2DecoderLayer: no pre-norms; x = fp16(x +
// post_attention_layernorm(o_proj(attn(x)))), then x = fp16(x + post_feedforward_layernorm(down(swiglu(gate|up(x))))).
// A norm sits between each projection and its add, so o_proj and down_proj write slot 1 (free without pre-norms) and
// rms_rows_kernel adds the normed rows to x.
template <typename E>
int sequential_layers(rsb_llm* h, const Fwd<E>& f, cudaStream_t st) {
    const int Hd = h->hidden, NQKV = h->qkv_n(), I = h->inter, T = f.T;
    const long long n8 = (long long)T * I / 8;
    const int sw_grid = (int)std::min<long long>((n8 + 255) / 256, 8LL * rsb::device_num_sms());
    const bool v2 = h->family == RSB_LLM_OLMO2;
    const E* in = v2 ? f.X : f.Hn;               // what q|k|v and gate|up read
    auto pre_norm = [&](const __half* w) {       // w: the Llama norm's weight
        if (h->family == RSB_LLM_LLAMA)
            rms_rows_kernel<E, false><<<T, 256, 0, st>>>(f.X, nullptr, nullptr, Hd, as<E>(w), h->eps, f.Hn);
        else if (h->family == RSB_LLM_OLMO)
            ln_rows_kernel<E><<<T, LN_THREADS, 0, st>>>(f.X, nullptr, nullptr, Hd, as<E>(h->final_g), as<E>(h->zero_bias),
                                                        nullptr, nullptr, h->eps, f.Hn, nullptr);
    };
    // x += A W^T, or for OLMo-2 x = fp16(x + norm(A W^T)) with the post-norm weight w
    auto residual = [&](const E* A, const __half* W, int K, int epi, const __half* w) -> int {
        if (!v2) return gemm(A, T, W, Hd, K, h->zero_bias, f.X, f.X, 2 | epi, st);
        const int rc = gemm(A, T, W, Hd, K, h->zero_bias, nullptr, f.Hn, 0, st);
        if (rc == RSB_OK) rms_rows_kernel<E, true><<<T, 256, 0, st>>>(f.X, f.Hn, nullptr, Hd, as<E>(w), h->eps, nullptr);
        return rc;
    };
    int rc;
    for (int li = 0; li < h->layers; ++li) {
        const LlmLayer& l = h->L[li];
        pre_norm(l.ln1);
        if ((rc = gemm(in, T, l.wqkv, NQKV, Hd, h->zero_bias, nullptr, f.QKV, 0, st)) != RSB_OK) return rc;
        attention_step(h, li, f.QKV, f.cu_seqlens, f.B, T, f.d_items, f.n_items, f.CTX, f.kv, st);
        if ((rc = residual(f.CTX, l.wo, Hd, 0, l.ln1)) != RSB_OK) return rc;
        pre_norm(l.ln2);
        if ((rc = gemm(in, T, l.wgu, 2 * I, Hd, h->zero_bias, nullptr, f.GU, 0, st)) != RSB_OK) return rc;
        swiglu_kernel<E><<<sw_grid, 256, 0, st>>>(f.GU, n8, I, f.ACT);
        if ((rc = residual(f.ACT, l.wdown, I, RSB_GEMM_REVERSED, l.ln2)) != RSB_OK) return rc;
    }
    return RSB_OK;
}

// GPTNeoXLayer x layers with the parallel residual: x = fp16(fp16(mlp(ln2(x)) + attn(ln1(x))) + x).  The MLP's last
// GEMM adds the attention block's output A in its residual epilogue (A = fp16(mlp + attn), in place); the next
// ln_rows_kernel adds A to x, writes x back and normalises it twice, for the next layer's ln1 and ln2.
template <typename E>
int neox_layers(rsb_llm* h, const Fwd<E>& f, cudaStream_t st) {
    const int Hd = h->hidden, NQKV = h->qkv_n(), I = h->inter, T = f.T;
    E *N1 = f.Hn, *N2 = f.Hn + (size_t)T * Hd, *FF = f.GU, *A = f.ACT;
    const LlmLayer& l0 = h->L[0];
    int rc;
    ln_rows_kernel<E><<<T, LN_THREADS, 0, st>>>(f.X, nullptr, nullptr, Hd, as<E>(l0.ln1), as<E>(l0.ln1b), as<E>(l0.ln2),
                                                as<E>(l0.ln2b), h->eps, N1, N2);
    for (int li = 0; li < h->layers; ++li) {
        const LlmLayer& l = h->L[li];
        if ((rc = gemm(N1, T, l.wqkv, NQKV, Hd, l.bqkv, nullptr, f.QKV, 0, st)) != RSB_OK) return rc;
        attention_step(h, li, f.QKV, f.cu_seqlens, f.B, T, f.d_items, f.n_items, f.CTX, f.kv, st);
        if ((rc = gemm(f.CTX, T, l.wo, Hd, Hd, l.bo, nullptr, A, 0, st)) != RSB_OK) return rc;
        if ((rc = gemm(N2, T, l.wgu, I, Hd, l.bgu, nullptr, FF, 1, st)) != RSB_OK) return rc;
        if ((rc = gemm(FF, T, l.wdown, Hd, I, l.bdown, A, A, 2 | RSB_GEMM_REVERSED, st)) != RSB_OK) return rc;
        const LlmLayer* nx = li + 1 < h->layers ? &h->L[li + 1] : nullptr;   // the last layer only adds
        ln_rows_kernel<E><<<T, LN_THREADS, 0, st>>>(f.X, A, nullptr, Hd, nx ? as<E>(nx->ln1) : nullptr,
                                                    nx ? as<E>(nx->ln1b) : nullptr, nx ? as<E>(nx->ln2) : nullptr,
                                                    nx ? as<E>(nx->ln2b) : nullptr, h->eps, N1, N2);
    }
    return RSB_OK;
}

// The decoder layers: X (workspace slot 0) ends as the residual stream after the last layer, before the final norm.
// Packed windows (cu, cu_seqlens), or with kv->pos one row per live sequence of a decode step (cu_seqlens unused).
template <typename E>
int trunk(rsb_llm* h, const int32_t* ids, const int32_t* cu_seqlens, int B, int T, const std::vector<int32_t>& cu,
          unsigned char* w, const size_t off[10], cudaStream_t st, const KvCache<E>* kv = nullptr) {
    Fwd<E> f;
    f.X = reinterpret_cast<E*>(w + off[0]);
    f.Hn = reinterpret_cast<E*>(w + off[1]);
    f.QKV = reinterpret_cast<E*>(w + off[2]);
    f.CTX = reinterpret_cast<E*>(w + off[3]);
    f.GU = reinterpret_cast<E*>(w + off[4]);
    f.ACT = reinterpret_cast<E*>(w + off[5]);
    f.cu_seqlens = cu_seqlens;
    f.B = B;
    f.T = T;
    f.kv = kv;
    int2* d_items = reinterpret_cast<int2*>(w + off[8]);
    f.d_items = d_items;
    f.n_items = 0;
    int rc;
    if (!(kv && kv->pos) && (rc = upload_attention_items(cu, B, d_items, st, &f.n_items)) != RSB_OK) return rc;
    embed_rows_kernel<E><<<T, 128, 0, st>>>(ids, as<E>(h->embed), h->hidden, f.X);
    return h->family == RSB_LLM_NEOX ? neox_layers(h, f, st) : sequential_layers(h, f, st);
}

// The final norm of the label rows X[rows[i]] into out[i], i < n.
template <typename E>
void final_norm(const rsb_llm* h, const E* X, const int* rows, int n, E* out, cudaStream_t st) {
    const bool neox = h->family == RSB_LLM_NEOX;
    if (neox || h->family == RSB_LLM_OLMO)       // OLMo: unit scale (final_g) and zero shift
        ln_rows_kernel<E><<<n, LN_THREADS, 0, st>>>(const_cast<E*>(X), nullptr, rows, h->hidden, as<E>(h->final_g),
                                                    as<E>(neox ? h->final_b : h->zero_bias), nullptr, nullptr, h->eps,
                                                    out, nullptr);
    else if (h->family == RSB_LLM_OLMO2)
        rms_rows_kernel<E, true><<<n, 256, 0, st>>>(const_cast<E*>(X), nullptr, rows, h->hidden, as<E>(h->final_g), h->eps,
                                                    out);
    else
        rms_rows_kernel<E, false><<<n, 256, 0, st>>>(const_cast<E*>(X), nullptr, rows, h->hidden, as<E>(h->final_g),
                                                     h->eps, out);
}

}  // namespace

// The reader forward and loss of src/evaluate_perplexity.py:126-134 (`lm(input_ids, labels=labels)` per window) over B
// packed windows.  ids / labels [T] int32 and cu_seqlens [B+1] int32 on the device; nll_out [T] fp32 receives, at
// every position t that is not the first of its sequence and whose label is not -100, -log p(labels[t] | ids of the
// sequence before t), and 0 elsewhere.  The ids, labels and offsets are read back and checked before any launch.
extern "C" int rsb_llm_nll(rsb_llm_t* h, const int32_t* ids, const int32_t* cu_seqlens, int B, int T, int max_seqlen,
                           const int32_t* labels, float* nll_out, void* ws, size_t ws_bytes, rsb_stream_t stream) {
    if (!h || !ids || !cu_seqlens || !labels || !nll_out || !ws) return lfail(RSB_ERR_INVALID, "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<int32_t> cu, lab;
    int rc = check_forward(h, ids, cu_seqlens, labels, B, T, max_seqlen, st, cu, lab);
    if (rc != RSB_OK) return rc;
    std::vector<int32_t> rows, labs, outi;
    for (int b = 0; b < B; ++b)
        for (int t = cu[b] + 1; t < cu[b + 1]; ++t)
            if (lab[t] != -100) { rows.push_back(t - 1); labs.push_back(lab[t]); outi.push_back(t); }
    const int nl = (int)rows.size();
    size_t off[10];
    const size_t need = llm_ws_layout(h, (size_t)T, (size_t)nl, off);
    if (ws_bytes < need) return lfail(RSB_ERR_OOM, "reader workspace too small (need %ld bytes)", (long)need);
    unsigned char* w = static_cast<unsigned char*>(ws);
    int* d_rows = reinterpret_cast<int*>(w + off[7]);
    int* d_labs = d_rows + nl;
    int* d_outi = d_labs + nl;
    if (nl > 0 && (cudaMemcpyAsync(d_rows, rows.data(), (size_t)nl * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
                   cudaMemcpyAsync(d_labs, labs.data(), (size_t)nl * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
                   cudaMemcpyAsync(d_outi, outi.data(), (size_t)nl * 4, cudaMemcpyHostToDevice, st) != cudaSuccess))
        return lfail(RSB_ERR_CUDA, "uploading the label rows failed");
    if (cudaMemsetAsync(nll_out, 0, (size_t)T * sizeof(float), st) != cudaSuccess)
        return lfail(RSB_ERR_CUDA, "clearing nll_out failed");
    rc = with_dtype(h, [&](auto tag) -> int {
        using E = decltype(tag);
        int rc = trunk<E>(h, ids, cu_seqlens, B, T, cu, w, off, st);
        if (rc != RSB_OK) return rc;
        // final norm and LM head on the label rows only, in chunks that bound the logits workspace; the logits are in
        // the handle's dtype and nll_rows_kernel takes their fp32 log-sum-exp (transformers' logits.float())
        E* X = reinterpret_cast<E*>(w + off[0]);
        E* Hn = reinterpret_cast<E*>(w + off[1]);
        E* LOG = reinterpret_cast<E*>(w + off[6]);
        const int Hd = h->hidden, chunk = h->chunk_rows();
        for (int c0 = 0; c0 < nl; c0 += chunk) {
            const int n = std::min(chunk, nl - c0);
            final_norm<E>(h, X, d_rows + c0, n, Hn, st);
            if ((rc = gemm<E>(Hn, n, h->lm_head, h->vocab_pad, Hd, h->zero_bias, nullptr, LOG, 0, st)) != RSB_OK) return rc;
            nll_rows_kernel<E><<<n, 256, 0, st>>>(LOG, h->vocab, h->vocab_pad, d_labs + c0, d_outi + c0, nll_out);
        }
        return RSB_OK;
    });
    if (rc != RSB_OK) return rc;
    const cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return lfail(RSB_ERR_CUDA, "reader launch failed: %s", cudaGetErrorString(e));
    return RSB_OK;
}

namespace {

// rsb_llm_loglikelihood's workspace: the forward's slots for T tokens with up to min(n, T) scored rows, then the
// target tables: distinct rows [R], CSR offsets [R + 1], and token and output index per target [n] each.
size_t ll_layout(const rsb_llm* h, size_t T, size_t n, size_t off[10], size_t* tables) {
    const size_t R = std::min(n, T);
    *tables = llm_ws_layout(h, T, R, off);
    return *tables + (2 * R + 1 + 2 * n) * sizeof(int);
}

}  // namespace

extern "C" size_t rsb_llm_loglikelihood_workspace_bytes(rsb_llm_t* h, int T, int n_targets) {
    if (!h || T <= 0 || n_targets < 0) return 0;
    size_t off[10], tables;
    return ll_layout(h, (size_t)T, (size_t)n_targets, off, &tables);
}

// The reader forward of rsb_llm_nll, scored at caller-chosen (row, token) pairs: out_logprob[i] = log_softmax(logits of
// packed row tgt_row[i])[tgt_token[i]] in fp32 and out_greedy[i] = whether tgt_token[i] is that row's argmax.  The final
// norm and LM head run once per distinct row.
extern "C" int rsb_llm_loglikelihood(rsb_llm_t* h, const int32_t* ids, const int32_t* cu_seqlens, int B, int T,
                                     int max_seqlen, const int32_t* tgt_row, const int32_t* tgt_token, int n_targets,
                                     float* out_logprob, int32_t* out_greedy, void* ws, size_t ws_bytes,
                                     rsb_stream_t stream) {
    if (!h || !ids || !cu_seqlens || !ws || (n_targets > 0 && (!tgt_row || !tgt_token || !out_logprob || !out_greedy)))
        return lfail(RSB_ERR_INVALID, "null argument");
    if (n_targets < 0) return lfail(RSB_ERR_INVALID, "n_targets %ld is negative", (long)n_targets);
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<int32_t> cu, lab;
    int rc = check_forward(h, ids, cu_seqlens, nullptr, B, T, max_seqlen, st, cu, lab);
    if (rc != RSB_OK) return rc;
    const int n = n_targets;
    std::vector<int32_t> row(n), tok(n);
    if (n > 0 && (cudaMemcpyAsync(row.data(), tgt_row, (size_t)n * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
                  cudaMemcpyAsync(tok.data(), tgt_token, (size_t)n * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
                  cudaStreamSynchronize(st) != cudaSuccess))
        return lfail(RSB_ERR_CUDA, "reading back the targets failed");
    for (int i = 0; i < n; ++i) {
        if (row[i] < 0 || row[i] >= T)
            return lfail(RSB_ERR_INVALID, "target %ld: row %ld is outside [0, T = %ld)", (long)i, (long)row[i], (long)T);
        if (tok[i] < 0 || tok[i] >= h->vocab)
            return lfail(RSB_ERR_INVALID, "target %ld: token %ld is outside the vocabulary", (long)i, (long)tok[i]);
    }
    size_t off[10], tables;
    const size_t need = ll_layout(h, (size_t)T, (size_t)n, off, &tables);
    if (ws_bytes < need) return lfail(RSB_ERR_OOM, "reader workspace too small (need %ld bytes)", (long)need);
    if (n == 0) return RSB_OK;
    // targets sorted by row: distinct rows, and per row a CSR run of (token, output index)
    std::vector<int32_t> order(n), rows, ptr{0}, stok(n), sout(n);
    for (int i = 0; i < n; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return row[a] < row[b]; });
    for (int j = 0; j < n; ++j) {
        const int i = order[j];
        if (rows.empty() || rows.back() != row[i]) {
            if (!rows.empty()) ptr.push_back(j);
            rows.push_back(row[i]);
        }
        stok[j] = tok[i];
        sout[j] = i;
    }
    ptr.push_back(n);
    const int R = (int)rows.size();
    unsigned char* w = static_cast<unsigned char*>(ws);
    int* d_rows = reinterpret_cast<int*>(w + tables);
    int* d_ptr = d_rows + R;
    int* d_tok = d_ptr + R + 1;
    int* d_out = d_tok + n;
    if (cudaMemcpyAsync(d_rows, rows.data(), (size_t)R * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(d_ptr, ptr.data(), (size_t)(R + 1) * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(d_tok, stok.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemcpyAsync(d_out, sout.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st) != cudaSuccess)
        return lfail(RSB_ERR_CUDA, "uploading the targets failed");
    rc = with_dtype(h, [&](auto tag) -> int {
        using E = decltype(tag);
        int rc = trunk<E>(h, ids, cu_seqlens, B, T, cu, w, off, st);
        if (rc != RSB_OK) return rc;
        // final norm and LM head on the distinct rows only, in rsb_llm_nll's chunks
        E* X = reinterpret_cast<E*>(w + off[0]);
        E* Hn = reinterpret_cast<E*>(w + off[1]);
        E* LOG = reinterpret_cast<E*>(w + off[6]);
        const int Hd = h->hidden, chunk = h->chunk_rows();
        for (int c0 = 0; c0 < R; c0 += chunk) {
            const int m = std::min(chunk, R - c0);
            final_norm<E>(h, X, d_rows + c0, m, Hn, st);
            if ((rc = gemm<E>(Hn, m, h->lm_head, h->vocab_pad, Hd, h->zero_bias, nullptr, LOG, 0, st)) != RSB_OK) return rc;
            choice_rows_kernel<E><<<m, 256, 0, st>>>(LOG, h->vocab, h->vocab_pad, d_ptr + c0, d_tok, d_out, out_logprob,
                                                     out_greedy);
        }
        return RSB_OK;
    });
    if (rc != RSB_OK) return rc;
    const cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return lfail(RSB_ERR_CUDA, "reader launch failed: %s", cudaGetErrorString(e));
    return RSB_OK;
}

// Diagnostic: the residual stream after the last layer (before the final norm) of the same forward, [T, hidden] in the
// handle's dtype.
extern "C" int rsb_llm_hidden_states(rsb_llm_t* h, const int32_t* ids, const int32_t* cu_seqlens, int B, int T,
                                     int max_seqlen, void* out, void* ws, size_t ws_bytes, rsb_stream_t stream) {
    if (!h || !ids || !cu_seqlens || !out || !ws) return lfail(RSB_ERR_INVALID, "null argument");
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<int32_t> cu, lab;
    int rc = check_forward(h, ids, cu_seqlens, nullptr, B, T, max_seqlen, st, cu, lab);
    if (rc != RSB_OK) return rc;
    size_t off[10];
    const size_t need = llm_ws_layout(h, (size_t)T, 0, off);
    if (ws_bytes < need) return lfail(RSB_ERR_OOM, "reader workspace too small (need %ld bytes)", (long)need);
    unsigned char* w = static_cast<unsigned char*>(ws);
    rc = with_dtype(h, [&](auto tag) -> int { return trunk<decltype(tag)>(h, ids, cu_seqlens, B, T, cu, w, off, st); });
    if (rc != RSB_OK) return rc;
    if (cudaMemcpyAsync(out, w + off[0], (size_t)T * h->hidden * 2, cudaMemcpyDeviceToDevice, st) != cudaSuccess)
        return lfail(RSB_ERR_CUDA, "copying the hidden states failed");
    const cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return lfail(RSB_ERR_CUDA, "reader launch failed: %s", cudaGetErrorString(e));
    return RSB_OK;
}

namespace {

// rsb_llm_generate's workspace: the forward's slots for the T context tokens with B label rows (every decode step runs
// at most B rows through the same slots), then the KV cache, the split-KV partials and four int tables of B entries
// (slot, position, id and chosen id of each decode row).  The cache holds max_seqlen + max_new_tokens - 1 positions per
// slot: the last chosen token is never fed back.
struct GenLayout {
    size_t off[10], k, v, part_o, part_ml, ints, total;
    int cap, chunks;
};
GenLayout gen_layout(const rsb_llm* h, size_t B, size_t T, int max_seqlen, int max_new_tokens) {
    auto al = [](size_t x) { return (x + 1023) / 1024 * 1024; };
    GenLayout g;
    size_t o = llm_ws_layout(h, T, B, g.off);
    g.cap = max_seqlen + max_new_tokens - 1;
    g.chunks = (g.cap + DCH - 1) / DCH;
    const size_t kv_bytes = (size_t)h->layers * B * h->kv_heads * (size_t)g.cap * h->head_dim * 2;
    const size_t parts = B * h->heads * (size_t)g.chunks;
    g.k = o; o += al(kv_bytes);
    g.v = o; o += al(kv_bytes);
    g.part_o = o; o += al(parts * h->head_dim * sizeof(float));
    g.part_ml = o; o += al(parts * sizeof(float2));
    g.ints = o; o += al(4 * B * sizeof(int));
    g.total = o;
    return g;
}

}  // namespace

extern "C" size_t rsb_llm_generate_workspace_bytes(rsb_llm_t* h, int B, int T, int max_seqlen, int max_new_tokens) {
    if (!h || B <= 0 || T <= 0 || max_seqlen <= 0 || max_new_tokens <= 0) return 0;
    return gen_layout(h, (size_t)B, (size_t)T, max_seqlen, max_new_tokens).total;
}

// Greedy decoding of HF `model.generate(do_sample=False, num_beams=1)` from B packed contexts (rsb.h): a prefill over
// the contexts that fills the KV cache and chooses each sequence's first token, then one decode step per token for the
// sequences still running, through the same layer loops at M = live rows.  One read-back of the chosen ids per step.
extern "C" int rsb_llm_generate(rsb_llm_t* h, const int32_t* ids, const int32_t* cu_seqlens, int B, int T, int max_seqlen,
                                int max_new_tokens, const int32_t* eos_ids, int n_eos, int32_t* out_tokens,
                                int32_t* out_lens, float* out_logprob, void* ws, size_t ws_bytes, rsb_stream_t stream) {
    if (!h || !ids || !cu_seqlens || !out_tokens || !out_lens || !ws || (n_eos > 0 && !eos_ids))
        return lfail(RSB_ERR_INVALID, "null argument");
    if (max_new_tokens <= 0 || n_eos < 0) return lfail(RSB_ERR_INVALID, "max_new_tokens must be positive and n_eos >= 0");
    if ((long long)max_seqlen + max_new_tokens > h->max_pos)
        return lfail(RSB_ERR_UNSUPPORTED, "a context of %ld tokens plus %ld new tokens is longer than "
                     "max_position_embeddings (%ld)", (long)max_seqlen, (long)max_new_tokens, (long)h->max_pos);
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<int32_t> cu, lab;
    int rc = check_forward(h, ids, cu_seqlens, nullptr, B, T, max_seqlen, st, cu, lab);
    if (rc != RSB_OK) return rc;
    for (int b = 0; b < B; ++b)
        if (cu[b + 1] == cu[b]) return lfail(RSB_ERR_INVALID, "context %ld is empty", (long)b);
    const GenLayout g = gen_layout(h, (size_t)B, (size_t)T, max_seqlen, max_new_tokens);
    if (ws_bytes < g.total) return lfail(RSB_ERR_OOM, "generate workspace too small (need %ld bytes)", (long)g.total);
    unsigned char* w = static_cast<unsigned char*>(ws);
    int* d_rows = reinterpret_cast<int*>(w + g.off[7]);
    int* d_ints = reinterpret_cast<int*>(w + g.ints);   // slot | pos | ids of n decode rows, then next at 3B
    int* d_next = d_ints + 3 * (size_t)B;
    std::vector<int32_t> ctx(B), rows(B);
    for (int b = 0; b < B; ++b) { ctx[b] = cu[b + 1] - cu[b]; rows[b] = cu[b + 1] - 1; }
    const size_t n_out = (size_t)B * max_new_tokens;
    if (cudaMemcpyAsync(d_rows, rows.data(), (size_t)B * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaMemsetAsync(out_tokens, 0xFF, n_out * 4, st) != cudaSuccess ||
        (out_logprob && cudaMemsetAsync(out_logprob, 0, n_out * 4, st) != cudaSuccess))
        return lfail(RSB_ERR_CUDA, "initialising the generate buffers failed");
    const std::vector<int32_t> eos(eos_ids, eos_ids + std::max(n_eos, 0));
    auto ends = [&](int tok, int len) { return len == max_new_tokens || std::find(eos.begin(), eos.end(), tok) != eos.end(); };
    std::vector<int32_t> tok(B), lens(B, 0), next(B), host(3 * (size_t)B), live;
    rc = with_dtype(h, [&](auto tag) -> int {
        using E = decltype(tag);
        KvCache<E> kv;
        kv.k = reinterpret_cast<E*>(w + g.k);
        kv.v = reinterpret_cast<E*>(w + g.v);
        kv.slots = B;
        kv.cap = g.cap;
        E* X = reinterpret_cast<E*>(w + g.off[0]);
        E* Hn = reinterpret_cast<E*>(w + g.off[1]);
        E* LOG = reinterpret_cast<E*>(w + g.off[6]);
        const int Hd = h->hidden, chunk = h->chunk_rows();
        // final norm, LM head and greedy choice of n rows (X rows[i], or X row i), read back into next
        auto choose = [&](const int* d_r, int n, const int* slot, int step) -> int {
            int rc;
            for (int c0 = 0; c0 < n; c0 += chunk) {
                const int m = std::min(chunk, n - c0);
                final_norm<E>(h, d_r ? X : X + (size_t)c0 * Hd, d_r ? d_r + c0 : nullptr, m, Hn, st);
                if ((rc = gemm<E>(Hn, m, h->lm_head, h->vocab_pad, Hd, h->zero_bias, nullptr, LOG, 0, st)) != RSB_OK) return rc;
                greedy_rows_kernel<E><<<m, 256, 0, st>>>(LOG, h->vocab, h->vocab_pad, slot ? slot + c0 : nullptr, c0, step,
                                                         max_new_tokens, d_next + c0, out_tokens, out_logprob);
            }
            if (cudaMemcpyAsync(next.data(), d_next, (size_t)n * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
                cudaStreamSynchronize(st) != cudaSuccess)
                return lfail(RSB_ERR_CUDA, "generate step failed: %s", cudaGetErrorString(cudaGetLastError()));
            return RSB_OK;
        };
        int rc = trunk<E>(h, ids, cu_seqlens, B, T, cu, w, g.off, st, &kv);
        if (rc != RSB_OK || (rc = choose(d_rows, B, nullptr, 0)) != RSB_OK) return rc;
        for (int b = 0; b < B; ++b) {
            tok[b] = next[b];
            lens[b] = 1;
            if (!ends(tok[b], 1)) live.push_back(b);
        }
        for (int step = 1; step < max_new_tokens && !live.empty(); ++step) {
            const int n = (int)live.size();
            int max_p = 0;
            for (int i = 0; i < n; ++i) {
                const int b = live[i];
                host[i] = b;
                host[n + i] = ctx[b] + step - 1;   // the token chosen at step - 1 sits right after the previous one
                host[2 * n + i] = tok[b];
                max_p = std::max(max_p, host[n + i]);
            }
            if (cudaMemcpyAsync(d_ints, host.data(), (size_t)3 * n * 4, cudaMemcpyHostToDevice, st) != cudaSuccess)
                return lfail(RSB_ERR_CUDA, "uploading the decode rows failed");
            kv.slot = d_ints;
            kv.pos = d_ints + n;
            kv.chunks = max_p / DCH + 1;
            kv.part_o = reinterpret_cast<float*>(w + g.part_o);
            kv.part_ml = reinterpret_cast<float2*>(w + g.part_ml);
            if ((rc = trunk<E>(h, d_ints + 2 * n, nullptr, n, n, cu, w, g.off, st, &kv)) != RSB_OK) return rc;
            if ((rc = choose(nullptr, n, d_ints, step)) != RSB_OK) return rc;
            std::vector<int32_t> still;
            for (int i = 0; i < n; ++i) {
                const int b = live[i];
                tok[b] = next[i];
                lens[b] = step + 1;
                if (!ends(tok[b], step + 1)) still.push_back(b);
            }
            live.swap(still);
        }
        return RSB_OK;
    });
    if (rc != RSB_OK) return rc;
    if (cudaMemcpyAsync(out_lens, lens.data(), (size_t)B * 4, cudaMemcpyHostToDevice, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess)
        return lfail(RSB_ERR_CUDA, "writing out_lens failed");
    const cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return lfail(RSB_ERR_CUDA, "generate launch failed: %s", cudaGetErrorString(e));
    return RSB_OK;
}

// Diagnostic: one attention step of the forward on a caller's fused QKV rows [T, (heads + 2 kv_heads) head_dim] in the
// handle's dtype (GPT-NeoX: [Q heads | K heads | V heads], as rsb_llm_load permutes query_key_value).
extern "C" int rsb_llm_attention(rsb_llm_t* h, void* qkv, const int32_t* cu_seqlens, int B, int T, int max_seqlen,
                                 void* ctx, rsb_stream_t stream) {
    if (!h || !qkv || !cu_seqlens || !ctx) return lfail(RSB_ERR_INVALID, "null argument");
    if (B <= 0 || T <= 0) return lfail(RSB_ERR_INVALID, "empty batch");
    if (max_seqlen > h->max_pos)
        return lfail(RSB_ERR_UNSUPPORTED, "sequence longer than max_position_embeddings (%ld)", (long)h->max_pos);
    if (h->family == RSB_LLM_OLMO2 && !(h->loaded.count("model.layers.0.self_attn.q_norm.weight") &&
                          h->loaded.count("model.layers.0.self_attn.k_norm.weight")))
        return lfail(RSB_ERR_STATE, "layer 0's self_attn.q_norm / k_norm weights are not loaded");
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<int32_t> cu(B + 1);
    if (cudaMemcpyAsync(cu.data(), cu_seqlens, cu.size() * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess)
        return lfail(RSB_ERR_CUDA, "reading back cu_seqlens failed");
    int rc = check_offsets(cu, B, T, max_seqlen);
    if (rc != RSB_OK) return rc;
    int2* d_items = nullptr;
    if (cu[B] > 0 && cudaMallocAsync(&d_items, (size_t)cu[B] * sizeof(int2), st) != cudaSuccess)
        return lfail(RSB_ERR_OOM, "allocating the attention work list failed");
    int n_items = 0;
    rc = upload_attention_items(cu, B, d_items, st, &n_items);
    if (rc == RSB_OK)
        with_dtype(h, [&](auto tag) -> int {
            using E = decltype(tag);
            attention_step<E>(h, 0, static_cast<E*>(qkv), cu_seqlens, B, cu[B], d_items, n_items,
                              static_cast<E*>(ctx), nullptr, st);
            return RSB_OK;
        });
    if (d_items) cudaFreeAsync(d_items, st);
    if (rc != RSB_OK) return rc;
    const cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return lfail(RSB_ERR_CUDA, "attention launch failed: %s", cudaGetErrorString(e));
    return RSB_OK;
}

// Diagnostic: one decode step of attention_step on caller-owned rows and one layer's KV cache (rsb.h).  The slots and
// positions are read back and checked first, so every launch stays inside the caller's buffers.  The split-KV partials
// are allocated here and filled with NaN bytes: a chunk read without having been written shows up in ctx.
extern "C" int rsb_llm_decode_attention(rsb_llm_t* h, void* qkv, const int32_t* slot, const int32_t* pos, int n_rows,
                                        void* k_cache, void* v_cache, int slots, int cap, void* ctx,
                                        rsb_stream_t stream) {
    if (!h || !qkv || !slot || !pos || !k_cache || !v_cache || !ctx) return lfail(RSB_ERR_INVALID, "null argument");
    if (n_rows <= 0 || slots <= 0 || cap <= 0) return lfail(RSB_ERR_INVALID, "n_rows, slots and cap must be positive");
    for (const void* p : {(const void*)qkv, (const void*)k_cache, (const void*)v_cache, (const void*)ctx})
        if (reinterpret_cast<uintptr_t>(p) % 16)
            return lfail(RSB_ERR_INVALID, "qkv, the caches and ctx must be 16-byte aligned");
    if (h->family == RSB_LLM_OLMO2 && !(h->loaded.count("model.layers.0.self_attn.q_norm.weight") &&
                                        h->loaded.count("model.layers.0.self_attn.k_norm.weight")))
        return lfail(RSB_ERR_STATE, "layer 0's self_attn.q_norm / k_norm weights are not loaded");
    cudaStream_t st = (cudaStream_t)stream;
    std::vector<int32_t> hs(n_rows), hp(n_rows);
    if (cudaMemcpyAsync(hs.data(), slot, (size_t)n_rows * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaMemcpyAsync(hp.data(), pos, (size_t)n_rows * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess)
        return lfail(RSB_ERR_CUDA, "reading back slot / pos failed");
    std::vector<char> used(slots, 0);
    int max_p = 0;
    for (int i = 0; i < n_rows; ++i) {
        if (hs[i] < 0 || hs[i] >= slots)
            return lfail(RSB_ERR_INVALID, "slot %ld of row %ld is outside [0, slots = %ld)", (long)hs[i], (long)i, (long)slots);
        if (used[hs[i]]) return lfail(RSB_ERR_INVALID, "two rows on slot %ld", (long)hs[i]);
        used[hs[i]] = 1;
        if (hp[i] < 0 || hp[i] >= cap)
            return lfail(RSB_ERR_INVALID, "position %ld of row %ld is outside [0, cap = %ld)", (long)hp[i], (long)i, (long)cap);
        if (hp[i] >= h->max_pos)
            return lfail(RSB_ERR_UNSUPPORTED, "position %ld is past max_position_embeddings (%ld)", (long)hp[i],
                         (long)h->max_pos);
        max_p = std::max(max_p, hp[i]);
    }
    const int chunks = max_p / DCH + 1;
    const size_t parts = (size_t)n_rows * h->heads * chunks;
    float* part_o = nullptr;
    float2* part_ml = nullptr;
    if (cudaMallocAsync(&part_o, parts * h->head_dim * sizeof(float), st) != cudaSuccess ||
        cudaMallocAsync(&part_ml, parts * sizeof(float2), st) != cudaSuccess) {
        if (part_o) cudaFreeAsync(part_o, st);
        return lfail(RSB_ERR_OOM, "allocating the split-KV partials failed");
    }
    int rc = RSB_OK;
    if (cudaMemsetAsync(part_o, 0xFF, parts * h->head_dim * sizeof(float), st) != cudaSuccess ||
        cudaMemsetAsync(part_ml, 0xFF, parts * sizeof(float2), st) != cudaSuccess)
        rc = lfail(RSB_ERR_CUDA, "filling the split-KV partials failed");
    if (rc == RSB_OK)
        with_dtype(h, [&](auto tag) -> int {
            using E = decltype(tag);
            KvCache<E> kv;
            kv.k = static_cast<E*>(k_cache);
            kv.v = static_cast<E*>(v_cache);
            kv.slots = slots;
            kv.cap = cap;
            kv.slot = slot;
            kv.pos = pos;
            kv.part_o = part_o;
            kv.part_ml = part_ml;
            kv.chunks = chunks;
            attention_step<E>(h, 0, static_cast<E*>(qkv), nullptr, 0, n_rows, nullptr, 0, static_cast<E*>(ctx), &kv, st);
            return RSB_OK;
        });
    cudaFreeAsync(part_o, st);
    cudaFreeAsync(part_ml, st);
    if (rc != RSB_OK) return rc;
    const cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return lfail(RSB_ERR_CUDA, "decode attention launch failed: %s", cudaGetErrorString(e));
    return RSB_OK;
}

// Diagnostic: greedy_rows_kernel on a caller's logits (rsb.h).  next and out_tokens are both ids: with slot = nullptr,
// base 0, step 0 and max_new 1, row i writes the same id to the same element through each.
extern "C" int rsb_llm_greedy(int dtype, const void* logits, int vocab, int ld, int n_rows, int32_t* ids,
                              float* logprob, rsb_stream_t stream) {
    if (dtype != RSB_DTYPE_F16 && dtype != RSB_DTYPE_BF16)
        return lfail(RSB_ERR_INVALID, "dtype %ld is neither RSB_DTYPE_F16 nor RSB_DTYPE_BF16", (long)dtype);
    if (!logits || !ids || !logprob) return lfail(RSB_ERR_INVALID, "null argument");
    if (vocab <= 0 || ld < vocab || ld % 8 || n_rows < 0)
        return lfail(RSB_ERR_INVALID, "vocab must be positive, ld >= vocab and a multiple of 8, n_rows >= 0");
    if (reinterpret_cast<uintptr_t>(logits) % 16) return lfail(RSB_ERR_INVALID, "logits must be 16-byte aligned");
    if (n_rows == 0) return RSB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    if (dtype == RSB_DTYPE_BF16)
        greedy_rows_kernel<__nv_bfloat16><<<n_rows, 256, 0, st>>>(static_cast<const __nv_bfloat16*>(logits), vocab, ld,
                                                                  nullptr, 0, 0, 1, ids, ids, logprob);
    else
        greedy_rows_kernel<__half><<<n_rows, 256, 0, st>>>(static_cast<const __half*>(logits), vocab, ld, nullptr, 0, 0,
                                                           1, ids, ids, logprob);
    const cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return lfail(RSB_ERR_CUDA, "greedy launch failed: %s", cudaGetErrorString(e));
    return RSB_OK;
}

// Diagnostic: ln_rows_kernel, the GPT-NeoX LayerNorm step of the forward, on a caller's rows (rsb.h).
extern "C" int rsb_llm_layernorm(int hidden, float eps, void* x, const void* add, const int32_t* rows, int n_rows,
                                 const void* w1, const void* b1, const void* w2, const void* b2, void* out1, void* out2,
                                 rsb_stream_t stream) {
    if (!x || (w1 && (!b1 || !out1)) || (w2 && (!b2 || !out2)) || (!w1 && w2))
        return lfail(RSB_ERR_INVALID, "null argument (x, or a norm's bias or output, or w2 without w1)");
    if (n_rows < 0 || !(eps > 0.f)) return lfail(RSB_ERR_INVALID, "n_rows must be >= 0 and eps positive");
    if (hidden <= 0 || hidden % 8 || hidden > LN_MAX_HIDDEN)
        return lfail(RSB_ERR_UNSUPPORTED, "hidden %ld: the LayerNorm kernel takes multiples of 8 up to %ld", (long)hidden,
                     (long)LN_MAX_HIDDEN);
    if (n_rows == 0) return RSB_OK;
    auto h16 = [](const void* p) { return static_cast<const __half*>(p); };
    ln_rows_kernel<__half><<<n_rows, LN_THREADS, 0, (cudaStream_t)stream>>>(
        static_cast<__half*>(x), h16(add), rows, hidden, h16(w1), h16(b1), h16(w2), h16(b2), eps,
        static_cast<__half*>(out1), static_cast<__half*>(out2));
    const cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return lfail(RSB_ERR_CUDA, "layernorm launch failed: %s", cudaGetErrorString(e));
    return RSB_OK;
}

// Diagnostic: rms_rows_kernel in OLMo-2's order, the post-norm residual add and final norm, on a caller's rows (rsb.h).
extern "C" int rsb_llm_olmo2_norm(int hidden, float eps, void* x, const void* a, const int32_t* rows, int n_rows,
                                  const void* w, void* out, rsb_stream_t stream) {
    if (!x || !w || (!a && !out)) return lfail(RSB_ERR_INVALID, "null argument (x, w, or out without a)");
    if (n_rows < 0 || !(eps > 0.f)) return lfail(RSB_ERR_INVALID, "n_rows must be >= 0 and eps positive");
    if (hidden <= 0 || hidden % 8)
        return lfail(RSB_ERR_UNSUPPORTED, "hidden %ld: the RMSNorm kernel takes positive multiples of 8", (long)hidden);
    if (n_rows == 0) return RSB_OK;
    rms_rows_kernel<__half, true><<<n_rows, 256, 0, (cudaStream_t)stream>>>(
        static_cast<__half*>(x), static_cast<const __half*>(a), rows, hidden, static_cast<const __half*>(w), eps,
        static_cast<__half*>(out));
    const cudaError_t e = cudaPeekAtLastError();
    if (e != cudaSuccess) return lfail(RSB_ERR_CUDA, "rmsnorm launch failed: %s", cudaGetErrorString(e));
    return RSB_OK;
}
