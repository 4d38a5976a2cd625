"""fp64 ORACLE (test infrastructure, NOT product code) of one attention step of the encoder, on the un-padded token
stream that `rsb_bert_attention` takes: qkv [T, 2304] fp16 (each token's Q | K | V, 12 heads of 64) and cu_seqlens
[B + 1].  Per sequence and head:

  BERT form (HF BertSelfAttention):  ctx = softmax(q k^T / 8) v
  T5 form (HF T5Attention in fp16):  scores = fp16(fp16(q k^T) + bias[h][key - query])   (no scaling)
                                     ctx = softmax(scores) v

Everything else is exact (fp64): the only roundings kept are the two fp16 roundings of the T5 score, the points at
which HF's fp16 T5 rounds (`torch.matmul` of halves, then the half `+=` of position_bias).  The dot products q.k of
fp16 operands are exact in fp64 (64 products of 11-bit significands).

`attention(..., with_bound=True)` also returns a per-element error bound for a kernel that computes the scores with
fp32 accumulation, the softmax in fp32 with hardware exp2, rounds the probabilities to fp16 before P.V and rounds its
output to fp16 (see `attention` for the terms).  The keyword arguments `scale`, `rel_sign`, `head_shift` and
`drop_last_key` build deliberately wrong references, used by the tests to show that their comparisons discriminate.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import t5_oracle

HEADS, HEAD_DIM, HIDDEN = 12, 64, 768
MAX_REL = 511                                  # relative positions -511..511: every pair of a 512-token sequence


def round16(x):
    """Round-to-nearest-even to fp16, back in float64."""
    return np.asarray(x, dtype=np.float64).astype(np.float16).astype(np.float64)


def ulp16(x):
    """Spacing of fp16 at |x| (2^-24 in the subnormal range)."""
    a = np.abs(np.asarray(x, dtype=np.float64))
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return np.exp2(np.maximum(e, -14.0) - 10.0)


def t5_buckets(num_buckets: int, max_distance: int) -> np.ndarray:
    """int [1023]: the bucket of r = key - query at r + 511, by `t5_oracle.relative_position_bucket`."""
    r = torch.arange(-MAX_REL, MAX_REL + 1)
    return t5_oracle.relative_position_bucket(r, num_buckets, max_distance).numpy()


def t5_bias_table(rel_weight, buckets) -> np.ndarray:
    """float64 [heads, 1023]: bias of head h at relative position r = key - query, index r + 511, from the fp16
    relative_attention_bias weight [num_buckets, heads] and a bucket table [1023]."""
    w = np.asarray(rel_weight, dtype=np.float16).astype(np.float64)
    return w[np.asarray(buckets)].T.copy()


def attention(qkv, cu_seqlens, form: str = "bert", bias=None, *, scale: float = 0.125, rel_sign: int = 1,
              head_shift: int = 0, drop_last_key: bool = False, with_bound: bool = False):
    """ctx [T, 768] float64 (rows of zero-length sequences stay 0), or (ctx, bound) with `with_bound`.

    bound[t, c] is the largest |kernel - ctx| a correct kernel can show at that element:
      (2^-11 + (S + 32) 2^-24) E       the fp16 rounding of each probability before P.V (relative 2^-11), plus the fp32
                                       accumulation of P.V and of the flash kernel's rescaling products; E = sum_j p_j |v_j|
      + S 2^-25 vmax                   probabilities below the fp16 normal range (absolute 2^-25 each)
      + 2 a (E + |ctx|)                a relative error `a` of each exp: hardware exp2 (2^-20), the fp32 rounding of the
                                       exponent argument (2^-22 max|s|), the fp32 sum of S exps (S 2^-24) and, for the
                                       BERT form, the fp32 accumulation of q.k (64 2^-23 sum|q||k| / 8)
      + sum_j p_j w_j (|v_j| + |ctx|)  T5 only: a score whose fp32 q.k (or fp32 bias sum) may round to the other fp16
                                       neighbour than the exact value does moves by up to w_j = ulp(q.k) + ulp(score)
      + 1/2 ulp_fp16                   the rounding of the output.
    The scores of the Q/K arm with small multiples of 1/4 are exact in fp32, so only the first, second and last terms
    remain there and the bound is tight."""
    qkv = np.asarray(qkv)
    assert qkv.dtype == np.float16 and qkv.shape[1] == 3 * HIDDEN
    cu = np.asarray(cu_seqlens, dtype=np.int64)
    T = int(cu[-1])
    lens = np.diff(cu)
    out = np.zeros((T, HIDDEN))
    bnd = np.zeros((T, HIDDEN)) if with_bound else None
    hsel = (np.arange(HEADS) + head_shift) % HEADS
    for S in np.unique(lens):
        S = int(S)
        if S == 0:
            continue
        seqs = np.nonzero(lens == S)[0]
        chunk = max(1, int(2e7 // (HEADS * S * S)))
        for c0 in range(0, len(seqs), chunk):
            sel = seqs[c0:c0 + chunk]
            n = len(sel)
            rows = cu[sel][:, None] + np.arange(S)[None, :]                        # [n, S]
            x = qkv[rows].astype(np.float64)
            q, k, v = (x[..., i * HIDDEN:(i + 1) * HIDDEN].reshape(n, S, HEADS, HEAD_DIM).transpose(0, 2, 1, 3)
                       for i in range(3))                                          # [n, 12, S, 64]
            s = q @ k.transpose(0, 1, 3, 2)                                        # exact
            amb_w = None
            if form == "bert":
                sc = s * scale
            elif form == "t5":
                r = (np.arange(S)[None, :] - np.arange(S)[:, None]) * rel_sign     # key - query
                bb = np.asarray(bias, dtype=np.float64)[hsel][:, r + MAX_REL]      # [12, S, S]
                s16 = round16(s)
                sc = round16(s16 + bb[None])
                if with_bound:
                    dq = 64 * 2.0 ** -23 * (np.abs(q) @ np.abs(k).transpose(0, 1, 3, 2))
                    amb = (round16(s - dq) != round16(s + dq))
                    sb = s16 + bb[None]
                    amb |= round16(sb * (1 - 2.0 ** -23)) != round16(sb * (1 + 2.0 ** -23))
                    amb_w = np.where(amb, ulp16(s) + ulp16(sc), 0.0)
            else:
                raise ValueError(form)
            if drop_last_key and S > 1:
                sc = sc.copy()
                sc[..., -1] = -np.inf
            m = sc.max(-1, keepdims=True)
            e = np.exp(sc - m)
            p = e / e.sum(-1, keepdims=True)
            o = p @ v
            out[rows] = o.transpose(0, 2, 1, 3).reshape(n, S, HIDDEN)
            if with_bound:
                av = np.abs(v)
                E = p @ av
                vmax = av.max(2, keepdims=True)
                a = 2.0 ** -20 + 2.0 ** -22 * np.abs(sc).max(-1, keepdims=True) + S * 2.0 ** -24
                if form == "bert":
                    a = a + scale * 64 * 2.0 ** -23 * (np.abs(q) @ np.abs(k).transpose(0, 1, 3, 2)).max(-1, keepdims=True)
                b = (2.0 ** -11 + (S + 32) * 2.0 ** -24) * E + S * 2.0 ** -25 * vmax + 2 * a * (E + np.abs(o))
                if amb_w is not None:
                    pw = p * amb_w
                    b = b + pw @ av + pw.sum(-1, keepdims=True) * np.abs(o)
                b = b + 0.5 * ulp16(np.abs(o) + b)
                bnd[rows] = b.transpose(0, 2, 1, 3).reshape(n, S, HIDDEN)
    return (out, bnd) if with_bound else out
