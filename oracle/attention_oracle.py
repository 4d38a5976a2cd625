"""fp64 ORACLE (test infrastructure, NOT product code) of one attention step of the encoder and of the Llama reader.

Encoder (`attention`): one attention step of the encoder, on the un-padded token
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

Reader (`rope_f16`, `causal_attention`): the step `rsb_llm_attention` takes, on fused rows [T, (heads + 2 kv_heads) 128]
of Q | K | V heads with head_dim 128.  `rope_f16` restates HF apply_rotary_pos_emb in fp16 (positions restart in every
window); `causal_attention` is causal softmax(q k^T / sqrt(128)) v per window in fp64 with grouped-query heads (query
head h reads KV head h // (heads / kv_heads), HF's repeat_kv) and a per-element bound of the same terms as the encoder's.
Both run on torch tensors on any device, so that the reference of production-width cases runs where the kernel does.
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


# ---------------------------------------------------------------------------------------------------------------
# reader: RoPE and causal grouped-query attention, head_dim 128
# ---------------------------------------------------------------------------------------------------------------
LLAMA_HEAD_DIM = 128


def window_positions(cu_seqlens, T: int) -> np.ndarray:
    """int64 [T]: the position of every row inside its window (0 at every window start); rows at or past cu[-1] get
    -1."""
    cu = np.asarray(cu_seqlens, dtype=np.int64)
    pos = np.full(T, -1, np.int64)
    for b in range(len(cu) - 1):
        pos[cu[b]:cu[b + 1]] = np.arange(cu[b + 1] - cu[b])
    return pos


def _r16(x):
    return x.to(torch.float16).to(torch.float64)


def _ulp16_t(x):
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e.clamp_min(-14) - 10)


def rope_f16(x, pos, theta: float, *, pairing: str = "half", angles: str = "fp32", cs_shift=(0, 0)):
    """HF LlamaRotaryEmbedding + apply_rotary_pos_emb on fp16 heads x [n, nh, 128] at integer positions pos [n], in
    HF's order: inv_freq = 1 / theta ** (arange(0, 128, 2) / 128) and the angles inv_freq * pos in fp32, cos / sin of
    the fp32 angle rounded to fp16, then x * cos + rotate_half(x) * sin with every product and the sum rounded to fp16.
    Returns (fp16 [n, nh, 128], bool [n, 1, 128] `near`): `near` marks the elements whose cos or sin lies within 2 fp32
    ulp of an fp16 rounding boundary, where an fp32 cos / sin that is correct to 2 ulp may round to the other fp16
    neighbour.  cs_shift = (i, j) in {-1, 0, 1}^2 moves cos / sin by i / j times 2 fp32 ulp before the fp16 rounding:
    over the nine shifts, the flagged elements take every result such a cos / sin can give.

    Deliberately wrong forms for the tests: pairing="adjacent" rotates the pairs (2i, 2i + 1) (GPT-J) instead of
    rotate_half; angles="fp64" computes inv_freq and the angles in fp64."""
    dev = x.device
    posd = torch.as_tensor(np.asarray(pos), dtype=torch.float64, device=dev)
    if angles == "fp32":
        # on the host, as HF builds the inv_freq buffer (a device pow may round some frequencies differently)
        inv = (1.0 / (theta ** (torch.arange(0, 128, 2, dtype=torch.int64).float() / 128))).double().to(dev)
        f = (posd[:, None] * inv[None, :]).float().double()               # one fp32 product: exact in fp64, rounded
    elif angles == "fp64":
        inv = 1.0 / (theta ** (torch.arange(0, 128, 2, dtype=torch.float64, device=dev) / 128))
        f = posd[:, None] * inv[None, :]
    else:
        raise ValueError(angles)
    c64, s64 = torch.cos(f), torch.sin(f)                                 # [n, 64]
    ulp32 = lambda v: torch.exp2(torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -126))) - 23)   # noqa: E731
    c, s = _r16(c64 + 2 * cs_shift[0] * ulp32(c64)), _r16(s64 + 2 * cs_shift[1] * ulp32(s64))
    near64 = ((_r16(c64 - 2 * ulp32(c64)) != _r16(c64 + 2 * ulp32(c64)))
              | (_r16(s64 - 2 * ulp32(s64)) != _r16(s64 + 2 * ulp32(s64))))
    xd = x.to(torch.float64)
    if pairing == "half":
        x1, x2 = xd[..., :64], xd[..., 64:]
        cc, ss = c[:, None, :], s[:, None, :]
        o1 = _r16(_r16(x1 * cc) + _r16(-x2 * ss))
        o2 = _r16(_r16(x2 * cc) + _r16(x1 * ss))
        out = torch.cat((o1, o2), dim=-1)
        near = torch.cat((near64, near64), dim=-1)[:, None, :]
    elif pairing == "adjacent":
        x1, x2 = xd[..., 0::2], xd[..., 1::2]
        cc, ss = c[:, None, :], s[:, None, :]
        o1 = _r16(_r16(x1 * cc) + _r16(-x2 * ss))
        o2 = _r16(_r16(x2 * cc) + _r16(x1 * ss))
        out = torch.stack((o1, o2), dim=-1).reshape(xd.shape)
        near = torch.stack((near64, near64), dim=-1).reshape(near64.shape[0], 128)[:, None, :]
    else:
        raise ValueError(pairing)
    return out.to(torch.float16), near


def causal_attention(qkv, cu_seqlens, heads: int, kv_heads: int, *, kv_map: str = "grouped", mask_shift: int = 0,
                     drop_key=None, with_bound: bool = False, budget: int = 1 << 25):
    """ctx [cu[-1], heads 128] float64 on qkv's device (rows of empty windows stay 0), or (ctx, bound) with
    `with_bound`, for fused rows qkv [>= cu[-1], (heads + 2 kv_heads) 128] fp16 whose Q / K heads are already rotated.
    Per window and query head h: ctx = softmax(q k^T / sqrt(128) over the keys j <= i) v with K / V of head
    h // (heads / kv_heads).

    bound[t, c] is the largest |kernel - ctx| of a kernel that scores in fp32 (mma.sync accumulation), runs the softmax in
    fp32 with hardware exp2, rounds the probabilities to fp16 before P.V and its output to fp16; the terms are those of
    `attention` with head_dim 128 and S_vis = i + 1 visible keys:
      (2^-11 + (S_vis + 32) 2^-24) E + S_vis 2^-25 vmax + 2 a (E + |ctx|) + 1/2 ulp_fp16,  E = sum_j p_j |v_j|,
      a = 2^-20 + 2^-22 max|s| + S_vis 2^-24 + 128 2^-23 max_j |q|.|k_j| / sqrt(128).

    Wrong forms for the tests: kv_map="interleaved" (KV head h % kv_heads), mask_shift=+1 / -1 (keys j <= i + 1 /
    j <= i - 1 visible), drop_key=j (key j of every window removed)."""
    D = LLAMA_HEAD_DIM
    dev = qkv.device
    cu = np.asarray(cu_seqlens, dtype=np.int64)
    T = int(cu[-1])
    hid = heads * D
    out = torch.zeros((T, hid), dtype=torch.float64, device=dev)
    bnd = torch.zeros((T, hid), dtype=torch.float64, device=dev) if with_bound else None
    grp = heads // kv_heads
    kvh = torch.arange(heads, device=dev) // grp if kv_map == "grouped" else torch.arange(heads, device=dev) % kv_heads
    if kv_map not in ("grouped", "interleaved"):
        raise ValueError(kv_map)
    scale = 1.0 / D ** 0.5
    lens = np.diff(cu)
    for S in np.unique(lens):
        S = int(S)
        if S == 0:
            continue
        seqs = np.nonzero(lens == S)[0]
        nwin = max(1, budget // (heads * S * max(S, D)))         # windows per step (scores and expanded K / V)
        qc = S if heads * S * S <= budget else max(1, budget // (heads * S))
        for c0 in range(0, len(seqs), nwin):
            sel = seqs[c0:c0 + nwin]
            rows = torch.as_tensor(cu[sel][:, None] + np.arange(S)[None, :], device=dev)       # [n, S]
            x = qkv[rows].to(torch.float64)
            n = len(sel)
            k = x[..., hid:hid + kv_heads * D].reshape(n, S, kv_heads, D).permute(0, 2, 1, 3)[:, kvh]   # [n, h, S, D]
            v = x[..., hid + kv_heads * D:].reshape(n, S, kv_heads, D).permute(0, 2, 1, 3)[:, kvh]
            q_all = x[..., :hid].reshape(n, S, heads, D).permute(0, 2, 1, 3)
            av = v.abs()
            for q0 in range(0, S, qc):
                q1 = min(S, q0 + qc)
                q = q_all[:, :, q0:q1]
                sc = (q @ k.transpose(-1, -2)) * scale                                       # [n, h, qc, S]
                i = torch.arange(q0, q1, device=dev)[:, None]
                j = torch.arange(S, device=dev)[None, :]
                vis = j <= i + mask_shift
                if drop_key is not None:
                    vis = vis & (j != drop_key)
                sc = sc.masked_fill(~vis, -torch.inf)
                m = sc.amax(-1, keepdim=True)
                m = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
                e = torch.exp(sc - m)
                tot = e.sum(-1, keepdim=True)
                p = torch.where(tot > 0, e / tot.clamp_min(1e-300), torch.zeros_like(e))
                o = p @ v
                out[rows[:, q0:q1]] = o.permute(0, 2, 1, 3).reshape(n, q1 - q0, hid)
                if with_bound:
                    E = p @ av
                    svis = vis.sum(-1, keepdim=True).to(torch.float64)                       # [qc, 1]
                    vmax = av.amax(2, keepdim=True)
                    qk = (q.abs() @ k.abs().transpose(-1, -2)).masked_fill(~vis, 0).amax(-1, keepdim=True)
                    smax = sc.abs().masked_fill(~vis, 0).amax(-1, keepdim=True)
                    a = 2.0 ** -20 + 2.0 ** -22 * smax + svis * 2.0 ** -24 + scale * D * 2.0 ** -23 * qk
                    b = (2.0 ** -11 + (svis + 32) * 2.0 ** -24) * E + svis * 2.0 ** -25 * vmax + 2 * a * (E + o.abs())
                    b = b + 0.5 * _ulp16_t(o.abs() + b)
                    bnd[rows[:, q0:q1]] = b.permute(0, 2, 1, 3).reshape(n, q1 - q0, hid)
    return (out, bnd) if with_bound else out
