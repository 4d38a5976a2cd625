"""CPU pins of the fp64 attention reference (oracle/attention_oracle.py) that tests/test_gpu_encoder_kernels.py compares
the attention kernels with, and the refusals of the encoder's diagnostic entry points that come before any device
call.  No GPU needed."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import attention_oracle as AO
from oracle import bert_oracle as BO
from oracle import t5_oracle as T5O
from retrieval_scaling_b200 import _lib

LENS = [1, 2, 15, 17, 32, 33, 64, 97]


def _padded(qkv, cu):
    """Un-padded [T, 2304] -> q, k, v [B, 12, S, 64] float32 (zeros at pad positions) and the key mask [B, S]."""
    lens = np.diff(cu)
    B, S = len(lens), int(lens.max())
    x = np.zeros((B, S, 3 * 768), np.float32)
    for b in range(B):
        x[b, :lens[b]] = qkv[cu[b]:cu[b + 1]].astype(np.float32)
    q, k, v = (torch.from_numpy(x[..., i * 768:(i + 1) * 768]).view(B, S, 12, 64).transpose(1, 2) for i in range(3))
    mask = torch.arange(S)[None, :] < torch.from_numpy(lens)[:, None]
    return q, k, v, mask


def _unpad(ctx, cu):
    """[B, 12, S, 64] -> un-padded [T, 768] float64."""
    B, _, S, _ = ctx.shape
    full = ctx.transpose(1, 2).reshape(B, S, 768).double().numpy()
    return np.concatenate([full[b, :cu[b + 1] - cu[b]] for b in range(B)])


def _cu(lens):
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)


def test_bert_form_matches_bert_oracle_attention_on_a_padded_batch():
    rng = np.random.default_rng(0)
    cu = _cu(LENS)
    qkv = (rng.standard_normal((cu[-1], 2304)) * 1.5).astype(np.float16)
    q, k, v, mask = _padded(qkv, cu)
    add_mask = torch.zeros(len(LENS), 1, 1, q.shape[2]).masked_fill(~mask[:, None, None, :], torch.finfo(torch.float32).min)
    ref = _unpad(BO.attention(q, k, v, add_mask, 64), cu)
    got = AO.attention(qkv, cu, "bert")
    assert np.abs(got - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max())


def test_t5_form_matches_t5_oracle_attention_on_a_padded_batch():
    """Exact-score inputs (Q, K multiples of 1/4 in [-1/2, 1/2], bias multiples of 1/8): both fp16 roundings of the T5
    score are exact, so the fp32 torch oracle and the fp64 reference compute the same scores."""
    rng = np.random.default_rng(1)
    cu = _cu(LENS)
    qkv = (rng.integers(-2, 3, (cu[-1], 2304)) / 4).astype(np.float16)
    qkv[:, 1536:] = rng.standard_normal((cu[-1], 768)).astype(np.float16)
    nb, md = 32, 128
    rel_w = torch.from_numpy(rng.integers(-24, 25, (nb, 12)) / 8).float()
    table = AO.t5_bias_table(rel_w.numpy(), AO.t5_buckets(nb, md))
    q, k, v, mask = _padded(qkv, cu)
    S = q.shape[2]
    pos = torch.arange(S)
    bucket = T5O.relative_position_bucket(pos[None, :] - pos[:, None], nb, md)
    position_bias = rel_w[bucket].permute(2, 0, 1)[None] + (~mask[:, None, None, :]).float() * torch.finfo(torch.float32).min
    ref = _unpad(T5O.attention(q, k, v, position_bias), cu)
    got = AO.attention(qkv, cu, "t5", table)
    assert np.abs(got - ref).max() <= 1e-5 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("nb,md", [(32, 128), (64, 256), (16, 32)])
def test_bias_expansion_matches_relative_position_bucket(nb, md):
    """The bucket table the product uploads, and the per-head table the reference expands from it, against
    t5_oracle.relative_position_bucket over every (query, key) pair of a 512-token sequence."""
    from retrieval_scaling_b200.encoder import t5_bucket_table
    assert np.array_equal(t5_bucket_table(nb, md).numpy(), AO.t5_buckets(nb, md))
    rng = np.random.default_rng(nb)
    w = rng.standard_normal((nb, 12)).astype(np.float16)
    table = AO.t5_bias_table(w, AO.t5_buckets(nb, md))
    pos = torch.arange(512)
    bucket = T5O.relative_position_bucket(pos[None, :] - pos[:, None], nb, md).numpy()
    full = w.astype(np.float64)[bucket]                                    # [query, key, head]
    rel = pos[None, :].numpy() - pos[:, None].numpy()
    assert np.array_equal(table[:, rel + 511].transpose(1, 2, 0), full)
    assert not np.array_equal(table[:, ::-1], table)                        # asymmetric in r: a sign flip is visible


def test_bound_terms_on_exact_scores():
    """On exact scores the bound reduces to the probability rounding, the P.V accumulation and the output rounding: it is
    no looser than 2^-10 E + 1 fp16 ulp."""
    rng = np.random.default_rng(2)
    cu = _cu([5, 40])
    qkv = (rng.integers(-2, 3, (cu[-1], 2304)) / 4).astype(np.float16)
    ctx, bnd = AO.attention(qkv, cu, "bert", with_bound=True)
    x = qkv.astype(np.float64)
    E = np.zeros_like(ctx)
    for b in range(2):
        r = slice(cu[b], cu[b + 1])
        for h in range(12):
            q, k, v = (x[r, i * 768 + h * 64:i * 768 + h * 64 + 64] for i in range(3))
            s = q @ k.T / 8
            p = np.exp(s - s.max(1, keepdims=True))
            p /= p.sum(1, keepdims=True)
            assert np.allclose(p @ v, ctx[r, h * 64:h * 64 + 64], rtol=0, atol=1e-12)
            E[r, h * 64:h * 64 + 64] = p @ np.abs(v)
    assert (bnd <= 2.0 ** -10 * E + AO.ulp16(ctx) + 1e-9).all()
    assert (bnd >= 2.0 ** -11 * E).all()


def test_ulp16_and_round16():
    assert AO.ulp16(1.0) == 2.0 ** -10 and AO.ulp16(1.5) == 2.0 ** -10 and AO.ulp16(2.0) == 2.0 ** -9
    assert AO.ulp16(0.0) == 2.0 ** -24 and AO.ulp16(2.0 ** -20) == 2.0 ** -24
    assert AO.round16(1 + 2.0 ** -11) == 1.0 and AO.round16(1 + 3 * 2.0 ** -11) == 1 + 2.0 ** -9


def test_attention_and_tokens_refusals_before_any_device_call():
    L = _lib.lib()
    p = ctypes.c_void_p(16)              # never dereferenced: the arguments are refused first
    assert L.rsb_bert_attention(None, p, p, 1, 1, 1, p, None) == _lib.RSB_ERR_INVALID
    assert b"null" in L.rsb_bert_last_error()
    assert L.rsb_bert_attention(p, None, p, 1, 1, 1, p, None) == _lib.RSB_ERR_INVALID
    assert L.rsb_bert_attention(p, p, None, 1, 1, 1, p, None) == _lib.RSB_ERR_INVALID
    assert L.rsb_bert_attention(p, p, p, 1, 1, 1, None, None) == _lib.RSB_ERR_INVALID
    for B in (0, -1):
        assert L.rsb_bert_attention(p, p, p, B, 1, 1, p, None) == _lib.RSB_ERR_INVALID
        assert b"empty batch" in L.rsb_bert_last_error()
        assert L.rsb_bert_forward(p, p, None, p, B, 1, 1, _lib.POOL_TOKENS, p, p, 1 << 20, None) == _lib.RSB_ERR_INVALID
    assert L.rsb_bert_forward(None, p, None, p, 1, 1, 1, _lib.POOL_TOKENS, p, p, 1 << 20, None) == _lib.RSB_ERR_INVALID
