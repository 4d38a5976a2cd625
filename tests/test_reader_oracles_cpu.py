"""CPU pinning of the reader's kernel-level references against transformers' own Llama code, so that the GPU tests of
tests/test_gpu_reader_kernels.py compare the kernels with HF and not with a restatement of the kernels:

  oracle/attention_oracle.rope_f16          HF LlamaRotaryEmbedding + apply_rotary_pos_emb in fp16
  oracle/attention_oracle.causal_attention  HF repeat_kv + eager_attention_forward in fp64, and tests/llama_oracle.py
  tests/llama_oracle.py                     per-layer hidden rows against transformers fp32, on an explicit device"""
import os
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import llama_fixture as F  # noqa: E402
import llama_oracle as O  # noqa: E402

from oracle import attention_oracle as AO  # noqa: E402

M = pytest.importorskip("transformers.models.llama.modeling_llama")


def _hf_rope(x, pos, theta):
    """x [n, nh, 128] fp16 at positions pos [n] through transformers' LlamaRotaryEmbedding and apply_rotary_pos_emb."""
    import transformers
    cfg = transformers.LlamaConfig(hidden_size=128, num_attention_heads=1, rope_theta=theta,
                                   max_position_embeddings=int(max(pos)) + 1, head_dim=128)
    rot = M.LlamaRotaryEmbedding(cfg)
    xt = x.permute(1, 0, 2)[None]                                       # [1, nh, n, 128]
    cos, sin = rot(xt, torch.as_tensor(pos, dtype=torch.long)[None])
    q, _ = M.apply_rotary_pos_emb(xt, xt, cos, sin)
    return q[0].permute(1, 0, 2)


@pytest.mark.parametrize("theta", [10000.0, 500000.0])
def test_rope_restatement_is_hf_apply_rotary_pos_emb_in_fp16(theta):
    """Bit-equal to HF in fp16 at positions up to 8191; where the fp32 cos / sin lie within 2 fp32 ulp of an fp16
    rounding boundary (flagged), bit-equal to the restatement with one of the two fp16 neighbours.  The wrong forms
    (rotate adjacent pairs, fp64 angles) are not: fp64 angles differ from HF's fp32 angles at positions >= 4096."""
    rng = np.random.default_rng(int(theta))
    pos = np.concatenate([np.arange(0, 70), rng.integers(70, 4096, 150), np.arange(4090, 4100), rng.integers(4096, 8192, 150),
                          np.arange(8180, 8192)])
    x = torch.from_numpy(rng.standard_normal((len(pos), 3, 128)) * 2).half()
    ours, near = AO.rope_f16(x, pos, theta)
    hf = _hf_rope(x, pos, theta)
    same = ours.view(torch.int16) == hf.view(torch.int16)
    assert same[~near.expand_as(same)].all()
    for i in (-1, 0, 1):                      # flagged elements: the result of either fp16 neighbour of cos / sin
        for j in (-1, 0, 1):
            same |= AO.rope_f16(x, pos, theta, cs_shift=(i, j))[0].view(torch.int16) == hf.view(torch.int16)
    assert same.all()
    assert near.float().mean() < 0.01
    assert not torch.equal(AO.rope_f16(x, pos, theta, pairing="adjacent")[0], hf)
    far = torch.from_numpy(pos >= 4096)
    f64 = AO.rope_f16(x, pos, theta, angles="fp64")[0]
    assert not torch.equal(f64[far], hf[far])


def _hf_attention(qkv, S, heads, kv_heads):
    """transformers' eager_attention_forward (repeat_kv inside) on one window, fp64, causal mask."""
    D = 128
    x = qkv.double()
    q = x[:, :heads * D].reshape(S, heads, D).transpose(0, 1)[None]
    k = x[:, heads * D:(heads + kv_heads) * D].reshape(S, kv_heads, D).transpose(0, 1)[None]
    v = x[:, (heads + kv_heads) * D:].reshape(S, kv_heads, D).transpose(0, 1)[None]
    mask = torch.full((S, S), -torch.inf, dtype=torch.float64).triu(1)[None, None]
    mod = types.SimpleNamespace(num_key_value_groups=heads // kv_heads, training=False)
    o, _ = M.eager_attention_forward(mod, q, k, v, mask, scaling=D ** -0.5)
    return o[0].reshape(S, heads * D)


@pytest.mark.parametrize("heads,kv_heads", [(4, 1), (4, 4), (8, 2), (6, 3)])
def test_causal_attention_matches_hf_repeat_kv_and_eager_attention(heads, kv_heads):
    """Per window, the fp64 oracle equals HF's eager attention (whose softmax runs in fp32) to 1e-6; the GQA map, the
    causal mask and the per-window restart come from HF.  The wrong references differ from HF."""
    rng = np.random.default_rng(heads * 10 + kv_heads)
    lens = [1, 5, 0, 70, 3]
    cu = np.concatenate([[0], np.cumsum(lens)])
    qkv = torch.from_numpy(rng.standard_normal((int(cu[-1]), (heads + 2 * kv_heads) * 128)) * 1.5).half()
    ref, bnd = AO.causal_attention(qkv, cu, heads, kv_heads, with_bound=True)
    assert (bnd > 0).all() and (bnd < 0.05).all()
    wrong = {"mask +1": AO.causal_attention(qkv, cu, heads, kv_heads, mask_shift=1),
             "mask -1": AO.causal_attention(qkv, cu, heads, kv_heads, mask_shift=-1),
             "key 63 dropped": AO.causal_attention(qkv, cu, heads, kv_heads, drop_key=63)}
    if 1 < kv_heads < heads:
        wrong["interleaved"] = AO.causal_attention(qkv, cu, heads, kv_heads, kv_map="interleaved")
    for b, S in enumerate(lens):
        if S == 0:
            continue
        hf = _hf_attention(qkv[cu[b]:cu[b + 1]], S, heads, kv_heads)
        np.testing.assert_allclose(ref[cu[b]:cu[b + 1]].numpy(), hf.numpy(), atol=1e-6, rtol=0)
    for name, w in wrong.items():
        assert (w - ref).abs().max() > 1e-3, name


def test_causal_attention_matches_the_llama_oracle_layer():
    """One layer of tests/llama_oracle.py with o_proj = I and down_proj = 0 adds exactly its attention output to the
    residual stream; fed the same rotated fp64 Q / K / V, causal_attention reproduces it (GQA 8 : 2)."""
    cfg = dict(F.CONFIG, num_hidden_layers=1, hidden_size=1024, num_attention_heads=8, num_key_value_heads=2,
               intermediate_size=256, vocab_size=300, max_position_embeddings=128)
    sd = F.seeded_state_dict(cfg, seed=4)
    H = cfg["hidden_size"]
    sd["model.layers.0.self_attn.o_proj.weight"] = torch.eye(H)
    sd["model.layers.0.mlp.down_proj.weight"].zero_()
    ids = np.random.default_rng(3).integers(0, cfg["vocab_size"], 90)
    x0, x1 = O.hidden_rows(sd, cfg, ids, device="cpu")
    W = {k: v.double() for k, v in sd.items()}
    h = O._rms(x0, W["model.layers.0.input_layernorm.weight"], cfg["rms_norm_eps"])
    S, D, kv = len(ids), 128, cfg["num_key_value_heads"]
    cos, sin = O.rope_tables(S, cfg["rope_theta"])
    q = (h @ W["model.layers.0.self_attn.q_proj.weight"].T).view(S, 8, D)
    k = (h @ W["model.layers.0.self_attn.k_proj.weight"].T).view(S, kv, D)
    v = h @ W["model.layers.0.self_attn.v_proj.weight"].T
    q = q * cos[:, None] + O._rotate_half(q) * sin[:, None]
    k = k * cos[:, None] + O._rotate_half(k) * sin[:, None]
    qkv = torch.cat([q.reshape(S, -1), k.reshape(S, -1), v], 1)
    np.testing.assert_allclose(AO.causal_attention(qkv, [0, S], 8, kv).numpy(), (x1 - x0).numpy(), atol=1e-10, rtol=0)
    assert (AO.causal_attention(qkv, [0, S], 8, kv, kv_map="interleaved") - (x1 - x0)).abs().max() > 1e-3


@pytest.mark.parametrize("kv_heads", [4, 1])
def test_oracle_hidden_rows_match_transformers_fp32(kv_heads):
    """Every layer's residual rows of llama_oracle.hidden_rows (on an explicit device) against transformers fp32: the
    decoder-layer outputs and the input of the final norm, to 1e-4."""
    cfg = dict(F.CONFIG, num_key_value_heads=kv_heads, max_position_embeddings=256)
    model = F.hf_model(cfg, dtype=torch.float32, seed=7)
    sd = F.seeded_state_dict(cfg, seed=7)
    ids = np.random.default_rng(1).integers(0, cfg["vocab_size"], 150)
    rows = O.hidden_rows(sd, cfg, ids, device=torch.device("cpu"))
    assert len(rows) == cfg["num_hidden_layers"] + 1
    got = []
    hooks = [layer.register_forward_hook(lambda m, a, o: got.append((o[0] if isinstance(o, tuple) else o)[0].double()))
             for layer in model.model.layers]
    with torch.no_grad():
        model(torch.as_tensor(ids)[None])
    for hk in hooks:
        hk.remove()
    np.testing.assert_allclose(rows[0].numpy(), sd["model.embed_tokens.weight"][ids].double().numpy(), rtol=0, atol=0)
    for i, g in enumerate(got):
        np.testing.assert_allclose(rows[i + 1].numpy(), g.numpy(), atol=1e-4, rtol=0)
    np.testing.assert_allclose(O.token_nll(sd, cfg, ids, device="cpu"), F.hf_token_nll(model, ids), atol=1e-4, rtol=0)
