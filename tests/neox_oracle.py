"""fp64 restatement of HF GPTNeoXForCausalLM's forward and shifted causal-LM loss, written from the published model
definition (embed_in -> [x + attn(LN1(x)) + mlp(LN2(x))] x L -> final LayerNorm -> embed_out), with the attention's
per-head interleaved query_key_value, partial rotary on the first rotary_ndims of every Q / K head, and the exact-erf
GELU MLP.  RoPE's inv_freq and angles are computed in fp32 as HF computes them in every dtype.  Test infrastructure,
independent of transformers and of the product code."""
from __future__ import annotations

import numpy as np
import torch


def rotary(cfg):
    """(rotary_ndims, base) from the Hub's fields (rotary_pct, rotary_emb_base) or transformers 5's rope_parameters."""
    d = cfg["hidden_size"] // cfg["num_attention_heads"]
    rp = cfg.get("rope_parameters") or {}
    pct = rp.get("partial_rotary_factor", cfg.get("rotary_pct", 0.25))
    base = rp.get("rope_theta", cfg.get("rotary_emb_base", 10000.0))
    return int(d * pct), float(base)


def rope_tables(S: int, base: float, rot: int):
    inv = 1.0 / (base ** (torch.arange(0, rot, 2, dtype=torch.int64).float() / rot))        # fp32, as HF
    f = inv[:, None] @ torch.arange(S, dtype=torch.float32)[None, :]                         # fp32 angles
    emb = torch.cat((f.T, f.T), dim=-1)
    return emb.cos().double(), emb.sin().double()


def _rotate_half(x):
    h = x.shape[-1] // 2
    return torch.cat((-x[..., h:], x[..., :h]), dim=-1)


def _ln(x, w, b, eps):
    mean = x.mean(-1, keepdim=True)
    var = (x - mean).pow(2).mean(-1, keepdim=True)
    return (x - mean) / torch.sqrt(var + eps) * w + b


def hidden_rows(sd, cfg, ids, device="cpu"):
    """[x_0, x_1, ..., x_L] float64 [S, hidden] on `device` for one window: the embedding rows and the residual stream
    after each layer (x_L is the input of final_layer_norm)."""
    W = {k: v.to(device=device, dtype=torch.float64) for k, v in sd.items() if v.is_floating_point()}
    H, nh = cfg["hidden_size"], cfg["num_attention_heads"]
    d, eps = H // nh, cfg["layer_norm_eps"]
    rot, base = rotary(cfg)
    ids = torch.as_tensor(np.asarray(ids), dtype=torch.long, device=device)
    S = len(ids)
    x = W["gpt_neox.embed_in.weight"][ids]
    cos, sin = (t.to(device) for t in rope_tables(S, base, rot))
    mask = torch.full((S, S), -torch.inf, dtype=torch.float64, device=device).triu(1)
    out = [x]
    for i in range(cfg["num_hidden_layers"]):
        p = f"gpt_neox.layers.{i}."
        h = _ln(x, W[p + "input_layernorm.weight"], W[p + "input_layernorm.bias"], eps)
        qkv = (h @ W[p + "attention.query_key_value.weight"].T + W[p + "attention.query_key_value.bias"])
        qkv = qkv.view(S, nh, 3 * d).transpose(0, 1)                       # per head: q_h | k_h | v_h
        q, k, v = qkv[..., :d], qkv[..., d:2 * d], qkv[..., 2 * d:]
        q = torch.cat((q[..., :rot] * cos + _rotate_half(q[..., :rot]) * sin, q[..., rot:]), dim=-1)
        k = torch.cat((k[..., :rot] * cos + _rotate_half(k[..., :rot]) * sin, k[..., rot:]), dim=-1)
        a = torch.softmax(q @ k.transpose(1, 2) / d ** 0.5 + mask, dim=-1) @ v
        a = a.transpose(0, 1).reshape(S, H) @ W[p + "attention.dense.weight"].T + W[p + "attention.dense.bias"]
        h2 = _ln(x, W[p + "post_attention_layernorm.weight"], W[p + "post_attention_layernorm.bias"], eps)
        m = torch.nn.functional.gelu(h2 @ W[p + "mlp.dense_h_to_4h.weight"].T + W[p + "mlp.dense_h_to_4h.bias"])
        m = m @ W[p + "mlp.dense_4h_to_h.weight"].T + W[p + "mlp.dense_4h_to_h.bias"]
        x = m + a + x
        out.append(x)
    return out


def token_nll(sd, cfg, ids, device="cpu") -> np.ndarray:
    """nll[t] = -log p(ids[t] | ids[:t]) in fp64 for one window, 0 at t = 0; the forward runs on `device`."""
    x = hidden_rows(sd, cfg, ids, device)[-1]
    f = lambda k: sd[k].to(device=device, dtype=torch.float64)   # noqa: E731
    x = _ln(x, f("gpt_neox.final_layer_norm.weight"), f("gpt_neox.final_layer_norm.bias"), cfg["layer_norm_eps"])
    lp = torch.log_softmax(x @ f("embed_out.weight").T, dim=-1)
    ids = torch.as_tensor(np.asarray(ids), dtype=torch.long, device=device)
    S = len(ids)
    out = np.zeros(S, np.float64)
    if S > 1:
        out[1:] = (-lp[:-1].gather(1, ids[1:, None]).squeeze(1)).cpu().numpy()
    return out


def qkv_permutation(heads: int, head_dim: int) -> np.ndarray:
    """Row order that takes query_key_value's per-head interleaved rows [heads, 3, head_dim] to [3, heads, head_dim]
    ([Q heads | K heads | V heads]): permuted[r] = original[perm[r]]."""
    return np.arange(3 * heads * head_dim).reshape(heads, 3, head_dim).transpose(1, 0, 2).reshape(-1)
