"""fp64 restatement of HF LlamaForCausalLM's forward and shifted causal-LM loss, written from the published model
definition (embedding -> [RMSNorm -> q/k/v -> RoPE (rotate_half) -> causal softmax(q k^T / sqrt(d)) v -> o -> residual ->
RMSNorm -> down(silu(gate) * up) -> residual] x L -> RMSNorm -> LM head).  RoPE's inv_freq and angles are computed in
fp32 as HF computes them in every dtype.  Test infrastructure, independent of transformers."""
from __future__ import annotations

import numpy as np
import torch


def _rms(x, w, eps):
    return w * (x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps))


def rope_tables(S: int, theta: float, dim: int = 128):
    inv = 1.0 / (theta ** (torch.arange(0, dim, 2, dtype=torch.int64).float() / dim))      # fp32, as HF
    f = inv[:, None] @ torch.arange(S, dtype=torch.float32)[None, :]                         # fp32 angles
    emb = torch.cat((f.T, f.T), dim=-1)
    return emb.cos().double(), emb.sin().double()


def _rotate_half(x):
    h = x.shape[-1] // 2
    return torch.cat((-x[..., h:], x[..., :h]), dim=-1)


def hidden_rows(sd, cfg, ids, device="cpu"):
    """[x_0, x_1, ..., x_L] float64 [S, hidden] on `device` for one window: the embedding rows and the residual stream
    after each decoder layer (x_L is the input of the final norm)."""
    W = {k: v.to(device=device, dtype=torch.float64) for k, v in sd.items()}
    H, nh, nkv = cfg["hidden_size"], cfg["num_attention_heads"], cfg["num_key_value_heads"]
    eps, d = cfg["rms_norm_eps"], 128
    ids = torch.as_tensor(np.asarray(ids), dtype=torch.long, device=device)
    S = len(ids)
    x = W["model.embed_tokens.weight"][ids]
    cos, sin = (t.to(device) for t in rope_tables(S, cfg["rope_theta"]))
    mask = torch.full((S, S), -torch.inf, dtype=torch.float64, device=device).triu(1)
    out = [x]
    for i in range(cfg["num_hidden_layers"]):
        p = f"model.layers.{i}."
        h = _rms(x, W[p + "input_layernorm.weight"], eps)
        q = (h @ W[p + "self_attn.q_proj.weight"].T).view(S, nh, d).transpose(0, 1)
        k = (h @ W[p + "self_attn.k_proj.weight"].T).view(S, nkv, d).transpose(0, 1)
        v = (h @ W[p + "self_attn.v_proj.weight"].T).view(S, nkv, d).transpose(0, 1)
        q = q * cos + _rotate_half(q) * sin
        k = k * cos + _rotate_half(k) * sin
        k = k.repeat_interleave(nh // nkv, dim=0)
        v = v.repeat_interleave(nh // nkv, dim=0)
        a = torch.softmax(q @ k.transpose(1, 2) / d ** 0.5 + mask, dim=-1) @ v
        x = x + a.transpose(0, 1).reshape(S, H) @ W[p + "self_attn.o_proj.weight"].T
        h = _rms(x, W[p + "post_attention_layernorm.weight"], eps)
        g = h @ W[p + "mlp.gate_proj.weight"].T
        x = x + (torch.nn.functional.silu(g) * (h @ W[p + "mlp.up_proj.weight"].T)) @ W[p + "mlp.down_proj.weight"].T
        out.append(x)
    return out


def token_nll(sd, cfg, ids, device="cpu") -> np.ndarray:
    """nll[t] = -log p(ids[t] | ids[:t]) in fp64 for one window, 0 at t = 0; the forward runs on `device`."""
    x = hidden_rows(sd, cfg, ids, device)[-1]
    eps = cfg["rms_norm_eps"]
    x = _rms(x, sd["model.norm.weight"].to(device=device, dtype=torch.float64), eps)
    head = sd["model.embed_tokens.weight"] if cfg.get("tie_word_embeddings") else sd["lm_head.weight"]
    lp = torch.log_softmax(x @ head.to(device=device, dtype=torch.float64).T, dim=-1)
    ids = torch.as_tensor(np.asarray(ids), dtype=torch.long, device=device)
    S = len(ids)
    out = np.zeros(S, np.float64)
    if S > 1:
        out[1:] = (-lp[:-1].gather(1, ids[1:, None]).squeeze(1)).cpu().numpy()
    return out


def mean_loss(nll: np.ndarray, labels) -> float:
    """HF's `loss` for one window: mean over positions t > 0 with labels[t] != -100, NaN without any."""
    labels = np.asarray(labels)
    pos = [t for t in range(1, len(labels)) if labels[t] != -100]
    return float(np.sum(nll[pos]) / len(pos)) if pos else float("nan")
