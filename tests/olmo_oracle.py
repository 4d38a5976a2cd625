"""fp64 restatement of HF OlmoForCausalLM's and Olmo2ForCausalLM's forwards and shifted causal-LM loss, written from
the published model definitions:

    OLMo    embed -> [x += attn(LN(x)); x += mlp(LN(x))] x L -> LN -> lm_head, LN without weight or bias (eps 1e-5),
            q, k and v clamped to +-clip_qkv when it is set
    OLMo-2  embed -> [x += RMS(attn(x)); x += RMS(mlp(x))] x L -> RMS -> lm_head, with q_norm / k_norm an RMSNorm over
            the whole q / k projection before RoPE

with SwiGLU MLPs, default RoPE (rotate_half, positions from 0) and causal GQA attention.  RoPE's inv_freq and angles
are computed in fp32 as HF computes them.  `prologue` restates the attention prologue alone, optionally with the fp16
roundings of a kernel's order.  Test infrastructure, independent of transformers and of the product code."""
from __future__ import annotations

import numpy as np
import torch

HD = 128


def version(cfg) -> int:
    return 2 if cfg["model_type"] == "olmo2" else 1


def rope_theta(cfg) -> float:
    rp = cfg.get("rope_parameters") or {}
    return float(rp.get("rope_theta", cfg.get("rope_theta", 10000.0)))


def eps(cfg) -> float:
    return 1e-5 if version(cfg) == 1 else float(cfg.get("rms_norm_eps", 1e-5))


def rope_angles(pos, theta: float):
    """fp32 angles [n, 64] at integer positions pos, as OlmoRotaryEmbedding computes them."""
    inv = 1.0 / (theta ** (torch.arange(0, HD, 2, dtype=torch.int64).float() / HD))
    p = torch.as_tensor(np.asarray(pos), dtype=torch.float32)
    return p[:, None] * inv[None, :]


def rotate(x, cos, sin):
    """x * cos + rotate_half(x) * sin on the last dim (128) of x, cos / sin [.., 64]."""
    h = HD // 2
    x1, x2 = x[..., :h], x[..., h:]
    return torch.cat((x1 * cos - x2 * sin, x2 * cos + x1 * sin), dim=-1)


def layer_norm(x, e=1e-5):
    mean = x.mean(-1, keepdim=True)
    return (x - mean) / torch.sqrt((x - mean).pow(2).mean(-1, keepdim=True) + e)


def rms_norm(x, w, e):
    return x / torch.sqrt(x.pow(2).mean(-1, keepdim=True) + e) * w


def prologue(q, k, v, pos, theta, clip=None, qn=None, kn=None, e=1e-5, r16=None):
    """The attention prologue on q [n, heads 128], k / v [n, kv 128] float64: clamp (clip), whole-projection RMSNorm
    (qn / kn), then RoPE at positions pos.  r16 (a rounding function) rounds where the kernel rounds to fp16: after the
    clamp and after each norm.  Returns (q, k, v) float64."""
    if clip is not None:
        q, k, v = (t.clamp(-clip, clip) for t in (q, k, v))
    if qn is not None:
        q, k = rms_norm(q, qn, e), rms_norm(k, kn, e)
    if r16 is not None:
        q, k, v = r16(q), r16(k), r16(v)
    f = rope_angles(pos, theta).to(device=q.device, dtype=torch.float64)
    c, s = f.cos()[:, None], f.sin()[:, None]
    n = q.shape[0]
    q = rotate(q.view(n, -1, HD), c, s).reshape(n, -1)
    k = rotate(k.view(n, -1, HD), c, s).reshape(n, -1)
    return q, k, v


def hidden_rows(sd, cfg, ids, device="cpu", stats=None):
    """[x_0, x_1, ..., x_L] float64 [S, hidden] on `device` for one window: the embedding rows and the residual stream
    after each layer (x_L is the input of the final norm).  stats (a dict), when given, receives the counts of q / k / v
    elements the clamp changed ('clipped') out of 'qkv'."""
    W = {k: v.to(device=device, dtype=torch.float64) for k, v in sd.items() if v.is_floating_point()}
    v2 = version(cfg) == 2
    H, nh = cfg["hidden_size"], cfg["num_attention_heads"]
    kv = cfg.get("num_key_value_heads") or nh
    e, theta = eps(cfg), rope_theta(cfg)
    clip = None if v2 else cfg.get("clip_qkv")
    ids = torch.as_tensor(np.asarray(ids), dtype=torch.long, device=device)
    S = len(ids)
    x = W["model.embed_tokens.weight"][ids]
    mask = torch.full((S, S), -torch.inf, dtype=torch.float64, device=device).triu(1)
    out = [x]
    for i in range(cfg["num_hidden_layers"]):
        p = f"model.layers.{i}."
        h = x if v2 else layer_norm(x)
        q, k, v = (h @ W[p + f"self_attn.{n}_proj.weight"].T for n in "qkv")
        if stats is not None and clip is not None:
            stats["clipped"] = stats.get("clipped", 0) + sum(int((t.abs() > clip).sum()) for t in (q, k, v))
            stats["qkv"] = stats.get("qkv", 0) + q.numel() + k.numel() + v.numel()
        q, k, v = prologue(q, k, v, np.arange(S), theta, clip,
                           W.get(p + "self_attn.q_norm.weight"), W.get(p + "self_attn.k_norm.weight"), e)
        q = q.view(S, nh, HD).transpose(0, 1)
        k = k.view(S, kv, HD).transpose(0, 1).repeat_interleave(nh // kv, dim=0)
        v = v.view(S, kv, HD).transpose(0, 1).repeat_interleave(nh // kv, dim=0)
        a = torch.softmax(q @ k.transpose(1, 2) / HD ** 0.5 + mask, dim=-1) @ v
        a = a.transpose(0, 1).reshape(S, H) @ W[p + "self_attn.o_proj.weight"].T
        x = x + (rms_norm(a, W[p + "post_attention_layernorm.weight"], e) if v2 else a)
        h = x if v2 else layer_norm(x)
        m = torch.nn.functional.silu(h @ W[p + "mlp.gate_proj.weight"].T) * (h @ W[p + "mlp.up_proj.weight"].T)
        m = m @ W[p + "mlp.down_proj.weight"].T
        x = x + (rms_norm(m, W[p + "post_feedforward_layernorm.weight"], e) if v2 else m)
        out.append(x)
    return out


def token_nll(sd, cfg, ids, device="cpu", stats=None) -> np.ndarray:
    """nll[t] = -log p(ids[t] | ids[:t]) in fp64 for one window, 0 at t = 0; the forward runs on `device`."""
    x = hidden_rows(sd, cfg, ids, device, stats)[-1]
    f = lambda k: sd[k].to(device=device, dtype=torch.float64)   # noqa: E731
    x = rms_norm(x, f("model.norm.weight"), eps(cfg)) if version(cfg) == 2 else layer_norm(x)
    head = f("model.embed_tokens.weight") if cfg.get("tie_word_embeddings") else f("lm_head.weight")
    lp = torch.log_softmax(x @ head.T, dim=-1)
    ids = torch.as_tensor(np.asarray(ids), dtype=torch.long, device=device)
    S = len(ids)
    out = np.zeros(S, np.float64)
    if S > 1:
        out[1:] = (-lp[:-1].gather(1, ids[1:, None]).squeeze(1)).cpu().numpy()
    return out
