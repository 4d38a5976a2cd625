"""CPU/torch ORACLE (test infrastructure, NOT product code) for the sentence-transformers retrievers.

Plain-torch restatement of what the reference executes for `SentenceTransformer(name).half().encode(...)`
(src/search.py:49-61, :244-258; src/embed.py:25-40, :130) when the model is a T5 encoder (GTR-T5) or a BERT-base
model (e5-base), followed by the sentence-transformers head:

  T5 encoder, HF `T5EncoderModel` (transformers/models/t5/modeling_t5.py) as it runs in fp16:
    x = embed_tokens[ids]                                       (not scaled, no position embedding)
    per block:  x += o(attn(rms(x))), fp16 clamp;  x += wo(relu(wi(rms(x)))), fp16 clamp
    x = final_layer_norm(x)
    rms(x) = w * half(x * rsqrt(mean(x^2) + eps))               (T5LayerNorm, fp32 statistics)
    attn: scores = q k^T (no 1/sqrt(d)) + bias[h][bucket(j - i)] + key mask; softmax in fp32, cast back; P V
    clamp: if any element of the (padded) hidden states is +-inf, clamp all to +-(65504 - 1000), else to +-65504
  head (sentence_transformers.models): Pooling (mean over the attention mask, or the first token) -> Dense (Linear,
  Identity activation) -> Normalize (torch.nn.functional.normalize, p=2, dim=1).

sentence_transformers is not a dependency: its modules are restated from their published behaviour.  The T5 forward is
pinned against `transformers.T5EncoderModel` by the goldens of tests/golden/make_t5_golden.py
(tests/golden/encoder_t5_*.npz), replayed by tests/test_st_encoder_cpu.py.
"""
from __future__ import annotations

import math
from typing import Dict

import torch
import torch.nn.functional as F

T5_CONFIG = dict(d_model=768, num_heads=12, d_kv=64, d_ff=3072, num_layers=12, vocab_size=32128,
                 relative_attention_num_buckets=32, relative_attention_max_distance=128, layer_norm_epsilon=1e-6,
                 feed_forward_proj="relu")


def seeded_state_dict(config: dict, seed: int, head: bool = True) -> Dict[str, torch.Tensor]:
    """Deterministic (CPU generator) fp32 weights with HF T5EncoderModel key names (embedding under both tied names),
    plus `dense.weight` / `dense.bias` of the sentence-transformers Dense head when `head`.  Same recipe as
    retrieval_scaling_b200.encoder.random_t5_state_dict (duplicated so that the oracle does not import the product)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    H, Fd = config["d_model"], config["d_ff"]

    def n(*shape, std):
        return torch.randn(*shape, generator=g) * std

    sd = {"shared.weight": n(config["vocab_size"], H, std=0.5),
          "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight":
              n(config["relative_attention_num_buckets"], config["num_heads"], std=0.5)}
    for i in range(config["num_layers"]):
        p = f"encoder.block.{i}.layer."
        sd[p + "0.SelfAttention.q.weight"] = n(H, H, std=0.02)
        for m in "kvo":
            sd[p + f"0.SelfAttention.{m}.weight"] = n(H, H, std=0.04)
        sd[p + "0.layer_norm.weight"] = 1.0 + n(H, std=0.1)
        sd[p + "1.DenseReluDense.wi.weight"] = n(Fd, H, std=0.04)
        sd[p + "1.DenseReluDense.wo.weight"] = n(H, Fd, std=0.02)
        sd[p + "1.layer_norm.weight"] = 1.0 + n(H, std=0.1)
    sd["encoder.final_layer_norm.weight"] = 1.0 + n(H, std=0.1)
    if head:
        sd["dense.weight"] = n(H, H, std=0.04)
        sd["dense.bias"] = n(H, std=0.02)
    sd["encoder.embed_tokens.weight"] = sd["shared.weight"]
    return sd


def relative_position_bucket(relative_position: torch.Tensor, num_buckets: int, max_distance: int) -> torch.Tensor:
    """T5Attention._relative_position_bucket, bidirectional (the encoder), with its fp32 log expression."""
    nb = num_buckets // 2
    ret = (relative_position > 0).to(torch.long) * nb
    n = torch.abs(relative_position)
    max_exact = nb // 2
    large = max_exact + (torch.log(n.float() / max_exact) / math.log(max_distance / max_exact)
                         * (nb - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, nb - 1))
    return ret + torch.where(n < max_exact, n, large)


def _rms(x, w, eps):
    var = x.to(torch.float32).pow(2).mean(-1, keepdim=True)
    y = x * torch.rsqrt(var + eps)
    if w.dtype in (torch.float16, torch.bfloat16):
        y = y.to(w.dtype)
    return w * y


def _clamp(x):
    if x.dtype != torch.float16:
        return x
    c = torch.where(torch.isinf(x).any(), torch.finfo(x.dtype).max - 1000, torch.finfo(x.dtype).max)
    return torch.clamp(x, min=-c, max=c)


def attention(q, k, v, position_bias):
    """HF T5Attention core on [B, heads, S, d_kv] tensors: scores = q k^T (no scaling) + position_bias (the relative
    bias plus the key mask), softmax in fp32 and cast back, times v."""
    scores = torch.matmul(q, k.transpose(3, 2))
    scores += position_bias
    att = torch.softmax(scores.float(), dim=-1).type_as(scores)
    return torch.matmul(att, v)


def t5_hidden(sd: Dict[str, torch.Tensor], config: dict, input_ids, attention_mask, dtype=torch.float32):
    """last_hidden_state [B, S, 768] of T5EncoderModel in `dtype` (float32 = exact restatement; float16 on CUDA
    mirrors `.half()`)."""
    dev = input_ids.device
    w = {k: v.to(device=dev, dtype=dtype) for k, v in sd.items()}
    B, S = input_ids.shape
    nh, hd, eps = config["num_heads"], config["d_kv"], config["layer_norm_epsilon"]
    x = w["shared.weight"][input_ids]
    pos = torch.arange(S, device=dev)
    bucket = relative_position_bucket(pos[None, :] - pos[:, None], config["relative_attention_num_buckets"],
                                      config["relative_attention_max_distance"])
    bias = w["encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"][bucket].permute(2, 0, 1)[None]
    mask = (1.0 - attention_mask[:, None, None, :].to(dtype)) * torch.finfo(dtype).min
    position_bias = bias + mask
    for i in range(config["num_layers"]):
        p = f"encoder.block.{i}.layer."
        h = _rms(x, w[p + "0.layer_norm.weight"], eps)
        q, k, v = (F.linear(h, w[p + f"0.SelfAttention.{m}.weight"]).view(B, S, nh, hd).transpose(1, 2) for m in "qkv")
        ctx = attention(q, k, v, position_bias).transpose(1, 2).reshape(B, S, nh * hd)
        x = _clamp(x + F.linear(ctx, w[p + "0.SelfAttention.o.weight"]))
        h = _rms(x, w[p + "1.layer_norm.weight"], eps)
        x = _clamp(x + F.linear(F.relu(F.linear(h, w[p + "1.DenseReluDense.wi.weight"])),
                                w[p + "1.DenseReluDense.wo.weight"]))
    return _rms(x, w["encoder.final_layer_norm.weight"], eps)


def st_head(tokens, attention_mask, pooling: str = "average", dense_w=None, dense_b=None, normalize: bool = False):
    """sentence_transformers Pooling (mean / cls) -> Dense (Identity) -> Normalize, in the dtype of `tokens`."""
    if pooling == "average":
        m = attention_mask.unsqueeze(-1).expand(tokens.size()).to(tokens.dtype)
        out = torch.sum(tokens * m, 1) / torch.clamp(m.sum(1), min=1e-9)
    else:
        out = tokens[:, 0]
    if dense_w is not None:
        out = F.linear(out, dense_w.to(out), None if dense_b is None else dense_b.to(out))
    if normalize:
        out = F.normalize(out, p=2, dim=1)
    return out


def t5_st_forward(sd, config, input_ids, attention_mask, pooling="average", dense=True, normalize=True,
                  dtype=torch.float32):
    """T5 encoder + sentence-transformers head: [B, 768] in `dtype`."""
    tok = t5_hidden(sd, config, input_ids, attention_mask, dtype)
    dev = input_ids.device
    dw = sd["dense.weight"].to(dev) if dense else None
    db = sd.get("dense.bias").to(dev) if dense and "dense.bias" in sd else None
    return st_head(tok, attention_mask.to(dev), pooling, dw, db, normalize)
