"""CPU/torch ORACLE (test infrastructure, NOT product code) for the encoder half of the hot path.

Plain-torch restatement of what the reference executes for a query batch:
  `Contriever.forward` (contriever/src/contriever.py:17-55) = HF `BertModel` (post-LN BERT, add_pooling_layer=False,
  contriever.py:13) -> zero padded positions (:46) -> sum / count mean pooling (:49) or CLS (:51); no L2-normalise
  on the hot path (:29,53).  HF BertModel math as of transformers 5.5.0 (SURVEY.md App. C): embeddings
  word+type+position -> LayerNorm(eps) ; per layer Q,K,V Linear -> softmax(QK^T/sqrt(64) + key mask) V -> Linear +
  residual -> LayerNorm -> Linear -> exact-erf GELU -> Linear + residual -> LayerNorm.

PINNED: unlike the ANN half, the reference's own class imports in the build container, so this restatement is
checked against `contriever.src.contriever.Contriever` itself: `tests/golden/make_encoder_golden.py` runs the
reference class on seeded weights / token batches and commits its outputs (`tests/golden/encoder_*.npz`);
`tests/test_encoder_oracle.py` replays them through this file on CPU.
"""
from __future__ import annotations

import math
from typing import Dict

import torch
import torch.nn.functional as F


def seeded_state_dict(config: dict, seed: int) -> Dict[str, torch.Tensor]:
    """Deterministic (CPU generator) fp32 weights with HF BertModel key names; same recipe as
    retrieval_scaling_b200.encoder.random_state_dict (duplicated here so the oracle does not import the product)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    H, I = config["hidden_size"], config["intermediate_size"]

    def n(*shape, std):
        return torch.randn(*shape, generator=g) * std

    sd = {
        "embeddings.word_embeddings.weight": n(config["vocab_size"], H, std=0.5),
        "embeddings.position_embeddings.weight": n(config["max_position_embeddings"], H, std=0.3),
        "embeddings.token_type_embeddings.weight": n(config["type_vocab_size"], H, std=0.3),
        "embeddings.LayerNorm.weight": 1.0 + n(H, std=0.1),
        "embeddings.LayerNorm.bias": n(H, std=0.1),
    }
    for i in range(config["num_hidden_layers"]):
        p = f"encoder.layer.{i}."
        for nm, (o, k_) in {"attention.self.query": (H, H), "attention.self.key": (H, H), "attention.self.value": (H, H),
                            "attention.output.dense": (H, H), "intermediate.dense": (I, H), "output.dense": (H, I)}.items():
            sd[p + nm + ".weight"] = n(o, k_, std=0.04)
            sd[p + nm + ".bias"] = n(o, std=0.02)
        for nm in ("attention.output.LayerNorm", "output.LayerNorm"):
            sd[p + nm + ".weight"] = 1.0 + n(H, std=0.1)
            sd[p + nm + ".bias"] = n(H, std=0.1)
    return sd


def attention(q, k, v, add_mask, head_dim: int):
    """HF BertSelfAttention core on [B, heads, S, hd] tensors: softmax(q k^T / sqrt(hd) + add_mask) v."""
    att = torch.softmax((q @ k.transpose(-1, -2)) / math.sqrt(head_dim) + add_mask, dim=-1)
    return att @ v


def bert_hidden(sd: Dict[str, torch.Tensor], config: dict, input_ids, attention_mask, token_type_ids=None,
                dtype=torch.float32):
    """last_hidden_state [B, S, hidden] of HF BertModel in `dtype` (pad positions not zeroed)."""
    dev = input_ids.device
    w = {k: v.to(device=dev, dtype=dtype) for k, v in sd.items()}
    B, S = input_ids.shape
    H, nh, eps = config["hidden_size"], config["num_attention_heads"], config["layer_norm_eps"]
    hd = H // nh
    if token_type_ids is None:
        token_type_ids = torch.zeros_like(input_ids)
    pos = torch.arange(S, device=dev)
    x = w["embeddings.word_embeddings.weight"][input_ids] + w["embeddings.token_type_embeddings.weight"][token_type_ids] \
        + w["embeddings.position_embeddings.weight"][pos][None]
    x = F.layer_norm(x, (H,), w["embeddings.LayerNorm.weight"], w["embeddings.LayerNorm.bias"], eps)
    mask = attention_mask.bool()
    add_mask = torch.zeros(B, 1, 1, S, device=dev, dtype=dtype).masked_fill(~mask[:, None, None, :], torch.finfo(dtype).min)
    for i in range(config["num_hidden_layers"]):
        p = f"encoder.layer.{i}."
        lin = lambda name, t: F.linear(t, w[p + name + ".weight"], w[p + name + ".bias"])  # noqa: E731
        q = lin("attention.self.query", x).view(B, S, nh, hd).transpose(1, 2)
        k = lin("attention.self.key", x).view(B, S, nh, hd).transpose(1, 2)
        v = lin("attention.self.value", x).view(B, S, nh, hd).transpose(1, 2)
        ctx = attention(q, k, v, add_mask, hd).transpose(1, 2).reshape(B, S, H)
        x = F.layer_norm(lin("attention.output.dense", ctx) + x, (H,), w[p + "attention.output.LayerNorm.weight"],
                         w[p + "attention.output.LayerNorm.bias"], eps)
        ff = F.gelu(lin("intermediate.dense", x))           # exact erf GELU (hidden_act="gelu")
        x = F.layer_norm(lin("output.dense", ff) + x, (H,), w[p + "output.LayerNorm.weight"],
                         w[p + "output.LayerNorm.bias"], eps)
    return x


def bert_forward(sd: Dict[str, torch.Tensor], config: dict, input_ids, attention_mask, token_type_ids=None,
                 pooling: str = "average", dtype=torch.float32):
    """Returns [B, hidden] in `dtype` (float32 = exact restatement; float16 on CUDA mirrors `.half()`)."""
    x = bert_hidden(sd, config, input_ids, attention_mask, token_type_ids, dtype)
    mask = attention_mask.bool()
    last = x.masked_fill(~mask[..., None], 0.0)              # contriever.py:46
    if pooling == "average":
        return last.sum(dim=1) / attention_mask.sum(dim=1)[..., None].to(dtype)   # contriever.py:49
    return last[:, 0]                                        # contriever.py:51
