"""Seeded OLMo and OLMo-2 reader fixtures: 2-layer OlmoForCausalLM (tied head, clip_qkv set so that the clamp acts on
a few per cent of the q / k / v elements, rope_theta 1e4) and Olmo2ForCausalLM (GQA 4:1, untied head, rope_theta 5e5),
both with head_dim 128 and a vocabulary that is not a multiple of 128.  Their config.json files use the Hub's field
names (rope_theta), as the released OLMo configs do.  Shared by make_olmo_golden.py, the CPU tests and the GPU tests;
the weights are regenerated from the seed, only the golden NLL is committed.

No released OLMo checkpoint is available offline, so parity is shown on these seeded weights."""
from __future__ import annotations

import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "olmo_golden.npz")

_COMMON = dict(num_hidden_layers=2, hidden_size=512, num_attention_heads=4, intermediate_size=1024, vocab_size=1000,
               max_position_embeddings=2048, hidden_act="silu", attention_bias=False, pad_token_id=1,
               bos_token_id=None, eos_token_id=0)
CONFIGS = {
    "olmo": dict(_COMMON, model_type="olmo", num_key_value_heads=4, rope_theta=10000.0, clip_qkv=3.0,
                 tie_word_embeddings=True),
    "olmo2": dict(_COMMON, model_type="olmo2", num_key_value_heads=1, rope_theta=500000.0, rms_norm_eps=1e-6,
                  tie_word_embeddings=False),
}
ARCH = {"olmo": "OlmoForCausalLM", "olmo2": "Olmo2ForCausalLM"}
# the share of q / k / v elements the OLMo fixture's clamp changes must be at least this (the golden's windows)
MIN_CLIPPED = 0.01
# window lengths of the golden: the attention kernel's 16-row warp tiles and 64-row blocks on both sides, and max_pos
LENGTHS = (1, 2, 15, 16, 17, 63, 64, 65, 127, 128, 129, 1000, 2048)
SEED = 20261019


def config(kind: str, **change) -> dict:
    return dict(CONFIGS[kind], **change)


def seeded_state_dict(cfg, seed: int = SEED):
    """HF Olmo / Olmo2ForCausalLM keys, fp32.  Scales are chosen so that attention is far from uniform, the logits
    spread over several nats and (OLMo) the clamp acts; every value is finite in fp16."""
    g = torch.Generator().manual_seed(seed)
    H, I, V = cfg["hidden_size"], cfg["intermediate_size"], cfg["vocab_size"]
    KV = (cfg.get("num_key_value_heads") or cfg["num_attention_heads"]) * 128
    v2 = cfg["model_type"] == "olmo2"

    def n(*shape, std):
        return (torch.randn(*shape, generator=g) * std).float()

    # a tied embedding is also the LM head: scaled as the untied head is
    sd = {"model.embed_tokens.weight": n(V, H, std=3.0 / H ** 0.5 if cfg.get("tie_word_embeddings") else 1.0)}
    for i in range(cfg["num_hidden_layers"]):
        p = f"model.layers.{i}."
        sd[p + "self_attn.q_proj.weight"] = n(H, H, std=1.5 / H ** 0.5)
        sd[p + "self_attn.k_proj.weight"] = n(KV, H, std=1.5 / H ** 0.5)
        sd[p + "self_attn.v_proj.weight"] = n(KV, H, std=1.5 / H ** 0.5)
        sd[p + "self_attn.o_proj.weight"] = n(H, H, std=1.0 / H ** 0.5)
        sd[p + "mlp.gate_proj.weight"] = n(I, H, std=1.0 / H ** 0.5)
        sd[p + "mlp.up_proj.weight"] = n(I, H, std=1.0 / H ** 0.5)
        sd[p + "mlp.down_proj.weight"] = n(H, I, std=1.0 / I ** 0.5)
        if v2:
            sd[p + "self_attn.q_norm.weight"] = 1.0 + n(H, std=0.1)
            sd[p + "self_attn.k_norm.weight"] = 1.0 + n(KV, std=0.1)
            sd[p + "post_attention_layernorm.weight"] = 1.0 + n(H, std=0.1)
            sd[p + "post_feedforward_layernorm.weight"] = 1.0 + n(H, std=0.1)
    if v2:
        sd["model.norm.weight"] = 1.0 + n(H, std=0.1)
    if not cfg.get("tie_word_embeddings"):
        sd["lm_head.weight"] = n(V, H, std=3.0 / H ** 0.5)
    return sd


def window_ids(kind: str, seed: int = SEED):
    """The golden's windows: seeded ids in [0, vocab), with the first and last id of the vocabulary present."""
    rng = np.random.default_rng(seed + (kind == "olmo2"))
    V = CONFIGS[kind]["vocab_size"]
    out = []
    for S in LENGTHS:
        ids = rng.integers(0, V, S).astype(np.int64)
        if S >= 4:
            ids[1], ids[-1] = 0, V - 1
        out.append(ids)
    return out


def hf_model(cfg, dtype=torch.float32, seed: int = SEED, attn_implementation: str = "eager", sd=None):
    """transformers Olmo / Olmo2ForCausalLM with the seeded weights (or `sd`)."""
    import transformers
    kw = {k: v for k, v in cfg.items() if k != "model_type"}
    if cfg["model_type"] == "olmo2":
        c, cls = transformers.Olmo2Config(**kw), transformers.Olmo2ForCausalLM
    else:
        c, cls = transformers.OlmoConfig(**kw), transformers.OlmoForCausalLM
    c._attn_implementation = attn_implementation
    model = cls(c).eval()
    missing, unexpected = model.load_state_dict(seeded_state_dict(cfg, seed) if sd is None else sd, strict=False)
    assert not unexpected and all(m == "lm_head.weight" and cfg.get("tie_word_embeddings") for m in missing), \
        (missing, unexpected)
    model = model.to(dtype)
    # `.to(dtype)` also casts the RoPE inverse frequencies; from_pretrained(torch_dtype=...) keeps them in fp32
    for mod in model.modules():
        if hasattr(mod, "inv_freq") and hasattr(mod, "compute_default_rope_parameters"):
            mod.inv_freq = mod.compute_default_rope_parameters(mod.config)[0].to(mod.inv_freq.device)
    return model


def hf_token_nll(model, ids) -> np.ndarray:
    """nll[t] = -log p(ids[t] | ids[:t]) from the model's logits in float64, 0 at t = 0."""
    x = torch.as_tensor(np.asarray(ids), dtype=torch.long, device=model.device)[None]
    with torch.no_grad():
        logits = model(x).logits[0].double()
    lp = torch.log_softmax(logits, dim=-1)
    out = np.zeros(len(ids), np.float64)
    if len(ids) > 1:
        out[1:] = (-lp[:-1].gather(1, x[0, 1:, None]).squeeze(1)).cpu().numpy()
    return out


def tokenizer():
    """An OLMo-style fast tokenizer over the fixture vocabulary: <|endoftext|> 0 (eos, never added to an encoding; no
    BOS, as OLMo's tokenizers add none), <|padding|> 1 and the words w2 .. w999 split on whitespace."""
    from tokenizers import Tokenizer, models, pre_tokenizers
    from transformers import PreTrainedTokenizerFast
    V = CONFIGS["olmo"]["vocab_size"]
    vocab = {"<|endoftext|>": 0, "<|padding|>": 1, **{f"w{i}": i for i in range(2, V)}}
    tok = Tokenizer(models.WordLevel(vocab, unk_token="<|endoftext|>"))
    tok.pre_tokenizer = pre_tokenizers.WhitespaceSplit()
    return PreTrainedTokenizerFast(tokenizer_object=tok, unk_token="<|endoftext|>", eos_token="<|endoftext|>",
                                   pad_token="<|padding|>")


def build_dir(root: str, cfg, seed: int = SEED) -> str:
    """An HF reader directory: config.json, model.safetensors and the tokenizer."""
    import json as _json

    from safetensors.torch import save_file
    os.makedirs(root, exist_ok=True)
    with open(os.path.join(root, "config.json"), "w") as f:
        _json.dump(dict(cfg, architectures=[ARCH[cfg["model_type"]]]), f)
    save_file({k: v.contiguous() for k, v in seeded_state_dict(cfg, seed).items()},
              os.path.join(root, "model.safetensors"))
    tokenizer().save_pretrained(root)
    return root
