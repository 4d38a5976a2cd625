"""Seeded Llama reader fixture: a 2-layer LlamaForCausalLM with the released models' head_dim 128, GQA 4:1 and a
vocabulary that is not a multiple of 128.  Shared by make_llama_golden.py, the CPU tests and the GPU tests; the
weights are regenerated from the seed, only the golden NLL is committed.

No released Llama checkpoint is available offline, so parity is shown on these seeded weights."""
from __future__ import annotations

import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "llama_golden.npz")

CONFIG = dict(model_type="llama", num_hidden_layers=2, hidden_size=512, num_attention_heads=4, num_key_value_heads=1,
              intermediate_size=1024, vocab_size=1000, max_position_embeddings=4096, rope_theta=10000.0,
              rms_norm_eps=1e-5, hidden_act="silu", tie_word_embeddings=False, attention_bias=False, mlp_bias=False,
              rope_scaling=None, head_dim=128, bos_token_id=1, eos_token_id=2)
# window lengths of the golden: the attention kernel's 16-row warp tiles and 64-row blocks on both sides, and max_pos
LENGTHS = (1, 2, 63, 64, 127, 128, 129, 1000, 4096)
SEED = 20261017


def seeded_state_dict(config=None, seed: int = SEED):
    """HF LlamaForCausalLM keys, fp32.  Scales are chosen so that attention is far from uniform and the logits spread
    over several nats; every value is finite in fp16."""
    c = dict(CONFIG, **(config or {}))
    g = torch.Generator().manual_seed(seed)
    H, I, V = c["hidden_size"], c["intermediate_size"], c["vocab_size"]
    KV = c["num_key_value_heads"] * 128

    def n(*shape, std):
        return (torch.randn(*shape, generator=g) * std).float()

    # a tied embedding is also the LM head: the head's scale keeps its logits in the same range
    embed_std = 3.0 / H ** 0.5 if c["tie_word_embeddings"] else 1.0
    sd = {"model.embed_tokens.weight": n(V, H, std=embed_std), "model.norm.weight": 1.0 + n(H, std=0.1)}
    for i in range(c["num_hidden_layers"]):
        p = f"model.layers.{i}."
        sd[p + "self_attn.q_proj.weight"] = n(H, H, std=1.5 / H ** 0.5)
        sd[p + "self_attn.k_proj.weight"] = n(KV, H, std=1.5 / H ** 0.5)
        sd[p + "self_attn.v_proj.weight"] = n(KV, H, std=1.0 / H ** 0.5)
        sd[p + "self_attn.o_proj.weight"] = n(H, H, std=1.0 / H ** 0.5)
        sd[p + "mlp.gate_proj.weight"] = n(I, H, std=1.0 / H ** 0.5)
        sd[p + "mlp.up_proj.weight"] = n(I, H, std=1.0 / H ** 0.5)
        sd[p + "mlp.down_proj.weight"] = n(H, I, std=1.0 / I ** 0.5)
        sd[p + "input_layernorm.weight"] = 1.0 + n(H, std=0.1)
        sd[p + "post_attention_layernorm.weight"] = 1.0 + n(H, std=0.1)
    if not c["tie_word_embeddings"]:
        sd["lm_head.weight"] = n(V, H, std=3.0 / H ** 0.5)
    return sd


def window_ids(seed: int = SEED):
    """The golden's windows: seeded ids in [0, vocab), with the first and last id of the vocabulary present."""
    rng = np.random.default_rng(seed)
    out = []
    for S in LENGTHS:
        ids = rng.integers(0, CONFIG["vocab_size"], S).astype(np.int64)
        if S >= 4:
            ids[1], ids[-1] = 0, CONFIG["vocab_size"] - 1
        out.append(ids)
    return out


def hf_model(config=None, dtype=torch.float32, seed: int = SEED, attn_implementation: str = "eager"):
    """transformers LlamaForCausalLM with the seeded weights."""
    import transformers
    c = dict(CONFIG, **(config or {}))
    kw = {k: v for k, v in c.items() if k != "model_type"}
    cfg = transformers.LlamaConfig(**kw)
    cfg._attn_implementation = attn_implementation
    model = transformers.LlamaForCausalLM(cfg).eval()
    sd = seeded_state_dict(c, seed)
    missing, unexpected = model.load_state_dict(sd, strict=False)
    tied = ["lm_head.weight"] if c["tie_word_embeddings"] else []
    assert not unexpected and all("rotary" in m or m in tied for m in missing), (missing, unexpected)
    if tied:
        assert model.lm_head.weight.data_ptr() == model.model.embed_tokens.weight.data_ptr()
    model = model.to(dtype)
    # `.to(dtype)` also casts the RoPE inverse frequencies; from_pretrained(torch_dtype=...) keeps them in fp32
    for mod in model.modules():
        if hasattr(mod, "inv_freq") and hasattr(mod, "compute_default_rope_parameters"):
            mod.inv_freq = mod.compute_default_rope_parameters(mod.config)[0]
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
    """A Llama-style fast tokenizer over the fixture vocabulary: <unk> 0, <s> 1 (BOS, prepended to every encoding),
    </s> 2 (EOS), and the words w3 .. w999 split on whitespace."""
    from tokenizers import Tokenizer, models, pre_tokenizers, processors
    from transformers import PreTrainedTokenizerFast
    V = CONFIG["vocab_size"]
    vocab = {"<unk>": 0, "<s>": 1, "</s>": 2, **{f"w{i}": i for i in range(3, V)}}
    tok = Tokenizer(models.WordLevel(vocab, unk_token="<unk>"))
    tok.pre_tokenizer = pre_tokenizers.WhitespaceSplit()
    tok.post_processor = processors.TemplateProcessing(single="<s> $A", special_tokens=[("<s>", 1)])
    return PreTrainedTokenizerFast(tokenizer_object=tok, unk_token="<unk>", bos_token="<s>", eos_token="</s>")


def build_dir(root: str, config=None, seed: int = SEED) -> str:
    """An HF reader directory: config.json, model.safetensors and the tokenizer."""
    import json as _json

    from safetensors.torch import save_file
    c = dict(CONFIG, **(config or {}))
    os.makedirs(root, exist_ok=True)
    with open(os.path.join(root, "config.json"), "w") as f:
        _json.dump(dict(c, architectures=["LlamaForCausalLM"]), f)
    save_file({k: v.contiguous() for k, v in seeded_state_dict(c, seed).items()}, os.path.join(root, "model.safetensors"))
    tokenizer().save_pretrained(root)
    return root
