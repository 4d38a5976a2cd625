"""Seeded GPT-NeoX reader fixture: a 2-layer GPTNeoXForCausalLM with pythia-1b's head_dim 256 and rotary_pct 0.25, and
a vocabulary that is not a multiple of 128.  Its config.json uses the Hub's field names (rotary_pct, rotary_emb_base),
as the released Pythia configs do.  Shared by make_neox_golden.py, the CPU tests and the GPU tests; the weights are
regenerated from the seed, only the golden NLL is committed.

No released Pythia checkpoint is available offline, so parity is shown on these seeded weights."""
from __future__ import annotations

import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "neox_golden.npz")

CONFIG = dict(model_type="gpt_neox", num_hidden_layers=2, hidden_size=512, num_attention_heads=2,
              intermediate_size=2048, vocab_size=1000, max_position_embeddings=2048, rotary_pct=0.25,
              rotary_emb_base=10000, layer_norm_eps=1e-5, hidden_act="gelu", use_parallel_residual=True,
              tie_word_embeddings=False, bos_token_id=0, eos_token_id=0)
# window lengths of the golden: the attention kernel's 16-row warp tiles and 64-row blocks on both sides, and max_pos
LENGTHS = (1, 2, 15, 16, 17, 63, 64, 65, 127, 128, 129, 1000, 2048)
SEED = 20261018
# non-weight buffers older GPT-NeoX checkpoints carry, per layer
LEGACY_BUFFERS = ("attention.bias", "attention.masked_bias", "attention.rotary_emb.inv_freq")


def seeded_state_dict(config=None, seed: int = SEED):
    """HF GPTNeoXForCausalLM keys, fp32.  Scales are chosen so that attention is far from uniform and the logits spread
    over several nats; every value is finite in fp16."""
    c = dict(CONFIG, **(config or {}))
    g = torch.Generator().manual_seed(seed)
    H, I, V = c["hidden_size"], c["intermediate_size"], c["vocab_size"]

    def n(*shape, std):
        return (torch.randn(*shape, generator=g) * std).float()

    sd = {"gpt_neox.embed_in.weight": n(V, H, std=1.0)}
    for i in range(c["num_hidden_layers"]):
        p = f"gpt_neox.layers.{i}."
        for ln in ("input_layernorm", "post_attention_layernorm"):
            sd[p + ln + ".weight"] = 1.0 + n(H, std=0.1)
            sd[p + ln + ".bias"] = n(H, std=0.1)
        sd[p + "attention.query_key_value.weight"] = n(3 * H, H, std=1.5 / H ** 0.5)
        sd[p + "attention.query_key_value.bias"] = n(3 * H, std=0.1)
        sd[p + "attention.dense.weight"] = n(H, H, std=1.0 / H ** 0.5)
        sd[p + "attention.dense.bias"] = n(H, std=0.1)
        sd[p + "mlp.dense_h_to_4h.weight"] = n(I, H, std=1.0 / H ** 0.5)
        sd[p + "mlp.dense_h_to_4h.bias"] = n(I, std=0.1)
        sd[p + "mlp.dense_4h_to_h.weight"] = n(H, I, std=1.0 / I ** 0.5)
        sd[p + "mlp.dense_4h_to_h.bias"] = n(H, std=0.1)
    sd["gpt_neox.final_layer_norm.weight"] = 1.0 + n(H, std=0.1)
    sd["gpt_neox.final_layer_norm.bias"] = n(H, std=0.1)
    sd["embed_out.weight"] = n(V, H, std=3.0 / H ** 0.5)
    return sd


def legacy_buffers(config=None):
    """The buffers of an older checkpoint: the causal mask (bool [1, 1, max_pos, max_pos]), masked_bias and inv_freq."""
    c = dict(CONFIG, **(config or {}))
    P, d = c["max_position_embeddings"], c["hidden_size"] // c["num_attention_heads"]
    rot = int(d * c["rotary_pct"])
    mask = torch.tril(torch.ones(P, P, dtype=torch.bool)).view(1, 1, P, P)
    inv = 1.0 / (c["rotary_emb_base"] ** (torch.arange(0, rot, 2).float() / rot))
    out = {}
    for i in range(c["num_hidden_layers"]):
        p = f"gpt_neox.layers.{i}."
        out[p + "attention.bias"] = mask
        out[p + "attention.masked_bias"] = torch.tensor(-1e9)
        out[p + "attention.rotary_emb.inv_freq"] = inv
    return out


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


def hf_model(config=None, dtype=torch.float32, seed: int = SEED, attn_implementation: str = "eager", sd=None):
    """transformers GPTNeoXForCausalLM with the seeded weights (or `sd`)."""
    import transformers
    c = dict(CONFIG, **(config or {}))
    kw = {k: v for k, v in c.items() if k != "model_type"}
    cfg = transformers.GPTNeoXConfig(**kw)
    cfg._attn_implementation = attn_implementation
    model = transformers.GPTNeoXForCausalLM(cfg).eval()
    missing, unexpected = model.load_state_dict(seeded_state_dict(c, seed) if sd is None else sd, strict=False)
    assert not unexpected and all("rotary" in m or "masked_bias" in m or m.endswith("attention.bias") for m in missing), \
        (missing, unexpected)
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
    """A GPT-NeoX-style fast tokenizer over the fixture vocabulary: <|endoftext|> 0 (eos, bos and unk, never added to
    an encoding) and the words w1 .. w999 split on whitespace."""
    from tokenizers import Tokenizer, models, pre_tokenizers
    from transformers import PreTrainedTokenizerFast
    V = CONFIG["vocab_size"]
    vocab = {"<|endoftext|>": 0, **{f"w{i}": i for i in range(1, V)}}
    tok = Tokenizer(models.WordLevel(vocab, unk_token="<|endoftext|>"))
    tok.pre_tokenizer = pre_tokenizers.WhitespaceSplit()
    return PreTrainedTokenizerFast(tokenizer_object=tok, unk_token="<|endoftext|>", bos_token="<|endoftext|>",
                                   eos_token="<|endoftext|>")


def build_dir(root: str, config=None, seed: int = SEED, pickle: bool = False) -> str:
    """An HF reader directory: config.json, model.safetensors (or, with pickle=True, a pytorch_model.bin that also
    carries the legacy buffers) and the tokenizer."""
    import json as _json

    from safetensors.torch import save_file
    c = dict(CONFIG, **(config or {}))
    os.makedirs(root, exist_ok=True)
    with open(os.path.join(root, "config.json"), "w") as f:
        _json.dump(dict(c, architectures=["GPTNeoXForCausalLM"]), f)
    sd = {k: v.contiguous() for k, v in seeded_state_dict(c, seed).items()}
    if pickle:
        torch.save(dict(sd, **legacy_buffers(c)), os.path.join(root, "pytorch_model.bin"))
    else:
        save_file(sd, os.path.join(root, "model.safetensors"))
    tokenizer().save_pretrained(root)
    return root
