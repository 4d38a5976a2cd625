"""Deterministic local stand-ins for DRAGON-RoBERTa's two encoders, rebuilt on demand (nothing large is committed):

    <root>/dragon-roberta-query-encoder-fixture/     HF RobertaModel directory (config.json, model.safetensors,
    <root>/dragon-roberta-context-encoder-fixture/   tokenizer.json + tokenizer_config.json ...), the layout
                                                     `AutoModel` / `AutoTokenizer.from_pretrained(dir)` read offline

Each is a 2-layer RoBERTa with roberta-base geometry (hidden 768, 12 heads, intermediate 3072, vocabulary 50265,
max_position_embeddings 514, type_vocab_size 1, layer_norm_eps 1e-5, pad_token_id 1); the two differ only in the seed
of their weights (`oracle.bert_oracle.seeded_state_dict`, CPU generator: identical on every machine, plus a seeded
pooler that the encoders do not read).  The tokenizer is a small byte-level BPE: the GPT-2 byte alphabet, <s> = 0,
<pad> = 1, </s> = 2, <unk> = 3, a fixed merge list built from WORDS, <mask> last; built with
`RobertaTokenizer(vocab=..., merges=...)` and saved with `save_pretrained`.  The directory names carry "dragon", the
reference's name dispatch (src/search.py:241, src/embed.py:123)."""
import json
import os

import torch

CONFIG = dict(hidden_size=768, num_hidden_layers=2, num_attention_heads=12, intermediate_size=3072, vocab_size=50265,
              max_position_embeddings=514, type_vocab_size=1, layer_norm_eps=1e-5)
SEEDS = {"query": 51, "context": 52}
NAMES = {"query": "dragon-roberta-query-encoder-fixture", "context": "dragon-roberta-context-encoder-fixture"}
WORDS = ["the", "of", "who", "what", "when", "how", "is", "in", "a", "did", "does", "many", "large", "and", "its",
         "capital", "wall", "fall", "moon", "mountain", "south", "america", "tall", "est", "wrote", "origin", "species",
         "australia", "berlin", "saturn", "largest", "band", "width", "cache", "have", "mega", "bytes", "title", "text",
         "passage", "question", "answer", "river", "city", "year", "first"]


def bytes_to_unicode():
    """GPT-2's reversible byte -> printable character map (the byte-level BPE alphabet)."""
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return dict(zip(bs, [chr(c) for c in cs]))


def vocab_and_merges():
    """({token: id}, [(left, right), ...]): specials, the 256 byte symbols, then the result of every merge in rank order;
    each word of WORDS is merged left to right, with and without the leading space symbol 'Ġ'."""
    vocab = {"<s>": 0, "<pad>": 1, "</s>": 2, "<unk>": 3}
    for ch in sorted(bytes_to_unicode().values()):
        vocab[ch] = len(vocab)
    merges = []
    for w in WORDS:
        for form in ("Ġ" + w, w):
            left = form[0]
            for ch in form[1:]:
                merged = left + ch
                if merged not in vocab:
                    merges.append((left, ch))
                    vocab[merged] = len(vocab)
                left = merged
    vocab["<mask>"] = len(vocab)
    return vocab, merges


def tokenizer():
    from transformers import RobertaTokenizer
    vocab, merges = vocab_and_merges()
    return RobertaTokenizer(vocab=vocab, merges=merges, model_max_length=512)


def hf_config(seed_name: str) -> dict:
    return {"model_type": "roberta", "architectures": ["RobertaModel"], "hidden_act": "gelu", "hidden_dropout_prob": 0.1,
            "attention_probs_dropout_prob": 0.1, "initializer_range": 0.02, "pad_token_id": 1, "bos_token_id": 0,
            "eos_token_id": 2, "position_embedding_type": "absolute", "_name_or_path": NAMES[seed_name], **CONFIG}


def state_dict(which: str):
    """HF RobertaModel weights of the query or context encoder (fp32, pooler included)."""
    from oracle.bert_oracle import seeded_state_dict
    seed = SEEDS[which]
    sd = seeded_state_dict(CONFIG, seed)
    g = torch.Generator().manual_seed(seed + 1000)
    sd["pooler.dense.weight"] = torch.randn(768, 768, generator=g) * 0.04
    sd["pooler.dense.bias"] = torch.randn(768, generator=g) * 0.02
    return sd


def build(root: str) -> dict:
    """Writes both directories under root; returns {"query" | "context": {"dir", "state_dict", "config"}}."""
    from safetensors.torch import save_file
    out = {}
    tok = tokenizer()
    for which in ("query", "context"):
        d = os.path.join(root, NAMES[which])
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, "config.json"), "w") as f:
            json.dump(hf_config(which), f, indent=1, sort_keys=True)
        sd = state_dict(which)
        save_file({k: v.contiguous() for k, v in sd.items()}, os.path.join(d, "model.safetensors"),
                  metadata={"format": "pt"})
        tok.save_pretrained(d)
        out[which] = {"dir": d, "state_dict": sd, "config": CONFIG}
    return out
