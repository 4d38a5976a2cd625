"""Deterministic local stand-in for a Contriever checkpoint, rebuilt on demand (nothing large is committed):

    <dir>/model_id/config.json + vocab.txt      a 2-layer BERT (hidden 768) with a 2048-entry WordPiece vocabulary
    <dir>/ckpt/checkpoint.pth                   {"opt": Namespace(retriever_model_id=<dir>/model_id),
                                                 "model": {"encoder_q.<HF key>": w, "encoder_k.<HF key>": junk, "queue": junk}}
                                                the MoCo form `contriever/src/contriever.py:103-126` loads
    <dir>/hf/                                   the same weights saved with `BertModel.save_pretrained` (the HF branch, :127-136)

Weights come from `oracle.bert_oracle.seeded_state_dict` (CPU generator: identical on every machine), so the golden
embeddings committed in tests/golden/retriever_ckpt.npz -- produced by the REFERENCE's `load_retriever` on exactly
this directory (make_retriever_golden.py) -- hold on any machine, without a reference checkout."""
import argparse
import json
import os

import torch

CONFIG = dict(hidden_size=768, num_hidden_layers=2, num_attention_heads=12, intermediate_size=3072, vocab_size=2048,
              max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12)
SEED = 21
QUERIES = ["who wrote the origin of species", "What is the capital of Australia?", "b200 hbm3e bandwidth",
           "when did the berlin wall fall", "a", "tallest mountain in south america ?", "largest moon of saturn",
           "how many sm does a b200 have and how large is its l2 cache in megabytes"]


def vocab_tokens():
    toks = ["[PAD]"] + [f"[unused{i}]" for i in range(99)] + ["[UNK]", "[CLS]", "[SEP]", "[MASK]"]
    toks += list("abcdefghijklmnopqrstuvwxyz0123456789?.,!") + ["##" + c for c in "abcdefghijklmnopqrstuvwxyz0123456789"]
    words = ["the", "of", "who", "what", "when", "how", "is", "in", "a", "did", "does", "many", "large", "and", "its",
             "capital", "wall", "fall", "moon", "mountain", "south", "america", "tall", "##est", "##er", "##s", "##ed", "##ing",
             "wrote", "origin", "species", "australia", "berlin", "saturn", "largest", "band", "##width", "cache", "have", "mega", "##bytes"]
    toks += words
    i = 0
    while len(toks) < CONFIG["vocab_size"]:
        toks.append(f"w{i}")
        i += 1
    return toks[: CONFIG["vocab_size"]]


def build(root: str) -> dict:
    from oracle.bert_oracle import seeded_state_dict
    mid, ck, hf = os.path.join(root, "model_id"), os.path.join(root, "ckpt"), os.path.join(root, "hf")
    for d in (mid, ck, hf):
        os.makedirs(d, exist_ok=True)
    cfg = {"model_type": "bert", "architectures": ["BertModel"], "hidden_act": "gelu", "hidden_dropout_prob": 0.1,
           "attention_probs_dropout_prob": 0.1, "initializer_range": 0.02, "pad_token_id": 0,
           "position_embedding_type": "absolute", **CONFIG}
    tok_cfg = {"do_lower_case": True, "tokenizer_class": "BertTokenizer", "model_max_length": 512}
    for d in (mid, hf):
        with open(os.path.join(d, "config.json"), "w") as f:
            json.dump(cfg, f)
        with open(os.path.join(d, "vocab.txt"), "w") as f:
            f.write("\n".join(vocab_tokens()) + "\n")
        with open(os.path.join(d, "tokenizer_config.json"), "w") as f:
            json.dump(tok_cfg, f)
    sd = seeded_state_dict(CONFIG, SEED)
    g = torch.Generator().manual_seed(SEED + 1)
    model = {f"encoder_q.{k}": v for k, v in sd.items()}
    model.update({f"encoder_k.{k}": torch.randn(v.shape, generator=g) for k, v in list(sd.items())[:3]})
    model["queue"] = torch.randn(8, 4, generator=g)
    torch.save({"opt": argparse.Namespace(retriever_model_id=mid), "model": model}, os.path.join(ck, "checkpoint.pth"))
    torch.save({f"bert.{k}" if False else k: v for k, v in sd.items()}, os.path.join(hf, "pytorch_model.bin"))
    return {"model_id": mid, "ckpt": ck, "hf": hf, "state_dict": sd}
