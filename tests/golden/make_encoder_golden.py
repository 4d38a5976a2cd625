"""Generates tests/golden/encoder_*.npz by running the REFERENCE's own class
(`contriever.src.contriever.Contriever`, contriever/src/contriever.py:11-55 of the reference checkout) on seeded weights
and fixed token batches.  Needs a checkout of the reference project, named by REFERENCE_ROOT:

    REFERENCE_ROOT=<reference checkout> python tests/golden/make_encoder_golden.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.environ["REFERENCE_ROOT"])
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from transformers import BertConfig  # noqa: E402

from contriever.src.contriever import Contriever  # noqa: E402  (the reference class)
from oracle.bert_oracle import seeded_state_dict  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def token_batch(rng, B, S, vocab, min_len):
    lens = rng.integers(min_len, S + 1, B)
    lens[0] = S
    ids = rng.integers(1000 % vocab, vocab, (B, S))
    mask = (np.arange(S)[None, :] < lens[:, None]).astype(np.int64)
    ids = ids * mask                                   # [PAD] = 0 on the right
    tt = np.zeros((B, S), np.int64)
    return ids.astype(np.int64), mask, tt


def main():
    cases = {
        "encoder_l2": dict(layers=2, vocab=2048, seed=11, B=6, S=24, min_len=3),
        "encoder_l12": dict(layers=12, vocab=30522, seed=12, B=4, S=40, min_len=5),
    }
    for name, c in cases.items():
        cfg = dict(hidden_size=768, num_hidden_layers=c["layers"], num_attention_heads=12, intermediate_size=3072,
                   vocab_size=c["vocab"], max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12)
        sd = seeded_state_dict(cfg, c["seed"])
        rng = np.random.default_rng(c["seed"])
        ids, mask, tt = token_batch(rng, c["B"], c["S"], c["vocab"], c["min_len"])
        out = {}
        for pooling in ("average", "cls"):
            model = Contriever(BertConfig(**cfg), pooling=pooling)
            missing, unexpected = model.load_state_dict(sd, strict=False)
            assert not unexpected and all("position_ids" in m for m in missing), (missing, unexpected)
            model.eval()
            with torch.no_grad():
                emb = model(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask),
                            token_type_ids=torch.from_numpy(tt))
            out[pooling] = emb.numpy().astype(np.float32)
        np.savez_compressed(os.path.join(HERE, name + ".npz"), input_ids=ids, attention_mask=mask, token_type_ids=tt,
                            out_average=out["average"], out_cls=out["cls"], seed=c["seed"],
                            **{"cfg_" + k: v for k, v in cfg.items()})
        print(name, out["average"].shape, float(np.abs(out["average"]).mean()))


if __name__ == "__main__":
    main()
