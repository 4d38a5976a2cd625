"""Generates tests/golden/encoder_t5_*.npz: `transformers.T5EncoderModel` (fp32, eager attention) on the seeded weights of
`oracle.t5_oracle.seeded_state_dict` and fixed token batches, followed by the restated sentence-transformers head
(`oracle.t5_oracle.st_head`).  Only token batches and outputs are committed; the weights are rebuilt from the seed.

    python tests/golden/make_t5_golden.py
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))

from transformers import T5Config, T5EncoderModel  # noqa: E402

from oracle.t5_oracle import T5_CONFIG, seeded_state_dict, st_head  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = {
    # 2 layers, small vocabulary, query-length sequences (the <= 32-token attention kernel)
    "encoder_t5_l2": dict(num_layers=2, vocab_size=2048, seed=31, B=6, S=24, min_len=3),
    # 12 layers (T5-base), sequences past 32 tokens (the flash attention kernel) mixed with short ones
    "encoder_t5_l12": dict(num_layers=12, vocab_size=32128, seed=32, B=5, S=160, min_len=5),
}


def token_batch(rng, B, S, vocab, min_len):
    lens = rng.integers(min_len, S + 1, B)
    lens[0] = S
    lens[-1] = min(lens[-1], 20)
    ids = rng.integers(3, vocab, (B, S))
    mask = (np.arange(S)[None, :] < lens[:, None]).astype(np.int64)
    return (ids * mask).astype(np.int64), mask            # <pad> = 0 on the right


def case_config(c):
    return dict(T5_CONFIG, num_layers=c["num_layers"], vocab_size=c["vocab_size"])


def main():
    for name, c in CASES.items():
        cfg = case_config(c)
        sd = seeded_state_dict(cfg, c["seed"])
        model = T5EncoderModel(T5Config(d_model=768, d_kv=64, d_ff=cfg["d_ff"], num_layers=cfg["num_layers"],
                                        num_heads=12, vocab_size=cfg["vocab_size"],
                                        relative_attention_num_buckets=cfg["relative_attention_num_buckets"],
                                        relative_attention_max_distance=cfg["relative_attention_max_distance"],
                                        layer_norm_epsilon=cfg["layer_norm_epsilon"], feed_forward_proj="relu",
                                        dropout_rate=0.0, attn_implementation="eager"))
        missing, unexpected = model.load_state_dict({k: v for k, v in sd.items() if not k.startswith("dense.")},
                                                    strict=False)
        assert not missing and not unexpected, (missing, unexpected)
        model.eval()
        rng = np.random.default_rng(c["seed"])
        ids, mask = token_batch(rng, c["B"], c["S"], c["vocab_size"], c["min_len"])
        with torch.no_grad():
            tok = model(input_ids=torch.from_numpy(ids), attention_mask=torch.from_numpy(mask)).last_hidden_state
            m = torch.from_numpy(mask)
            out = dict(out_mean=st_head(tok, m, "average"), out_cls=st_head(tok, m, "cls"),
                       out_head=st_head(tok, m, "average", sd["dense.weight"], sd["dense.bias"], normalize=True))
        np.savez_compressed(os.path.join(HERE, name + ".npz"), input_ids=ids, attention_mask=mask, seed=c["seed"],
                            **{k: v.numpy().astype(np.float32) for k, v in out.items()},
                            **{"cfg_" + k: v for k, v in cfg.items()})
        print(name, ids.shape, float(out["out_mean"].abs().mean()))


if __name__ == "__main__":
    main()
