"""Writes tests/golden/olmo_golden.npz: the fp64 per-token NLL of transformers' OlmoForCausalLM and Olmo2ForCausalLM
(run in float64 on the CPU) over each fixture's seeded windows (olmo_fixture.window_ids, regenerated from the seed).
Contents, per kind k in {olmo, olmo2}: k_cu_seqlens [B+1] int32 and k_nll [T] (float64 rounded to float32, 0 at the
first position of each window), plus k_config as JSON and k_clipped, the share of q / k / v elements the OLMo clamp
changed.

    python tests/golden/make_olmo_golden.py
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import olmo_fixture as F  # noqa: E402
import olmo_oracle as O  # noqa: E402


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    out = {}
    for kind, cfg in F.CONFIGS.items():
        model = F.hf_model(cfg, dtype=torch.float64)
        windows = F.window_ids(kind)
        nll = [F.hf_token_nll(model, w) for w in windows]
        stats = {}
        for w in windows[:-2]:                   # the clamp's share over the windows up to 129 tokens
            O.hidden_rows(F.seeded_state_dict(cfg), cfg, w, stats=stats)
        clipped = stats["clipped"] / stats["qkv"] if stats else 0.0
        assert kind != "olmo" or clipped >= F.MIN_CLIPPED, clipped
        cu = np.concatenate([[0], np.cumsum([len(w) for w in windows])]).astype(np.int32)
        out.update({f"{kind}_cu_seqlens": cu, f"{kind}_nll": np.concatenate(nll).astype(np.float32), f"{kind}_config": np.array(json.dumps(cfg)),
                    f"{kind}_clipped": np.array(clipped)})
        print(kind, int(cu[-1]), "tokens, mean nll", float(np.concatenate(nll).mean()), "clipped", clipped)
    np.savez_compressed(F.GOLDEN, **out)


if __name__ == "__main__":
    main()
