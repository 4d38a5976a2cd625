"""Writes tests/golden/neox_golden.npz: the fp64 per-token NLL of transformers' GPTNeoXForCausalLM (run in float64 on
the CPU) over the fixture's seeded windows (neox_fixture.LENGTHS).  Contents: ids [T] int32, cu_seqlens [B+1] int32 and
nll [T] float64 (0 at the first position of each window), plus the config as JSON.

    python tests/golden/make_neox_golden.py
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import neox_fixture as F  # noqa: E402


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    model = F.hf_model(dtype=torch.float64)
    windows = F.window_ids()
    nll = [F.hf_token_nll(model, w) for w in windows]
    cu = np.concatenate([[0], np.cumsum([len(w) for w in windows])]).astype(np.int32)
    np.savez_compressed(F.GOLDEN, ids=np.concatenate(windows).astype(np.int32), cu_seqlens=cu,
                        nll=np.concatenate(nll), config=np.array(json.dumps(F.CONFIG)))
    print(F.GOLDEN, int(cu[-1]), "tokens, mean nll", float(np.concatenate(nll).mean()))


if __name__ == "__main__":
    main()
