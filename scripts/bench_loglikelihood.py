#!/usr/bin/env python
"""Multiple-choice scoring on the GPU: librsb's reader (`_Reader.loglikelihood`, rsb_llm_loglikelihood) against HF
transformers running the lm-eval fork's procedure (HFLM._loglikelihood_tokens: a right-padded batch of windows, full
logits, log_softmax, the four choices' tokens gathered from the last row) on the same GPU, weights and windows.

Seeded weights as bench_generate.py makes them (HF's own initialisation on the device), at the full-depth geometry of
Pythia-1B and Llama-3-8B, in bf16.  MMLU-shaped questions: one context of --prompt tokens (five shots plus k retrieved
passages come to about 1 500) and four one-token choices, so each question is one window on both paths.  Per model:
  questions/s        --questions / the time of one loglikelihood call over all of them (a device synchronise ends it)
  prefill tokens/s   questions x --prompt / that time
  agree              share of questions whose argmax choice is the same on both paths
The GPU's name and power limit are read in the same run.  One JSON line per model to stdout.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from bench_generate import GEOMETRY, gpu_card, hf_model, ours, timed  # noqa: E402


def hf_loglikelihood(hf, ctxs, letters, batch):
    """The fork's procedure: one window per question (its group_by="contexts" cache shares a context's logits among
    one-token continuations), right-padded into batches of `batch`, log_softmax of the full logits, the four choices'
    log-probabilities gathered from the window's last row.  [questions, 4]."""
    out = []
    with torch.no_grad():
        for i in range(0, len(ctxs), batch):
            chunk = ctxs[i:i + batch]
            n = max(len(x) for x in chunk)
            x = torch.tensor([c + [0] * (n - len(c)) for c in chunk], device="cuda")
            lp = torch.log_softmax(hf(x).logits, dim=-1)
            for b, c in enumerate(chunk):
                out.append(lp[b, len(c) - 1, letters].float().cpu().numpy())
    return np.stack(out)


def run(name, n_q, L, dtype, hf_batch, card):
    geom = dict(GEOMETRY[name])
    hf = hf_model(geom, 1)
    m = ours(geom, hf, dtype)
    g = torch.Generator().manual_seed(3)
    ctxs = torch.randint(0, geom["vocab_size"], (n_q, L), generator=g).tolist()
    letters = torch.randint(0, geom["vocab_size"], (4,), generator=g).tolist()   # " A" .. " D"
    reqs = [(c, [t]) for c in ctxs for t in letters]
    ml = geom["max_position_embeddings"]
    m.loglikelihood(reqs[:8], ml)                                   # warm-up
    t, res = timed(lambda: m.loglikelihood(reqs, ml))
    ours_pred = np.array([r[0] for r in res]).reshape(n_q, 4).argmax(1)
    out = dict(model=name, dtype=str(dtype).split(".")[-1], questions=n_q, prompt=L, seconds=t,
               questions_per_s=n_q / t, prefill_tokens_per_s=n_q * L / t, gpu=card)
    hf_loglikelihood(hf, ctxs[:hf_batch], letters, hf_batch)
    th, hres = timed(lambda: hf_loglikelihood(hf, ctxs, letters, hf_batch))
    hf_pred = hres.argmax(1)
    out.update(hf_batch=hf_batch, hf_questions_per_s=n_q / th, hf_prefill_tokens_per_s=n_q * L / th,
               speedup=th / t, agree=float((ours_pred == hf_pred).mean()))
    print(json.dumps(out), flush=True)
    del m, hf
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--models", default="pythia-1b,llama3-8b")
    ap.add_argument("--questions", type=int, default=256)
    ap.add_argument("--prompt", type=int, default=1500)
    ap.add_argument("--hf-batch", type=int, default=8, help="HF windows per forward (the harness's --batch_size)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_loglikelihood.py measures on a CUDA device; there is none")
    card = gpu_card()
    print(f"# {card}", flush=True)
    for name in a.models.split(","):
        run(name, a.questions, a.prompt, torch.bfloat16, a.hf_batch, card)


if __name__ == "__main__":
    main()
