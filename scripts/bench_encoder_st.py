"""T5 encoder (GTR-T5 geometry: 12 layers, d_model 768, 12 heads of 64, d_ff 3072, with the sentence-transformers
Dense + Normalize head) and RoBERTa-base (DRAGON-RoBERTa geometry: 12 layers, vocabulary 50265, 514 positions, CLS
row) against the BERT-base forward (Contriever, mean pooling), in one process, the three alternated.  RoBERTa runs on
the BERT arm's token streams themselves (ids 3 .. 30521, valid and never the pad id 1 in its vocabulary).

Workloads (seeded weights, random token ids; only the lengths matter to the kernels):
  q64 / q2048   10 000 queries whose token counts are drawn from tests/golden/nq_open_token_lengths.npy (NQ-open
                questions under the BERT tokenizer), encoded in forwards of 64 (the reference's per_gpu_batch_size)
                and of 2048 sequences (the query encoder's `encode_group`)
  p256 / p512   512 passages of 256 and of 512 tokens (the passage side at its reference batch size)

Per workload: median ms over `--steps` alternated repetitions of the whole workload, and TFLOP/s of its Linear-layer
work: 169.9 MFLOP per token for all three models (2 x (4 x 768^2 + 2 x 768 x 3072) x 12 layers; T5 only drops the biases).
Attention and the head are not counted.  The card's name and power limit are read in the same run.

    python scripts/bench_encoder_st.py --steps 5 --warmup 2 [--out results.json]
    RSB_BERT_PROFILE=1 python scripts/bench_encoder_st.py --profile     # per-kernel split, a separate run
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

LINEAR_FLOP_PER_TOKEN = 2 * (4 * 768 * 768 + 2 * 768 * 3072) * 12      # 169.9 M


def gpu_identity(device) -> dict:
    out = {"gpu": torch.cuda.get_device_name(device), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", f"--id={device.index or 0}", "--query-gpu=power.limit",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return out


def workloads(rng):
    nq = np.load(os.path.join(ROOT, "tests", "golden", "nq_open_token_lengths.npy")).astype(np.int64)
    qlens = rng.choice(nq, 10_000)
    return {"q64": (qlens, 64), "q2048": (qlens, 2048), "p256": (np.full(512, 256), 512), "p512": (np.full(512, 512), 512)}


def batches(lens, group, vocab, rng, device):
    """Pre-built un-padded forwards: (ids [T] int32, cu_seqlens [B+1] int32, max_seqlen, T)."""
    out = []
    for i in range(0, len(lens), group):
        L = lens[i:i + group]
        cu = np.zeros(len(L) + 1, np.int32)
        cu[1:] = np.cumsum(L)
        ids = torch.from_numpy(rng.integers(3, vocab, int(cu[-1])).astype(np.int32)).to(device)
        out.append((ids, torch.from_numpy(cu).to(device), int(L.max()), int(cu[-1])))
    return out


def run(model, fwd):
    for ids, cu, mx, T in fwd:
        model.forward_varlen(ids, cu, mx, total_tokens=T)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", default="", help="comma-separated workload names (default: all)")
    ap.add_argument("--profile", action="store_true", help="one forward per workload and model (RSB_BERT_PROFILE=1)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    from retrieval_scaling_b200.encoder import (BERT_BASE, ROBERTA_BASE, T5_BASE, B200Contriever, B200Roberta,
                                                B200T5Encoder, random_state_dict, random_t5_state_dict)
    t5 = B200T5Encoder(T5_BASE, "average", dense=True, normalize=True)
    t5.load_state_dict(random_t5_state_dict(T5_BASE, 0))
    t5.require_all_weights("bench")
    bert = B200Contriever(BERT_BASE, "average")
    bert.load_state_dict(random_state_dict(BERT_BASE, 0))
    roberta = B200Roberta(ROBERTA_BASE, "cls")
    roberta.load_state_dict(random_state_dict(ROBERTA_BASE, 0))
    roberta.require_all_weights("bench")
    models = {"t5": t5, "bert": bert, "roberta": roberta}
    vocab = {"t5": T5_BASE["vocab_size"], "bert": BERT_BASE["vocab_size"]}
    ident = gpu_identity(dev)
    rng = np.random.default_rng(0)
    results = []
    for name, (lens, group) in workloads(rng).items():
        if a.only and name not in a.only.split(","):
            continue
        seed = int(rng.integers(1 << 30))
        fwd = {m: batches(lens, group, vocab[m], np.random.default_rng(seed), dev) for m in vocab}
        fwd["roberta"] = fwd["bert"]
        tokens = int(lens.sum())
        if a.profile:
            for m in models:
                print(f"# {name} {m}", file=sys.stderr, flush=True)
                run(models[m], fwd[m][:1])
                torch.cuda.synchronize()
            continue
        for _ in range(a.warmup):
            for m in models:
                run(models[m], fwd[m])
        torch.cuda.synchronize()
        ms = {m: [] for m in models}
        for _ in range(a.steps):
            for m in models:                                # alternated: both see the same clock and neighbours
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run(models[m], fwd[m])
                e1.record()
                e1.synchronize()
                ms[m].append(e0.elapsed_time(e1))
        line = {"workload": name, "sequences": len(lens), "batch": group, "tokens": tokens, **ident}
        for m in models:
            med = statistics.median(ms[m])
            line[m] = {"ms": round(med, 3), "ms_min": round(min(ms[m]), 3), "ms_max": round(max(ms[m]), 3),
                       "linear_tflops": round(LINEAR_FLOP_PER_TOKEN * tokens / (med * 1e-3) / 1e12, 1)}
        line["t5_over_bert"] = round(line["t5"]["ms"] / line["bert"]["ms"], 3)
        line["roberta_over_bert"] = round(line["roberta"]["ms"] / line["bert"]["ms"], 3)
        print(json.dumps(line), flush=True)
        results.append(line)
    if a.out and results:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
