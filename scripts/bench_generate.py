#!/usr/bin/env python
"""Greedy generation on the GPU: librsb's reader (`_Reader.generate`, rsb_llm_generate) against HF `model.generate` in
bf16 with the lm-eval fork's settings (greedy, max_gen_toks new tokens, left-padded batch), on the same GPU, weights
and prompts.

Seeded weights (HF's own initialisation, made on the device) with the full-depth geometry of Pythia-1B (the reference's
default reader, head_dim 256) and Llama-3-8B (GQA 4:1).  Prompts of --prompt tokens (five shots plus three 256-word
passages are ~1.2k), --new new tokens with no EOS, so every sequence runs every step on both paths.  Per batch size:
  prefill ms    generate(max_new_tokens=1): the prefill and one LM-head pass
  decode ms     (generate(--new) - generate(1)) / (--new - 1), per step
  tokens/s      batch x --new / generate(--new)
  HBM share     bytes one decode step must read (every weight once, the input embedding only at the batch's rows,
                plus each sequence's cached K / V at the step's mean length) over the decode step time, as a share
                of the 3.35 TB/s data-sheet bandwidth
The GPU's name and power limit are read in the same run.  --profile instead takes the per-kernel split of decode steps
with torch.profiler (a run of its own).  One JSON line per configuration to stdout.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GEOMETRY = {
    "pythia-1b": dict(model_type="gpt_neox", num_hidden_layers=16, hidden_size=2048, num_attention_heads=8,
                      intermediate_size=8192, vocab_size=50304, max_position_embeddings=2048, rotary_pct=0.25,
                      rotary_emb_base=10000, layer_norm_eps=1e-5, hidden_act="gelu", use_parallel_residual=True,
                      tie_word_embeddings=False),
    "llama3-8b": dict(model_type="llama", num_hidden_layers=32, hidden_size=4096, num_attention_heads=32,
                      num_key_value_heads=8, intermediate_size=14336, vocab_size=128256, max_position_embeddings=8192,
                      rope_theta=500000.0, rms_norm_eps=1e-5, hidden_act="silu", tie_word_embeddings=False),
}
HBM_BYTES_PER_S = 3.35e12


def gpu_card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def hf_model(geom, seed):
    import transformers
    kw = {k: v for k, v in geom.items() if k != "model_type"}
    cfg = (transformers.GPTNeoXConfig if geom["model_type"] == "gpt_neox" else transformers.LlamaConfig)(**kw)
    cfg._attn_implementation = "sdpa"
    torch.manual_seed(seed)
    with torch.device("cuda"):
        model = transformers.AutoModelForCausalLM.from_config(cfg, torch_dtype=torch.bfloat16).eval()
    model.generation_config.eos_token_id = None
    model.generation_config.pad_token_id = 0
    return model


def ours(geom, hf, dtype):
    from retrieval_scaling_b200 import reader
    cls = reader.B200NeoX if geom["model_type"] == "gpt_neox" else reader.B200Llama
    m = cls(geom, dtype=dtype)
    with torch.no_grad():
        for name, t in hf.state_dict().items():
            m.load_weight(name, t)
    m.require_all_weights("the HF model")
    return m


def step_bytes(geom, hf, B, L, new):
    """Every weight once except the input embedding, of which a step reads its B rows, plus the cached K / V of every
    sequence at the mean decode length."""
    embed = hf.get_input_embeddings().weight.numel() * 2
    weights = sum(p.numel() for p in hf.parameters()) * 2 - embed + B * geom["hidden_size"] * 2
    kv_heads = geom.get("num_key_value_heads", geom["num_attention_heads"])
    head_dim = geom["hidden_size"] // geom["num_attention_heads"]
    per_token = geom["num_hidden_layers"] * 2 * kv_heads * head_dim * 2
    return weights + B * (L + new / 2) * per_token


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def hf_generate(hf, prompts, new):
    x = torch.tensor(prompts, device="cuda")
    with torch.no_grad():
        return hf.generate(x, attention_mask=torch.ones_like(x), do_sample=False, num_beams=1, max_new_tokens=new,
                           min_new_tokens=new)


def run(name, batches, L, new, dtype, with_hf, card):
    geom = dict(GEOMETRY[name])
    hf = hf_model(geom, 1)
    m = ours(geom, hf, dtype)
    g = torch.Generator().manual_seed(2)
    for B in batches:
        prompts = torch.randint(0, geom["vocab_size"], (B, L), generator=g).tolist()
        m.generate(prompts, 2, [])                                   # warm-up of every shape
        t1, _ = timed(lambda: m.generate(prompts, 1, []))
        tn, toks = timed(lambda: m.generate(prompts, new, []))
        assert all(len(t) == new for t in toks)
        dec = (tn - t1) / (new - 1)
        sb = step_bytes(geom, hf, B, L, new)
        res = dict(model=name, dtype=str(dtype).split(".")[-1], batch=B, prompt=L, new=new, prefill_ms=1e3 * t1,
                   decode_ms_per_step=1e3 * dec, tokens_per_s=B * new / tn, step_gb=sb / 1e9,
                   hbm_share=sb / dec / HBM_BYTES_PER_S, gpu=card)
        if with_hf:
            hf_generate(hf, prompts[:1], 2)
            h1, _ = timed(lambda: hf_generate(hf, prompts, 1))
            hn, _ = timed(lambda: hf_generate(hf, prompts, new))
            res.update(hf_prefill_ms=1e3 * h1, hf_decode_ms_per_step=1e3 * (hn - h1) / (new - 1),
                       hf_tokens_per_s=B * new / hn, speedup=hn / tn)
        print(json.dumps(res), flush=True)
    del m, hf
    torch.cuda.empty_cache()


def profile(name, B, L, dtype):
    from torch.profiler import ProfilerActivity
    geom = dict(GEOMETRY[name])
    hf = hf_model(geom, 1)
    m = ours(geom, hf, dtype)
    prompts = torch.randint(0, geom["vocab_size"], (B, L), generator=torch.Generator().manual_seed(2)).tolist()
    m.generate(prompts, 2, [])
    steps = 16
    with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.generate(prompts, 1, [])
    pre = {e.key: e.device_time_total for e in prof.key_averages()}
    with torch.profiler.profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.generate(prompts, 1 + steps, [])
    rows = []
    for e in prof.key_averages():
        us = (e.device_time_total - pre.get(e.key, 0.0)) / steps
        if us > 0:
            rows.append((us, e.key))
    rows.sort(reverse=True)
    total = sum(r[0] for r in rows)
    print(json.dumps(dict(model=name, batch=B, prompt=L, decode_step_kernel_us=total, gpu=gpu_card())))
    for us, key in rows[:15]:
        print(f"{us:10.1f} us/step  {100 * us / total:5.1f} %  {key[:110]}")


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--models", default="pythia-1b,llama3-8b")
    ap.add_argument("--batches", default="1,16,64")
    ap.add_argument("--prompt", type=int, default=1200)
    ap.add_argument("--new", type=int, default=256)
    ap.add_argument("--dtype", default="bfloat16", choices=["float16", "bfloat16"])
    ap.add_argument("--no-hf", action="store_true")
    ap.add_argument("--profile", action="store_true", help="per-kernel split of decode steps (first model and batch)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_generate.py measures on a CUDA device; there is none")
    dtype = getattr(torch, a.dtype)
    models, batches = a.models.split(","), [int(b) for b in a.batches.split(",")]
    if a.profile:
        profile(models[0], batches[0], a.prompt, dtype)
        return
    card = gpu_card()
    print(f"# {card}", flush=True)
    for name in models:
        run(name, batches, a.prompt, a.new, dtype, not a.no_hf, card)


if __name__ == "__main__":
    main()
