#!/usr/bin/env python
"""Reader-LM perplexity forward on the GPU: librsb's Llama reader (rsb_llm_nll) against HF LlamaForCausalLM in bf16 with
sdpa attention, the reference's reader path minus flash-attn-2 (src/evaluate_perplexity.py:98-134), on the same GPU
and the same windows.

Seeded weights with the full-depth geometry of Llama-2-7B (MHA, vocab 32000) and Llama-3-8B (GQA 4:1, vocab 128256),
or of Pythia-1B (head_dim 256), Pythia-1.4B and Pythia-6.9B (GPT-NeoX: librsb's B200NeoX against HF GPTNeoXForCausalLM),
or of OLMo-1B (tied head), OLMo-7B-0424 (clip_qkv 8) and OLMo-2-7B (librsb's B200Olmo against HF OlmoForCausalLM /
Olmo2ForCausalLM), generated on the device.  --windows windows of --context context tokens (retrieved documents + query, label -100)
followed by --answer answer tokens (the labels), as the reference builds them with concate_k documents in front of a
1024-token evaluation chunk.  Timed with CUDA events after --warmup passes, --repeats passes per model, the median
reported.  Per-kernel times come from a separate torch.profiler pass.  Achieved TFLOP/s counts the model's FLOPs with
the LM head on the label rows only (what rsb_llm_nll computes), for both paths, against the 989 TFLOP/s dense
fp16 / bf16 data-sheet peak of the H100 SXM.  The GPU's name and power limit are read in the same run.
One JSON line per model and a final JSON line to stdout (and to --out).
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GEOMETRY = {
    "llama2-7b": dict(model_type="llama", num_hidden_layers=32, hidden_size=4096, num_attention_heads=32,
                      num_key_value_heads=32, intermediate_size=11008, vocab_size=32000, max_position_embeddings=4096,
                      rope_theta=10000.0, rms_norm_eps=1e-5, hidden_act="silu", tie_word_embeddings=False),
    "llama3-8b": dict(model_type="llama", num_hidden_layers=32, hidden_size=4096, num_attention_heads=32,
                      num_key_value_heads=8, intermediate_size=14336, vocab_size=128256, max_position_embeddings=8192,
                      rope_theta=500000.0, rms_norm_eps=1e-5, hidden_act="silu", tie_word_embeddings=False),
}
_PYTHIA = dict(model_type="gpt_neox", max_position_embeddings=2048, rotary_pct=0.25, rotary_emb_base=10000,
               layer_norm_eps=1e-5, hidden_act="gelu", use_parallel_residual=True, tie_word_embeddings=False)
GEOMETRY.update({
    "pythia-1b": dict(_PYTHIA, num_hidden_layers=16, hidden_size=2048, num_attention_heads=8, intermediate_size=8192,
                      vocab_size=50304),
    "pythia-1.4b": dict(_PYTHIA, num_hidden_layers=24, hidden_size=2048, num_attention_heads=16, intermediate_size=8192,
                        vocab_size=50304),
    "pythia-6.9b": dict(_PYTHIA, num_hidden_layers=32, hidden_size=4096, num_attention_heads=32,
                        intermediate_size=16384, vocab_size=50432),
})
_OLMO = dict(hidden_act="silu", attention_bias=False, rope_theta=10000.0, max_position_embeddings=2048,
             tie_word_embeddings=False)
GEOMETRY.update({
    "olmo-1b": dict(_OLMO, model_type="olmo", num_hidden_layers=16, hidden_size=2048, num_attention_heads=16,
                    num_key_value_heads=16, intermediate_size=8192, vocab_size=50304, clip_qkv=None,
                    tie_word_embeddings=True),
    "olmo-7b": dict(_OLMO, model_type="olmo", num_hidden_layers=32, hidden_size=4096, num_attention_heads=32,
                    num_key_value_heads=32, intermediate_size=11008, vocab_size=50304, clip_qkv=8.0,
                    max_position_embeddings=4096),
    "olmo2-7b": dict(_OLMO, model_type="olmo2", num_hidden_layers=32, hidden_size=4096, num_attention_heads=32,
                     num_key_value_heads=32, intermediate_size=11008, vocab_size=100352, rope_theta=500000.0,
                     rms_norm_eps=1e-6, max_position_embeddings=4096),
})
PEAK_TFLOPS = 989.0


def neox(cfg):
    return cfg["model_type"] == "gpt_neox"


def head_dim(cfg):
    return cfg["hidden_size"] // cfg["num_attention_heads"]


def kv_heads(cfg):
    return cfg.get("num_key_value_heads", cfg["num_attention_heads"])


def neox_weights(cfg, seed=0):
    """GPTNeoXForCausalLM (name, fp16 tensor on the device) in HF order, regenerated from the seed for each path."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    H, I, V = cfg["hidden_size"], cfg["intermediate_size"], cfg["vocab_size"]

    def n(*shape, std):
        return torch.randn(*shape, generator=g, device="cuda", dtype=torch.float16) * std

    yield "gpt_neox.embed_in.weight", n(V, H, std=1.0)
    for i in range(cfg["num_hidden_layers"]):
        p = f"gpt_neox.layers.{i}."
        for ln in ("input_layernorm", "post_attention_layernorm"):
            yield p + ln + ".weight", 1.0 + n(H, std=0.05)
            yield p + ln + ".bias", n(H, std=0.05)
        for name, shape, fan in (("attention.query_key_value", (3 * H, H), H), ("attention.dense", (H, H), H),
                                 ("mlp.dense_h_to_4h", (I, H), H), ("mlp.dense_4h_to_h", (H, I), I)):
            yield p + name + ".weight", n(*shape, std=fan ** -0.5)
            yield p + name + ".bias", n(shape[0], std=0.02)
    yield "gpt_neox.final_layer_norm.weight", 1.0 + n(H, std=0.05)
    yield "gpt_neox.final_layer_norm.bias", n(H, std=0.05)
    yield "embed_out.weight", n(V, H, std=2.0 * H ** -0.5)


def weights(cfg, seed=0):
    """(name, fp16 tensor on the device) in HF order, regenerated from the seed for each path.  Llama, OLMo (no norm
    weights) and OLMo-2 (post-norms and QK-norms) share the projections."""
    if neox(cfg):
        yield from neox_weights(cfg, seed)
        return
    g = torch.Generator(device="cuda").manual_seed(seed)
    H, I, V = cfg["hidden_size"], cfg["intermediate_size"], cfg["vocab_size"]
    KV = cfg["num_key_value_heads"] * 128
    mt, tied = cfg["model_type"], cfg["tie_word_embeddings"]

    def n(*shape, std):
        return torch.randn(*shape, generator=g, device="cuda", dtype=torch.float16) * std

    yield "model.embed_tokens.weight", n(V, H, std=2.0 * H ** -0.5 if tied else 1.0)
    for i in range(cfg["num_hidden_layers"]):
        p = f"model.layers.{i}."
        for name, shape, fan in (("self_attn.q_proj", (H, H), H), ("self_attn.k_proj", (KV, H), H),
                                 ("self_attn.v_proj", (KV, H), H), ("self_attn.o_proj", (H, H), H),
                                 ("mlp.gate_proj", (I, H), H), ("mlp.up_proj", (I, H), H), ("mlp.down_proj", (H, I), I)):
            yield p + name + ".weight", n(*shape, std=fan ** -0.5)
        norms = {"llama": (("input_layernorm", H), ("post_attention_layernorm", H)), "olmo": (),
                 "olmo2": (("self_attn.q_norm", H), ("self_attn.k_norm", KV), ("post_attention_layernorm", H),
                           ("post_feedforward_layernorm", H))}[mt]
        for name, width in norms:
            yield p + name + ".weight", 1.0 + n(width, std=0.05)
    if mt != "olmo":
        yield "model.norm.weight", 1.0 + n(H, std=0.05)
    if not tied:
        yield "lm_head.weight", n(V, H, std=2.0 * H ** -0.5)


def windows(cfg, n, context, answer, seed=1):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, cfg["vocab_size"], (n, context + answer), generator=g)
    labels = ids.clone()
    labels[:, :context] = -100
    return ids, labels


def model_flops(cfg, context, answer):
    """FLOPs of one window: linear layers on every token, causal attention, LM head on the label rows."""
    H, I, L = cfg["hidden_size"], cfg["intermediate_size"], cfg["num_hidden_layers"]
    KV = kv_heads(cfg) * head_dim(cfg)
    S = context + answer
    mlp = (2 if neox(cfg) else 3) * H * I            # GELU MLP: two matrices; SwiGLU: three
    lin = 2 * S * L * (H * (H + 2 * KV) + H * H + mlp)
    att = 2 * 2 * L * cfg["num_attention_heads"] * head_dim(cfg) * S * (S + 1) // 2
    head = 2 * answer * H * cfg["vocab_size"]
    return lin + att + head


def timed(fn, warmup, repeats):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return ms


def kernel_table(fn, n_windows):
    """Device time per kernel name, ms per window, from one profiled pass."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    tab = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = getattr(ev, "cuda_time_total", 0)
        if t > 0 and ev.key not in ("cudaDeviceSynchronize",):
            tab[ev.key] = round(t / 1000.0 / n_windows, 4)
    return dict(sorted(tab.items(), key=lambda kv: -kv[1])[:16])


def bench_rsb(cfg, ids, labels, args, dtype="float16"):
    from retrieval_scaling_b200.reader import READERS
    m = READERS[cfg["model_type"]][1](cfg, dtype=dtype)
    for name, w in weights(cfg):
        m.load_weight(name, w)
        del w
    m.require_all_weights("seeded weights")
    ids_l, lab_l = ids.tolist(), labels.tolist()
    run = lambda: m.nll(ids_l, lab_l, max_tokens=args.token_budget)   # noqa: E731
    ms = timed(run, args.warmup, args.repeats)
    kernels = kernel_table(run, len(ids_l))
    losses = m.loss(ids_l[:4], lab_l[:4])
    del m
    gc.collect()
    torch.cuda.empty_cache()
    return ms, kernels, losses


def bench_hf(cfg, ids, labels, args):
    import transformers
    kw = {k: v for k, v in cfg.items() if k != "model_type"}
    conf, cls = {"llama": (transformers.LlamaConfig, transformers.LlamaForCausalLM),
                 "gpt_neox": (transformers.GPTNeoXConfig, transformers.GPTNeoXForCausalLM),
                 "olmo": (transformers.OlmoConfig, transformers.OlmoForCausalLM),
                 "olmo2": (transformers.Olmo2Config, transformers.Olmo2ForCausalLM)}[cfg["model_type"]]
    hc = conf(**kw)
    hc._attn_implementation = "sdpa"
    with torch.device("meta"):
        lm = cls(hc)
    lm = lm.to_empty(device="cuda").to(torch.bfloat16).eval()
    lm.tie_weights()                             # to_empty gives a tied head storage of its own: share it again
    params = dict(lm.named_parameters())
    with torch.no_grad():
        for name, w in weights(cfg):
            params[name].copy_(w)
            del w
        for mod in lm.modules():                 # buffers are not parameters: recompute RoPE's inv_freq (fp32)
            if hasattr(mod, "inv_freq") and hasattr(mod, "compute_default_rope_parameters"):
                mod.inv_freq = mod.compute_default_rope_parameters(mod.config, device="cuda")[0]
    dev_ids, dev_lab = ids.cuda(), labels.cuda()

    def run():                                   # the reference's loop: one window per forward
        out = []
        with torch.no_grad():
            for i in range(dev_ids.shape[0]):
                out.append(lm(dev_ids[i:i + 1], labels=dev_lab[i:i + 1]).loss)
        return out
    ms = timed(run, args.warmup, args.repeats)
    losses = [float(x) for x in run()[:4]]
    del lm, params
    gc.collect()
    torch.cuda.empty_cache()
    return ms, losses


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="llama2-7b,llama3-8b")
    ap.add_argument("--windows", type=int, default=32)
    ap.add_argument("--context", type=int, default=768, help="retrieved documents + query tokens (label -100)")
    ap.add_argument("--answer", type=int, default=1024, help="evaluation tokens (the labels)")
    ap.add_argument("--token-budget", type=int, default=16384)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--dtype", default="float16",
                    help="librsb reader dtypes, comma-separated: float16 (reported as 'rsb') and / or bfloat16 "
                         "('rsb_bf16'); every run is timed against the same HF bf16 sdpa arm")
    ap.add_argument("--no-hf", action="store_true")
    ap.add_argument("--out", default=None, help="also write the result as JSON here")
    args = ap.parse_args()
    dtypes = args.dtype.split(",")
    if not dtypes or any(d not in ("float16", "bfloat16") for d in dtypes):
        raise SystemExit(f"--dtype {args.dtype!r}: float16 and / or bfloat16")
    if not torch.cuda.is_available():
        raise SystemExit("bench_reader.py measures the GPU path: no CUDA device")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    result = {"gpu": smi, "windows": args.windows, "context": args.context, "answer": args.answer, "models": {}}
    for name in args.models.split(","):
        cfg = GEOMETRY[name]
        ids, labels = windows(cfg, args.windows, args.context, args.answer)
        tokens = ids.numel()
        flops = model_flops(cfg, args.context, args.answer) * args.windows
        r, meds = {}, {}
        for dt in dtypes:
            ms, kernels, l_rsb = bench_rsb(cfg, ids, labels, args, dt)
            med = meds[dt] = statistics.median(ms)
            r["rsb" if dt == "float16" else "rsb_bf16"] = {
                "ms_runs": [round(x, 2) for x in ms], "ms_per_sample": round(med / args.windows, 3),
                "tokens_per_s": round(tokens / med * 1e3), "tflops": round(flops / med / 1e9, 1),
                "share_of_peak": round(flops / med / 1e9 / PEAK_TFLOPS, 3), "kernels_ms_per_sample": kernels,
                "loss_first_windows": [round(x, 4) for x in l_rsb]}
        if not args.no_hf:
            ms_h, l_hf = bench_hf(cfg, ids, labels, args)
            med_h = statistics.median(ms_h)
            r["hf_bf16_sdpa"] = {"ms_runs": [round(x, 2) for x in ms_h], "ms_per_sample": round(med_h / args.windows, 3),
                                 "tokens_per_s": round(tokens / med_h * 1e3), "tflops": round(flops / med_h / 1e9, 1),
                                 "loss_first_windows": [round(x, 4) for x in l_hf]}
            for dt, key in (("float16", "speedup"), ("bfloat16", "speedup_bf16")):
                if dt in meds:
                    r[key] = round(med_h / meds[dt], 2)
        result["models"][name] = r
        print(json.dumps({name: r}), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
