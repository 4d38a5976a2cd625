"""Times the IVF coarse stage (rsb_coarse: query split, fp16 hi/lo fused scorer, select_cands, exact_rows, refine_exact)
at bench.py's geometry: nlist 16384, d 768, nprobe 32, for nq in {1, 1250, 10000} (1250 = the per-GPU share of 10k
queries at 8 GPUs).

    python scripts/bench_coarse.py [--steps 20] [--warmup 5] [--out DIR]

Stage time: CUDA events around `steps` back-to-back calls.  Per-kernel split: torch.profiler in a separate run (CUDA
activities), kernel time summed per kernel name.  For the GEMM it also prints the achieved TFLOP/s of fp16 tensor
work (3 products) against the 989 TFLOP/s dense fp16 data-sheet figure, and the operand bytes the tile schedule
implies (2-byte hi + lo operands): DRAM (each band of query tiles once, the centroid operand once per band) and
L2 -> SM (every tile loads its hi + lo query and centroid tiles)."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import retrieval_scaling_b200 as r  # noqa: E402

F16_PEAK = 989e12
KERNELS = ("split_f16_kernel", "gemm_ip_tc_kernel", "select_cands_kernel", "exact_rows_kernel", "refine_exact_kernel")


def schedule_bytes(nq, nlist, d, l2_bytes):
    """Operand bytes of one fused pass under the kernel's tile order (tile_band in rsb_tf32.cu)."""
    tiles_m, tiles_n = -(-nq // 128), -(-nlist // 128)
    a_tile = 128 * d * 2 * 2                                  # fp16 hi + lo
    band = max(1, min(l2_bytes // 3 // a_tile, tiles_m))
    bands = -(-tiles_m // band)
    dram = nq * d * 4 + bands * nlist * d * 4
    l2_to_sm = tiles_m * tiles_n * 2 * a_tile
    return band, dram, l2_to_sm


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--nlist", type=int, default=16384)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--nprobe", type=int, default=32)
    ap.add_argument("--nq", type=int, nargs="+", default=[1, 1250, 10000])
    ap.add_argument("--out", default=None, help="directory for the profiler trace (none written if unset)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_coarse.py needs a CUDA device")
    props = torch.cuda.get_device_properties(0)
    l2 = props.L2_cache_size
    rng = np.random.default_rng(0)
    cent = rng.standard_normal((a.nlist, a.d)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    ivf = r.IndexIVFFlat(a.d, a.nlist)
    ivf.set_centroids(cent)
    qs = torch.from_numpy(rng.standard_normal((max(a.nq), a.d)).astype(np.float32)).cuda()
    out = {"gpu": props.name, "l2_bytes": l2, "nlist": a.nlist, "d": a.d, "nprobe": a.nprobe, "runs": []}
    for nq in a.nq:
        q = qs[:nq].contiguous()
        for _ in range(a.warmup):
            ivf.coarse(q, a.nprobe)
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(a.steps):
            ivf.coarse(q, a.nprobe)
        t1.record()
        torch.cuda.synchronize()
        stage_ms = t0.elapsed_time(t1) / a.steps
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.steps):
                ivf.coarse(q, a.nprobe)
            torch.cuda.synchronize()
        split = {}
        for ev in prof.key_averages():
            name = next((k for k in KERNELS if k in ev.key), None)
            if name:
                split[name] = split.get(name, 0.0) + ev.device_time_total / 1e3 / a.steps   # ms per call
        if a.out:
            os.makedirs(a.out, exist_ok=True)
            prof.export_chrome_trace(os.path.join(a.out, f"coarse_nq{nq}.pt.trace.json"))
        band, dram, l2sm = schedule_bytes(nq, a.nlist, a.d, l2)
        gemm_ms = split.get("gemm_ip_tc_kernel", float("nan"))
        flop = 3 * 2 * nq * a.nlist * a.d
        row = {"nq": nq, "stage_ms": round(stage_ms, 4), "kernel_ms": {k: round(v, 4) for k, v in split.items()},
               "gemm_tflops": round(flop / (gemm_ms * 1e-3) / 1e12, 1), "gemm_share_of_f16_peak": round(flop / F16_PEAK / (gemm_ms * 1e-3), 3),
               "band_query_tiles": band, "dram_operand_mb": round(dram / 1e6, 1), "l2_to_sm_operand_gb": round(l2sm / 1e9, 2)}
        out["runs"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
