#!/usr/bin/env python
"""Tiered fp16 Flat index (index.IndexFlatIP(dtype="float16", device_rows=R), DESIGN §4.6): prints one JSON line per
configuration.

    python scripts/bench_flat_tiered.py [--n 20000000] [--nq 1,64,1024,4096] [--steps 3 --warmup 1]

The corpus is synth.Corpus (gmm, d = 768) in fp16, k = 100.  Config "c1_large" builds two indexes of the same n rows:
  * device: R = n (every row in HBM: the all-device search);
  * host:   R = 0 (every row in pinned host memory, streamed through two staging buffers by every search);
and times them alternated (CUDA events around each search) at every --nq batch size.  Per arm: ms per search, QPS, host
GB streamed per search and the effective rate; per batch size the overlap ratio t_host / max(t_device, host_bytes /
memcpy_bw), where memcpy_bw is a plain pinned -> device cudaMemcpy of 1 GB measured in the same run.  Parity: the first
16 queries of both arms against a float64 exhaustive search of the same fp16 rows (oracle/parity.py topk_parity, the
tie-aware comparison of oracle/ann_oracle.py), and tiered vs all-device ids / scores.

Config "c1_beyond_hbm" is the index that cannot be built all-device: --big-n rows (68M) with R = --big-dev (36M), 49 GB
in host memory, at --big-nq.  It is skipped (and says so) when its host tier would exceed half of MemAvailable, or when
--big-n is 0; `--n 0` skips "c1_large", so the big config can run in a process of its own.  Every line records the
card's name and power limit and the host's MemAvailable."""
import argparse
import gc
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np
import torch

from bench_refine import gpu_identity, mem_available, pinned_copy_gbs
from oracle import parity as P
from retrieval_scaling_b200 import index as rsb_index
from retrieval_scaling_b200.synth import Corpus

CHUNK = 1_000_000


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=20_000_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--nq", default="1,64,1024,4096")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--staging-mb", type=int, default=256)
    ap.add_argument("--parity-queries", type=int, default=16)
    ap.add_argument("--big-n", type=int, default=68_000_000)
    ap.add_argument("--big-dev", type=int, default=36_000_000)
    ap.add_argument("--big-nq", default="1024,4096")
    return ap.parse_args()


def build(corpus, n, device_rows, staging_bytes):
    ix = rsb_index.IndexFlatIP(corpus.d, dtype="float16", device_rows=device_rows, staging_bytes=staging_bytes)
    t0 = time.time()
    for c in range(0, (n + CHUNK - 1) // CHUNK):
        rows = min(CHUNK, n - c * CHUNK)
        ix.add(corpus.chunk(c, CHUNK)[:rows].half())
    ix.finalize()
    torch.cuda.synchronize()
    return ix, time.time() - t0


def time_search(ix, q, k):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    ix.search_ids(q, k)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def exact_reference(corpus, n, q, k):
    """float64 exhaustive top-k of q against the fp16 rows (regenerated chunk by chunk on the device)"""
    D = torch.full((q.shape[0], 0), -np.inf, dtype=torch.float64, device=q.device)
    I = torch.zeros((q.shape[0], 0), dtype=torch.int64, device=q.device)
    for c in range(0, (n + CHUNK - 1) // CHUNK):
        rows = min(CHUNK, n - c * CHUNK)
        S = q.double() @ corpus.chunk(c, CHUNK)[:rows].half().double().T
        D = torch.cat([D, S], 1)
        I = torch.cat([I, torch.arange(c * CHUNK, c * CHUNK + rows, device=q.device).expand(q.shape[0], -1)], 1)
        D, j = torch.topk(D, k, dim=1)
        I = torch.gather(I, 1, j)
    return D.float().cpu().numpy(), I.cpu().numpy()


def parity(ix, corpus, n, q, k):
    I, D = (t.cpu().numpy() for t in ix.search_ids(q, k))
    Dr, Ir = exact_reference(corpus, n, q, k)
    return P.topk_parity(D, I, Dr, Ir, rtol=1e-5, atol=2e-5 * float(np.abs(Dr[:, 0]).max())), (I, D)


def arm_stats(ms, nq, host_bytes):
    t = float(np.median(ms))
    out = {"ms": round(t, 3), "qps": round(nq / (t / 1e3), 1)}
    if host_bytes:
        out["host_gb_streamed"] = round(host_bytes / 1e9, 3)
        out["host_gbs_effective"] = round(host_bytes / 1e9 / (t / 1e3), 2)
    return out


def main():
    a = parse()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    ident = {**gpu_identity(dev), "mem_available_gb": round(mem_available() / 1e9, 1)}
    memcpy_gbs = pinned_copy_gbs(dev)
    corpus = Corpus(d=a.d)
    sb = a.staging_mb << 20
    row_bytes = a.d * 2

    # ---- c1_large: all-device vs all-host, alternated
    host_bytes = a.n * row_bytes
    line = {"config": "c1_large", "n": a.n, "d": a.d, "k": a.k, "staging_mb": a.staging_mb, **ident,
            "memcpy_h2d_gbs": round(memcpy_gbs, 2)}
    if a.n <= 0 or host_bytes > mem_available() // 2:
        line["skipped"] = "--n 0" if a.n <= 0 else f"the host tier ({host_bytes / 1e9:.1f} GB) exceeds half of MemAvailable"
        print(json.dumps(line), flush=True)
    else:
        ixd, td = build(corpus, a.n, a.n, sb)
        ixh, th = build(corpus, a.n, 0, sb)
        line.update(build_s={"device": round(td, 1), "host": round(th, 1)}, host_bytes=ixh.host_bytes,
                    device_index_bytes={"device": ixd.index_bytes, "host": ixh.index_bytes})
        qall = corpus.queries(max(int(x) for x in a.nq.split(",")))
        arms = {}
        for nq in (int(x) for x in a.nq.split(",")):
            q = qall[:nq].contiguous()
            ms = {"device": [], "host": []}
            for _ in range(a.warmup):
                time_search(ixd, q, a.k); time_search(ixh, q, a.k)
            for _ in range(a.steps):
                ms["device"].append(time_search(ixd, q, a.k))
                ms["host"].append(time_search(ixh, q, a.k))
            dstat, hstat = arm_stats(ms["device"], nq, 0), arm_stats(ms["host"], nq, host_bytes)
            copy_ms = host_bytes / (memcpy_gbs * 1e9) * 1e3
            arms[nq] = {"device": dstat, "host": hstat, "memcpy_bound_ms": round(copy_ms, 2),
                        "overlap_ratio": round(hstat["ms"] / max(dstat["ms"], copy_ms), 3),
                        "host_over_device": round(hstat["ms"] / dstat["ms"], 3)}
        line["nq"] = arms
        qp = qall[:a.parity_queries].contiguous()
        pd, (Id, Dd) = parity(ixd, corpus, a.n, qp, a.k)
        ph, (Ih, Dh) = parity(ixh, corpus, a.n, qp, a.k)
        same = Id == Ih
        line["parity"] = {"device": pd, "host": ph, "ids_equal_fraction": float(same.mean()),
                          "scores_bit_equal_where_ids_equal": bool(np.array_equal(Dd[same], Dh[same]))}
        print(json.dumps(line), flush=True)
        del ixd, ixh
        gc.collect()
        torch.cuda.empty_cache()

    # ---- c1_beyond_hbm: more rows than one H100 holds in fp16
    line = {"config": "c1_beyond_hbm", "n": a.big_n, "device_rows": a.big_dev, "d": a.d, "k": a.k,
            "staging_mb": a.staging_mb, **ident, "mem_available_gb": round(mem_available() / 1e9, 1),
            "memcpy_h2d_gbs": round(memcpy_gbs, 2)}
    big_host = max(0, a.big_n - a.big_dev) * row_bytes
    if a.big_n <= 0:
        line["skipped"] = "--big-n 0"
    elif big_host > mem_available() // 2:
        line["skipped"] = f"the host tier ({big_host / 1e9:.1f} GB) exceeds half of MemAvailable"
    else:
        ix, tb = build(corpus, a.big_n, a.big_dev, sb)
        line.update(build_s=round(tb, 1), host_bytes=ix.host_bytes, device_index_bytes=ix.index_bytes)
        qall = corpus.queries(max(int(x) for x in a.big_nq.split(",")))
        arms = {}
        for nq in (int(x) for x in a.big_nq.split(",")):
            q = qall[:nq].contiguous()
            for _ in range(a.warmup):
                time_search(ix, q, a.k)
            st = arm_stats([time_search(ix, q, a.k) for _ in range(a.steps)], nq, big_host)
            st["memcpy_bound_ms"] = round(big_host / (memcpy_gbs * 1e9) * 1e3, 2)
            arms[nq] = st
        line["nq"] = arms
        line["parity"], _ = parity(ix, corpus, a.big_n, qall[:a.parity_queries].contiguous(), a.k)
        del ix
        gc.collect()
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
