"""Tiered IVF-Flat / IVF-SQ8 (list_device_rows) against the all-device index on C2-shaped data.

Arms, alternated per repetition: all-device, R = 0 (every list in host memory) and R = ntotal / 2, at nq in {1, 64,
2048}, for fp16 rows and SQ8 codes with residuals.  Reports ms and QPS, the host bytes a search copies (computed here
from the coarse lists and the list sizes: each probed host list once per query batch), a pinned-memcpy rate measured in
the same run, the overlap ratio t / max(t_all_device, host_bytes / memcpy_rate), and parity (tiered vs all-device on
256 queries: equal ids and scores).  The card name and power limit are printed with the numbers.

    python scripts/bench_ivf_tiered.py [--n 10000000] [--d 768] [--nlist 4096] [--nprobe 64] [--k 100] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import retrieval_scaling_b200 as rsb  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return out
    except Exception as e:  # pragma: no cover
        return f"unknown ({e})"


def memcpy_rate(nbytes=1 << 30, reps=5):
    src = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
    dst = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    dst.copy_(src, non_blocking=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        dst.copy_(src, non_blocking=True)
    torch.cuda.synchronize()
    return nbytes * reps / (time.perf_counter() - t0)


def gmm(n, d, cent, rng_seed, chunk=1 << 20):
    """fp16 rows: centre + noise, generated on the device a chunk at a time."""
    g = torch.Generator(device="cuda").manual_seed(rng_seed)
    out = torch.empty((n, d), dtype=torch.float16)
    for a in range(0, n, chunk):
        m = min(chunk, n - a)
        lab = torch.randint(0, cent.shape[0], (m,), device="cuda", generator=g)
        x = cent[lab] + 0.3 * torch.randn((m, d), device="cuda", generator=g)
        out[a:a + m] = (x / x.norm(dim=1, keepdim=True)).half().cpu()
    return out


def build(kind, d, nlist, cent, sq, rows, lists, R=None, step=1 << 20):
    tier = {} if R is None else {"list_device_rows": R}
    if kind == "sq8":
        ix = rsb.IndexIVFScalarQuantizer(d, nlist, by_residual=True, **tier)
        ix.set_centroids(cent)
        ix.sq_params = sq
    else:
        ix = rsb.IndexIVFFlat(d, nlist, dtype="float16", **tier)
        ix.set_centroids(cent)
    if R is not None:
        ix.reserve_lists(np.bincount(lists, minlength=nlist))
    for a in range(0, rows.shape[0], step):
        ix.add_preassigned(rows[a:a + step], lists[a:a + step])
    ix.finalize()
    return ix


def timed(ix, q, k, nprobe, reps):
    ix.search_ids(q, k, nprobe)
    torch.cuda.synchronize()
    t = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ix.search_ids(q, k, nprobe)
        e1.record()
        torch.cuda.synchronize()
        t.append(e0.elapsed_time(e1))
    return float(np.median(t))


def host_bytes_per_search(lists_probed, sizes, l_dev, rb, qb=16384):
    """Bytes of the probed host lists, each copied once per query batch of qb queries."""
    total = 0
    for a in range(0, lists_probed.shape[0], qb):
        u = np.unique(lists_probed[a:a + qb])
        u = u[(u >= l_dev)]
        total += int(sizes[u].sum()) * rb
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--nlist", type=int, default=4096)
    ap.add_argument("--nprobe", type=int, default=64)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--kinds", default="float16,sq8")
    ap.add_argument("--nqs", default="1,64,2048")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    print(json.dumps({"card": card(), "n": a.n, "d": a.d, "nlist": a.nlist, "nprobe": a.nprobe, "k": a.k}), flush=True)
    rate = memcpy_rate()
    print(json.dumps({"pinned_memcpy_GBps": rate / 1e9}), flush=True)
    g = torch.Generator(device="cuda").manual_seed(0)
    cent = torch.randn((a.nlist, a.d), device="cuda", generator=g)
    cent = cent / cent.norm(dim=1, keepdim=True)
    t0 = time.perf_counter()
    rows = gmm(a.n, a.d, cent, 1)
    qs = gmm(max(int(x) for x in a.nqs.split(",")), a.d, cent, 2).float().cuda()
    print(json.dumps({"data_s": time.perf_counter() - t0}), flush=True)
    probe = rsb.IndexIVFFlat(a.d, a.nlist, dtype="float16")
    probe.set_centroids(cent)
    lists = np.concatenate([probe.assign(rows[i:i + (1 << 20)]).cpu().numpy() for i in range(0, a.n, 1 << 20)])
    sizes = np.bincount(lists, minlength=a.nlist)
    off = np.concatenate([[0], np.cumsum(sizes)])
    for kind in a.kinds.split(","):
        sq = None
        if kind == "sq8":
            tr = rsb.IndexIVFScalarQuantizer(a.d, a.nlist, by_residual=True)
            tr.set_centroids(cent)
            tr.train_sq(rows[:1_000_000])
            sq = torch.stack(tr.sq_params)
            del tr
        rb = a.d * (1 if kind == "sq8" else 2)
        arms = {}
        for name, R in (("all_device", None), ("R0", 0), ("Rhalf", a.n // 2)):
            t0 = time.perf_counter()
            arms[name] = build(kind, a.d, a.nlist, cent, sq, rows, lists, R)
            print(json.dumps({"kind": kind, "arm": name, "R": R, "build_s": time.perf_counter() - t0,
                              "host_GB": arms[name].host_bytes / 1e9, "n_dev": arms[name].n_dev}), flush=True)
        par = qs[:256]
        Ia, Da = arms["all_device"].search_ids(par, a.k, a.nprobe)
        for name in ("R0", "Rhalf"):
            Ib, Db = arms[name].search_ids(par, a.k, a.nprobe)
            print(json.dumps({"kind": kind, "arm": name, "parity_256": bool(torch.equal(Ia, Ib) and torch.equal(Da, Db))}),
                  flush=True)
        for nq in (int(x) for x in a.nqs.split(",")):
            q = qs[:nq]
            lp = probe.coarse(q, a.nprobe)[0].cpu().numpy()
            res = {name: [] for name in arms}
            for _ in range(a.reps):                          # alternate the arms
                for name, ix in arms.items():
                    res[name].append(timed(ix, q, a.k, a.nprobe, 1))
            t_dev = float(np.median(res["all_device"]))
            for name, ix in arms.items():
                t = float(np.median(res[name]))
                l_dev = int(np.searchsorted(off, ix.n_dev, side="right")) - 1 if name != "all_device" else a.nlist
                hb = host_bytes_per_search(lp, sizes, l_dev, rb)
                ratio = t / max(t_dev, 1e3 * hb / rate) if name != "all_device" else 1.0
                print(json.dumps({"kind": kind, "arm": name, "nq": nq, "ms": t, "qps": nq / t * 1e3,
                                  "host_GB_per_search": hb / 1e9, "overlap_ratio": ratio,
                                  "ms_all_reps": res[name]}), flush=True)
        del arms
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
