#!/usr/bin/env python
"""What one tiered search puts on each CUDA stream: kernel names in order, and every copy and memset with its byte
count, from a torch.profiler trace (CUDA activities).  Two builds of librsb are compared by recording each in a
process of its own and comparing the records:

    RSB_LIBRARY=<build A>/librsb.so python scripts/trace_tiered_streams.py --out a.json
    RSB_LIBRARY=<build B>/librsb.so python scripts/trace_tiered_streams.py --out b.json
    python scripts/trace_tiered_streams.py --compare a.json b.json

Workloads (seeded): a tiered fp16 Flat index with R = ntotal / 2 and a staging size that splits the host tier into 5
chunks, and a tiered IVF-SQ8 index (by residual) with half its rows in device memory and a staging size that gives
several chunks per query batch.  Streams are numbered by their first activity in the trace, so records of different
processes line up.  --compare exits non-zero when any stream differs."""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--compare", nargs=2)
    ap.add_argument("--n", type=int, default=200_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--nq", type=int, default=1024)
    ap.add_argument("--k", type=int, default=100)
    return ap.parse_args()


def streams_of(search):
    """Runs search() once to warm up, then once under the profiler -> {stream number: [activity, ...]}."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    search()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        search()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "trace.json")
        prof.export_chrome_trace(path)
        with open(path) as f:
            events = json.load(f)["traceEvents"]
    acts = sorted((e for e in events if e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset")), key=lambda e: e["ts"])
    number, out = {}, {}
    for e in acts:
        s = number.setdefault(e["args"]["stream"], len(number))
        item = e["name"] if e["cat"] == "kernel" else f'{e["name"]} {e["args"].get("bytes")} B'
        out.setdefault(str(s), []).append(item)
    return out


def record(a):
    import numpy as np
    import torch
    import retrieval_scaling_b200 as rsb
    torch.cuda.set_device(0)
    rng = np.random.default_rng(0)
    n, d, nq, k = a.n, a.d, a.nq, a.k
    xb = rng.standard_normal((n, d)).astype(np.float16)
    q = torch.from_numpy(rng.standard_normal((nq, d)).astype(np.float32)).cuda()
    out = {"gpu": subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                 capture_output=True, text=True).stdout.strip()}

    host = n - n // 2
    flat = rsb.IndexFlatIP(d, dtype="float16", device_rows=n // 2, staging_bytes=(host // 5) * d * 2)
    flat.add(xb)
    out["flat"] = streams_of(lambda: flat.search_ids(q, k))

    nlist, nprobe = 256, 64
    cent = rng.standard_normal((nlist, d)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    ivf = rsb.IndexIVFScalarQuantizer(d, nlist, by_residual=True, list_device_rows=n // 2, staging_bytes=8 << 20)
    ivf.set_centroids(cent)
    ivf.train_sq(xb)
    lists = ivf.assign(xb)
    ivf.reserve_lists(np.bincount(lists.cpu().numpy(), minlength=nlist))
    ivf.add_preassigned(xb, lists)
    out["ivf_sq8"] = streams_of(lambda: ivf.search_ids(q, k, nprobe))

    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    for w in ("flat", "ivf_sq8"):
        print(w, {s: len(v) for s, v in out[w].items()})


def compare(pa, pb):
    with open(pa) as f:
        A = json.load(f)
    with open(pb) as f:
        B = json.load(f)
    same = True
    for w in ("flat", "ivf_sq8"):
        for s in sorted(set(A[w]) | set(B[w])):
            ea, eb = A[w].get(s, []), B[w].get(s, [])
            kern = sum(1 for x in ea if not x.startswith("Mem"))
            print(f"{w} stream {s}: {len(ea)} / {len(eb)} activities ({kern} kernels, {len(ea) - kern} copies / "
                  f"memsets): {'same' if ea == eb else 'DIFFERENT'}")
            same &= ea == eb
    print("SAME" if same else "DIFFERENT")
    return 0 if same else 1


if __name__ == "__main__":
    args = parse()
    if args.compare:
        sys.exit(compare(*args.compare))
    record(args)
