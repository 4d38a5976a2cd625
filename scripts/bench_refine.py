#!/usr/bin/env python
"""Exact re-ranking (index.IndexRefine, DESIGN §4.4) on the benchmark's IVF-PQ index: prints one JSON line.

    python scripts/bench_refine.py --n 20000000 --k-factor 8 [--steps 5 --warmup 2]

The index, corpus, queries and exact ground truth are bench.py's (same builder, same seeds, same defaults for nlist / M
/ nprobe / k / nq).  The synthetic corpus is fp32; the re-rank store holds it in fp16, as the embedding task would have
written it.  Reported:
  * unrefined and refined QPS over the same queries (CUDA events around --steps searches each);
  * the two stages on their own, CUDA events between them: base search at k' = k * k_factor, then the re-rank kernel
    (rsb_refine); gathered bytes = valid candidates x d x 2 (every candidate row is read once per query), achieved
    bytes/s against the HBM peak;
  * recall@k, exact top-1 / top-10 inside the returned k, refined and unrefined, against bench.py's fp32 ground truth;
  * parity: the re-rank of the first --parity-queries queries equals oracle/refine_oracle.py (faiss IndexRefine::search)
    on the same candidates, every returned pair re-scored in float64 from the store;
  * the card's name and power limit.
The fp16 store (n x d x 2 bytes: 154 GB at 100M) must fit in device memory next to the index; sizes that do not are
refused before anything is built.

    python scripts/bench_refine.py --n 20000000 --device-rows 0 [--staging-gb 1] [--compare-device]

--device-rows R makes the store tiered (rows [0, R) in device memory, the rest in pinned host memory) and reports, at
every --tiered-nq batch size (k = --k, k_factor = --k-factor):
  * refined and unrefined QPS, and the re-rank alone;
  * the re-rank's sort / gather / score milliseconds (CUDA events per query chunk, rsb_refine_tiered_profile);
  * distinct host rows gathered per re-rank and their fraction of the host-tier candidates; gathered GB/s against a
    plain pinned -> device cudaMemcpy measured in the same run (the achievable PCIe reference);
  * with R = 0, the zero-copy baseline: the all-device kernel (rsb_refine) handed the mapped host pointer directly;
  * with --compare-device, the all-device store in the same run: byte-identical results required;
  * recall@k refined and unrefined and the parity block, at the largest batch;
  * the card's name and power limit, the PCIe link generation and width, the host's MemAvailable.
The host tier is capped at half of MemAvailable (larger sizes are refused before anything is built) and freed at exit.

    python scripts/bench_refine.py --n 20000000 --k-factor 8 --store-dtype sq8 --compare-store float16

--store-dtype picks the store: float16 (default), float32, or sq8 (8-bit scalar-quantizer codes, faiss Refine(SQ8),
trained on the first --sq-train-rows corpus rows).  --compare-store builds a second store of another dtype on the same
index in the same run.  With either set to something other than a lone float16 store, the line holds one block per store
under "stores": dtype, device / host bytes, build seconds, and per --store-nq batch size the refined QPS, the re-rank
kernel milliseconds and gathered GB/s (nq x k' x d x element bytes over the kernel time), with recall@k, exact
top-1 / top-10 and parity at the largest batch.  With --device-rows the same options apply to the tiered store (the
comparison store is then all-device and must be byte-identical for sq8 vs sq8 only).

    python scripts/bench_refine.py --n 20000000 --k-factor 8 --pq-arms 64x8,64x4,128x4

--pq-arms builds one IVF-PQ index per arm MxNBITS (4-bit codes: two per byte, faiss' packing) on the same corpus and
coarse centroids, and one fp16 and one sq8 re-rank store shared by all arms (the re-rank depends on the candidates only).
Per --store-nq batch size the arms are measured one after the other (alternated), each unrefined and refined from both
stores (base search at k' = k * k_factor, then the re-rank kernel: rsb_search_refine gives the same result in one call).
Per arm: QPS, the LUT and scan milliseconds of the base search (RSB_PROF), recall@k / top-1 / top-10 at the largest batch,
build seconds, and the parity block (the re-rank against oracle/refine_oracle.py as above, plus every pair of the
unrefined result re-scored in float64 from the exported codes, oracle/pq4_oracle.py).  --nbits applies to the other
modes' single index (default 8: bench.py's index)."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np
import torch

import bench as B


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k-factor", type=int, default=8)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--n", type=int, default=20_000_000)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--nlist", type=int, default=16384)
    ap.add_argument("--m", type=int, default=64)
    ap.add_argument("--nprobe", type=int, default=32)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--train-per-centroid", type=int, default=64)
    ap.add_argument("--recall-queries", type=int, default=1000)
    ap.add_argument("--parity-queries", type=int, default=256)
    ap.add_argument("--device-rows", type=int, default=None, help="tiered store: rows kept in device memory")
    ap.add_argument("--staging-gb", type=float, default=1.0, help="tiered store: staging buffer (GiB)")
    ap.add_argument("--tiered-nq", default="1,64,10000", help="tiered store: batch sizes to report")
    ap.add_argument("--compare-device", action="store_true", help="tiered store: also build the all-device store")
    ap.add_argument("--store-dtype", default="float16", choices=("float16", "float32", "sq8"))
    ap.add_argument("--compare-store", default=None, choices=("float16", "float32", "sq8"),
                    help="all-device runs: also build a store of this dtype on the same index")
    ap.add_argument("--store-nq", default="10000,64,1", help="batch sizes reported per store (--store-dtype / --compare-store)")
    ap.add_argument("--sq-train-rows", type=int, default=1_000_000, help="sq8: corpus rows the quantizer is trained on")
    ap.add_argument("--nbits", type=int, default=8, choices=(8, 4), help="bits per sub-quantizer of the single index")
    ap.add_argument("--pq-arms", default=None, help="compare IVF-PQ arms MxNBITS, e.g. 64x8,64x4,128x4")
    a = ap.parse_args()
    a.partition = "list"
    return a


ELEM_BYTES = {"float16": 2, "float32": 4, "sq8": 1}


def store_bytes(args, dtype="float16") -> int:
    return args.n * args.d * ELEM_BYTES[dtype]


def train_sq8(refs, corpus, args):
    """Trains every sq8 store in refs on the first min(n, --sq-train-rows) corpus rows."""
    refs = [r for r in refs if r.store_dtype == "sq8"]
    if not refs:
        return
    n = min(args.n, args.sq_train_rows)
    x = torch.cat([corpus.chunk(c, B.CHUNK_ROWS) for c in range((n + B.CHUNK_ROWS - 1) // B.CHUNK_ROWS)])[:n]
    for r in refs:
        r.train_store(x)
    del x


def fill_stores(stores, corpus, args):
    """Trains the sq8 stores, then adds every corpus chunk to every store; returns the build seconds per store."""
    secs = {}
    for name, ref in stores.items():
        t0 = time.time()
        train_sq8([ref], corpus, args)
        ref.reserve(args.n)
        secs[name] = time.time() - t0
    for c in range((args.n + B.CHUNK_ROWS - 1) // B.CHUNK_ROWS):
        x = corpus.chunk(c, B.CHUNK_ROWS)[: min(B.CHUNK_ROWS, args.n - c * B.CHUNK_ROWS)]
        for name, ref in stores.items():
            torch.cuda.synchronize()
            t0 = time.time()
            ref.add_store(x)
            torch.cuda.synchronize()
            secs[name] += time.time() - t0
    return secs


def decoded_rows(ref, rows: torch.Tensor) -> np.ndarray:
    """Store rows as the re-rank scores them: sq8 codes decoded by the oracle's rule, others upcast."""
    if ref.store_dtype != "sq8":
        return rows.cpu().numpy()
    from oracle import sq8_oracle as S
    sq = torch.stack(ref.sq_params).cpu().numpy()
    return S.sq8_decode(rows.cpu().numpy().reshape(-1, ref.d), sq).reshape(rows.shape)


def gpu_identity(device) -> dict:
    out = {"gpu": torch.cuda.get_device_name(device), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", f"--id={device.index or 0}", "--query-gpu=power.limit",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception:
        pass
    return out


def build_arms(args, device, arms, gt_queries):
    """IVF-PQ indexes (M, nbits) for every arm on bench.py's corpus, with bench.build_index's rules: coarse k-means on
    the same training sample, each PQ codebook trained on the residuals of its first 256 * 256 rows (the sample bench.py
    uses), rows added chunk by chunk with ids = row numbers.  The coarse assignment of a chunk and the exact top-k ground
    truth are computed once for all arms.  The 8-bit arm is the index bench.py builds.  Returns (indexes, corpus,
    gt_I, build seconds per arm)."""
    import retrieval_scaling_b200 as rsb
    from retrieval_scaling_b200 import synth, train
    t0 = time.time()
    corpus = synth.Corpus(d=args.d, mode="gmm", n_centres=max(16, args.nlist // 4), device=device)
    xt = corpus.train_sample(min(args.n, args.nlist * args.train_per_centroid))
    cent = train.kmeans(xt, args.nlist, niter=10, metric="ip", spherical=True, seed=1234)
    xs = xt[: 256 * 256]
    a = train.assign_ip(xs, cent)
    t_coarse = time.time() - t0
    indexes, secs = {}, {}
    for m, nbits in arms:
        t1 = time.time()
        ix = rsb.IndexIVFPQ(args.d, args.nlist, m, nbits, device=device)
        ix.nprobe = args.nprobe
        ix.set_centroids(cent)
        ix.set_codebook(train.train_pq(xs - cent[a], m, 1 << nbits, niter=25, seed=1234))
        torch.cuda.synchronize()
        indexes[(m, nbits)], secs[(m, nbits)] = ix, t_coarse + time.time() - t1
    del xt, xs, a
    first = next(iter(indexes.values()))
    gt = {"D": None, "I": None, "pD": [], "pI": []}
    t_gt = 0.0
    for c in range((args.n + B.CHUNK_ROWS - 1) // B.CHUNK_ROWS):
        rows = min(B.CHUNK_ROWS, args.n - c * B.CHUNK_ROWS)
        t1 = time.time()
        x = corpus.chunk(c, B.CHUNK_ROWS)[:rows]
        D, I = rsb.knn_ip(gt_queries, x, args.k, id_offset=c * B.CHUNK_ROWS)
        gt["pD"].append(D); gt["pI"].append(I)
        if len(gt["pD"]) == 15:
            B._fold_gt(gt, args.k)
        lists = first.assign(x)
        ids = torch.arange(c * B.CHUNK_ROWS, c * B.CHUNK_ROWS + rows, dtype=torch.int64, device=device)
        torch.cuda.synchronize()
        t_shared = time.time() - t1                   # corpus chunk + coarse assignment: charged to every arm
        t_gt += t_shared
        for key, ix in indexes.items():
            t1 = time.time()
            ix.add_preassigned(x, lists, ids)
            secs[key] += t_shared + time.time() - t1
        del x, lists, ids
    for key, ix in indexes.items():
        t1 = time.time()
        ix.finalize()
        torch.cuda.synchronize()
        secs[key] += time.time() - t1
    B._fold_gt(gt, args.k)
    return indexes, corpus, gt["I"], secs


def build_index(args, device, gt_queries):
    """bench.py's index (--nbits 8), or the same build with 4-bit sub-quantizers."""
    if args.nbits == 8:
        return B.build_index(args, 0, 1, device, gt_queries=gt_queries)
    indexes, corpus, gt_I, secs = build_arms(args, device, [(args.m, args.nbits)], gt_queries)
    return indexes[(args.m, args.nbits)], corpus, None, gt_I, {"total_s": secs[(args.m, args.nbits)]}


def arm_parity(index, xq, D, I, npq):
    """Every (query, id, score) of the unrefined result re-scored in float64 from the exported codes."""
    from oracle import pq4_oracle as P4
    off, codes, ids = (t.cpu().numpy() for t in index.export_lists())
    host = P4.host_ivfpq(index.get_centroids().cpu().numpy(), index.get_codebook().cpu().numpy(), off, codes, ids)
    r = host.verify_pairs(xq[:npq].cpu().numpy(), D[:npq].cpu().numpy(), I[:npq].cpu().numpy(), rtol=1e-5, atol=2e-4)
    r["oracle"] = "oracle/pq4_oracle.host_ivfpq (parity.HostIVFPQ on unpacked codes): <q, c_l + decode(code)> in float64"
    r["ok"] = bool(r["rescore_out_of_tol"] == 0 and r["unknown_ids"] == 0)
    return r


def arms_main(args, device):
    """IVF-PQ arms MxNBITS on one corpus, each unrefined and re-ranked from a shared fp16 and a shared sq8 store."""
    import retrieval_scaling_b200 as rsb
    from retrieval_scaling_b200 import synth
    arms = [tuple(int(v) for v in s.lower().split("x")) for s in args.pq_arms.split(",")]
    dtypes = ["float16", "sq8"]
    need = sum(store_bytes(args, t) for t in dtypes) + sum(args.n * (m * nb // 8 + 8) for m, nb in arms) \
        + 2 * B.CHUNK_ROWS * args.d * 4
    free, _ = torch.cuda.mem_get_info(device)
    if need > 0.9 * free:
        raise SystemExit(f"the stores and the {len(arms)} indexes need ~{need} bytes, {free} are free on {device}")
    k, kf = args.k, args.k_factor
    kb = k * kf
    probe = synth.Corpus(d=args.d, mode="gmm", n_centres=max(16, args.nlist // 4), device=device)
    xq_all = probe.queries(args.nq)
    del probe
    n_gt = min(args.recall_queries, args.nq)
    indexes, corpus, gt_I, build_s = build_arms(args, device, arms, xq_all[:n_gt].contiguous())
    first = next(iter(indexes.values()))
    stores = {t: rsb.IndexRefine(first, t, kf) for t in dtypes}
    store_s = fill_stores(stores, corpus, args)
    info = gpu_identity(device)
    strip = lambda r: {kk: vv for kk, vv in r.items() if kk != "ground_truth"}   # noqa: E731
    nqs = sorted({min(int(v), args.nq) for v in args.store_nq.split(",")}, reverse=True)
    name = lambda key: f"PQ{key[0]}x{key[1]}"                                    # noqa: E731
    blocks = {name(key): {"M": key[0], "nbits": key[1], "code_bytes": key[0] * key[1] // 8,
                          "index_bytes": ix.index_bytes, "build_s": build_s[key], "per_nq": []}
              for key, ix in indexes.items()}

    def refined(ix, ref, xq):
        Ib, _ = ix.search_ids(xq, kb)
        return ref.rerank(xq, Ib, k)

    for nq in nqs:
        xq = xq_all[:nq].contiguous()
        for key, ix in indexes.items():                 # arms alternated inside every batch size
            blk = blocks[name(key)]
            ms_u, (Iu, Du) = timed(lambda: ix.search_ids(xq, k), args.steps, args.warmup)
            ix.set_profiling(True)
            for _ in range(args.steps):
                ix.search_ids(xq, k)
            prof = ix.profile()
            ix.set_profiling(False)
            row = {"nq": nq, "qps_unrefined": nq / (ms_u / 1e3), "ms_per_step_unrefined": ms_u,
                   "lut_ms": prof["lut_ms"], "scan_ms": prof["scan_ms"], "coarse_ms": prof["coarse_ms"]}
            for t, ref in stores.items():
                ms_r, (I, D) = timed(lambda: refined(ix, ref, xq), args.steps, args.warmup)
                row[f"qps_refined_{t}"] = nq / (ms_r / 1e3)
                row[f"ms_per_step_refined_{t}"] = ms_r
                if nq == nqs[0]:
                    ng = min(n_gt, nq)
                    blk[f"recall_refined_{t}"] = strip(B.recall_block(I[:ng], gt_I[:ng], k))
                    Ib, _ = ix.search_ids(xq, kb)
                    Ir, Dr = ref.rerank(xq, Ib, k)
                    blk[f"parity_refined_{t}"] = parity(ref, xq, Ib, Ir, Dr, k, min(args.parity_queries, nq))
            if nq == nqs[0]:
                ng = min(n_gt, nq)
                blk["recall_unrefined"] = strip(B.recall_block(Iu[:ng], gt_I[:ng], k))
                blk["recall_nq"] = ng
                blk["parity_unrefined"] = arm_parity(ix, xq, Du, Iu, min(args.parity_queries, nq))
            blk["per_nq"].append(row)
    out = {"metric": f"IVF-PQ arms {args.pq_arms}: unrefined and exact re-ranking of k x {kf} candidates, "
                     f"{args.n // 1_000_000}M x {args.d}",
           "config": {**{kk: vv for kk, vv in B.make_config(args, 1).items() if kk not in ("M", "nbits")},
                      "k_factor": kf, "k_base": kb},
           "arms": blocks, "stores": {t: {"bytes": store_bytes(args, t), "build_s": store_s[t]} for t in dtypes},
           **info, "refined_timing": "base search at k x k_factor, then the re-rank kernel (two calls per step)",
           "recall_ground_truth": "exact fp32 inner-product search over the same corpus (librsb Flat kernels)",
           "steps": args.steps, "warmup": args.warmup}
    print(json.dumps(out), flush=True)
    return 0


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, out


def parity(ref, xq, Ib, Ir, Dr, k, npq):
    """The re-rank result is the exact top-k of the base's k' candidates: oracle on the same candidates, float64."""
    from oracle import parity as P
    from oracle import refine_oracle as R
    kb = Ib.shape[1]
    Ib_h = Ib[:npq].cpu().numpy()
    rows = decoded_rows(ref, ref.store_rows(Ib[:npq].clamp_min(0).reshape(-1)).reshape(npq, kb, -1))   # [npq, k', d]
    xq_h = xq[:npq].cpu().numpy()
    Dref = np.full((npq, k), np.finfo(np.float32).min, np.float32)
    Iref = np.full((npq, k), -1, np.int64)
    exact = {}
    for i in range(npq):
        loc = np.where(Ib_h[i] >= 0, np.arange(kb), -1)
        Dl, Il = R.refine_candidates(xq_h[i:i + 1], rows[i], loc[None], k, dtype=np.float64)
        Dref[i], Iref[i] = Dl[0], np.where(Il[0] >= 0, Ib_h[i][Il[0].clip(0)], -1)
        s64 = rows[i].astype(np.float64) @ xq_h[i].astype(np.float64)
        exact.update({(i, int(c)): float(s64[j]) for j, c in enumerate(Ib_h[i]) if c >= 0})
    Dg, Ig = Dr[:npq].cpu().numpy(), Ir[:npq].cpu().numpy()
    par = P.topk_parity(Dg, Ig, Dref, Iref, rtol=1e-5, atol=1e-5,
                        score_of=lambda qs, ids: [exact.get((int(a), int(b)), np.nan) for a, b in zip(qs, ids)])
    pairs = [(i, int(c), float(Dg[i, r])) for i in range(npq) for r, c in enumerate(Ig[i]) if c >= 0]
    bad = sum(1 for i, c, s in pairs if (i, c) not in exact or abs(exact[(i, c)] - s) > 1e-5 + 1e-5 * abs(exact[(i, c)]))
    par.update({"queries": f"the first {npq} queries", "rescored_pairs": len(pairs), "rescore_out_of_tol": bad,
                "oracle": "oracle/refine_oracle.py (faiss IndexRefine::search) on the GPU's base candidates, float64"})
    par["ok"] = bool(par["non_tie_mismatches"] == 0 and par["scores_out_of_tol"] == 0 and par["padding_mismatches"] == 0
                     and bad == 0)
    return par


def host_identity(device) -> dict:
    """PCIe link (read-only nvidia-smi query) and the host's MemAvailable."""
    out = {"host_mem_available_bytes": mem_available()}
    for key, field in (("pcie_link_gen", "pcie.link.gen.current"), ("pcie_link_width", "pcie.link.width.current"),
                       ("pcie_link_gen_max", "pcie.link.gen.max"), ("pcie_link_width_max", "pcie.link.width.max")):
        out[key] = None
        try:
            r = subprocess.run(["nvidia-smi", f"--id={device.index or 0}", f"--query-gpu={field}",
                                "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20)
            v = (r.stdout.strip() or r.stderr.strip()).splitlines()[0].strip()
            out[key] = int(v) if v.isdigit() else v
        except Exception:
            pass
    return out


def mem_available() -> int:
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    raise SystemExit("MemAvailable not found in /proc/meminfo")


def pinned_copy_gbs(device, nbytes=1 << 30, reps=10) -> float:
    """Plain pinned host -> device copy bandwidth (cudaMemcpyAsync of a page-locked buffer): the PCIe reference."""
    from retrieval_scaling_b200 import _lib
    from retrieval_scaling_b200.index import _pinned_rows
    src = _pinned_rows(_lib.lib(), nbytes // 16, 16, torch.uint8, device)
    dst = torch.empty_like(src, device=device)
    dst.copy_(src, non_blocking=True)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        dst.copy_(src, non_blocking=True)
    e1.record()
    torch.cuda.synchronize()
    return nbytes * reps / (e0.elapsed_time(e1) / 1e3) / 1e9


def tiered_profile(L, enable):
    import ctypes
    ms = (ctypes.c_double * 3)()
    from retrieval_scaling_b200 import _lib
    _lib.check(L.rsb_refine_tiered_profile(int(enable), ms))
    return list(ms)


def zero_copy_rerank(ref, q, Ib, k):
    """The all-device kernel (rsb_refine with n_dev = ntotal) handed the mapped host tier of a --device-rows 0 store
    directly as its device rows: every candidate row crosses PCIe once per query, no de-duplication, no staging."""
    from retrieval_scaling_b200 import _lib
    from retrieval_scaling_b200.index import _ptr, _stream
    nq, kb = Ib.shape
    D = torch.empty((nq, k), dtype=torch.float32, device=ref.device)
    I = torch.empty((nq, k), dtype=torch.int64, device=ref.device)
    dt = _lib.RSB_DTYPE_F16 if ref.store_dtype == "float16" else _lib.RSB_DTYPE_F32
    ws = ref.base._workspace(ref.L.rsb_refine_workspace_bytes(nq, kb, k, ref.d, dt, ref.ntotal, ref.ntotal, 0))
    _lib.check(ref.L.rsb_refine(_ptr(q), nq, _ptr(ref.host_store), ref.ntotal, None, dt, None, ref.d, ref.ntotal,
                                _ptr(Ib), kb, k, _ptr(D), _ptr(I), _ptr(ws), ws.numel(), 0, None, _stream()))
    return I, D


def tiered_main(args, device):
    import retrieval_scaling_b200 as rsb
    from retrieval_scaling_b200 import synth
    k, kf = args.k, args.k_factor
    kb = k * kf
    n_dev = min(args.device_rows, args.n)
    dtype, eb = args.store_dtype, ELEM_BYTES[args.store_dtype]
    host_bytes = (args.n - n_dev) * args.d * eb
    avail = mem_available()
    if host_bytes > avail // 2:
        raise SystemExit(f"the host tier of {args.n - n_dev} x {args.d} {dtype} needs {host_bytes} bytes of pinned memory; "
                         f"the cap is half of MemAvailable = {avail // 2} bytes: use a larger --device-rows or a smaller --n")
    free, _ = torch.cuda.mem_get_info(device)
    dev_bytes = n_dev * args.d * eb + (store_bytes(args, dtype) if args.compare_device else 0)
    # + the corpus generator's fp32 chunk and its temporary while the store is filled
    need = dev_bytes + args.n * (args.m + 8) + int(args.staging_gb * (1 << 30)) + 2 * B.CHUNK_ROWS * args.d * 4
    if need > 0.9 * free:
        raise SystemExit(f"the device tier, the index and the staging buffer need ~{need} bytes, {free} are free on "
                         f"{device}: use a smaller --device-rows or drop --compare-device")
    info = {**gpu_identity(device), **host_identity(device), "pinned_to_device_memcpy_gbs": pinned_copy_gbs(device)}
    probe = synth.Corpus(d=args.d, mode="gmm", n_centres=max(16, args.nlist // 4), device=device)
    xq_all = probe.queries(args.nq)
    del probe
    n_gt = min(args.recall_queries, args.nq)
    index, corpus, _, gt_I, build = build_index(args, device, xq_all[:n_gt].contiguous())

    stores = {"tiered": rsb.IndexRefine(index, dtype, kf, device_rows=n_dev)}
    if args.compare_device:
        stores["device"] = rsb.IndexRefine(index, dtype, kf)
    for ref in stores.values():
        ref.staging_bytes = int(args.staging_gb * (1 << 30))
    store_s = fill_stores(stores, corpus, args)["tiered"]
    ref = stores["tiered"]
    L = ref.L

    per_nq = []
    for nq in [int(v) for v in args.tiered_nq.split(",")]:
        nq = min(nq, args.nq)
        xq = xq_all[:nq].contiguous()
        ms_unref, (Iu, _) = timed(lambda: index.search_ids(xq, k), args.steps, args.warmup)
        ms_ref, (I, D) = timed(lambda: ref.search_ids(xq, k), args.steps, args.warmup)
        Ib, _ = index.search_ids(xq, kb)
        ms_rerank, (Ir, Dr) = timed(lambda: ref.rerank(xq, Ib, k), args.steps, args.warmup)
        rows = torch.zeros(1, dtype=torch.int64, device=device)
        tiered_profile(L, 1)
        for _ in range(args.steps):
            ref.rerank(xq, Ib, k, host_rows=rows)
        split = [v / args.steps for v in tiered_profile(L, 0)]
        uniq = int(rows.item()) / args.steps
        host_cand = int(((Ib >= n_dev) & (Ib < args.n)).sum().item())
        row = {"nq": nq, "qps_refined": nq / (ms_ref / 1e3), "qps_unrefined": nq / (ms_unref / 1e3),
               "ms_per_step_refined": ms_ref, "ms_per_step_unrefined": ms_unref, "rerank_ms": ms_rerank,
               "sort_ms": split[0], "gather_ms": split[1], "score_ms": split[2],
               "host_tier_candidates": host_cand, "unique_host_rows": uniq,
               "unique_frac_of_host_candidates": uniq / host_cand if host_cand else None,
               "gathered_bytes": uniq * args.d * eb,
               "gathered_gbs": uniq * args.d * eb / (split[1] / 1e3) / 1e9 if split[1] > 0 else None}
        row["gathered_frac_of_memcpy"] = (row["gathered_gbs"] / info["pinned_to_device_memcpy_gbs"]
                                          if row["gathered_gbs"] else None)
        row["same_result_as_two_stage"] = bool(torch.equal(I, Ir) and torch.equal(D, Dr))
        if n_dev == 0 and dtype != "sq8":
            ms_zc, (Iz, Dz) = timed(lambda: zero_copy_rerank(ref, xq, Ib, k), args.steps, args.warmup)
            row["zero_copy_rerank_ms"] = ms_zc
            row["zero_copy_same_result"] = bool(torch.equal(Iz, Ir) and torch.equal(Dz, Dr))
        else:
            row["zero_copy_rerank_ms"] = ("not measured (needs --device-rows 0: rsb_refine reads one contiguous store)"
                                          if dtype != "sq8" else "not measured (fp16 / fp32 stores only)")
        if "device" in stores:
            full = stores["device"]
            ms_dev, (Id, Dd) = timed(lambda: full.search_ids(xq, k), args.steps, args.warmup)
            ms_dev_rr, (Idr, Ddr) = timed(lambda: full.rerank(xq, Ib, k), args.steps, args.warmup)
            row.update({"device_store_qps_refined": nq / (ms_dev / 1e3), "device_store_rerank_ms": ms_dev_rr,
                        "identical_to_device_store": bool(torch.equal(I, Id) and torch.equal(D, Dd)
                                                          and torch.equal(Ir, Idr) and torch.equal(Dr, Ddr))})
        per_nq.append(row)
        last = (xq, I, Iu, Ib, Ir, Dr, nq)

    xq, I, Iu, Ib, Ir, Dr, nq = last
    strip = lambda r: {kk: vv for kk, vv in r.items() if kk != "ground_truth"}   # noqa: E731
    ng = min(n_gt, nq)
    out = {"metric": f"exact re-ranking of k x {kf} candidates from a tiered {dtype} store ({n_dev} device rows, "
                     f"{args.n - n_dev} pinned host rows), {args.n // 1_000_000}M x {args.d} IVF-PQ",
           "config": {**B.make_config(args, 1), "k_factor": kf, "k_base": kb, "device_rows": n_dev,
                      "host_rows": args.n - n_dev, "staging_bytes": ref.staging_bytes},
           "per_nq": per_nq, **info,
           "store": {"dtype": dtype, "device_bytes": n_dev * args.d * eb, "host_bytes": host_bytes, "build_s": store_s},
           "recall_nq": ng, "recall": strip(B.recall_block(I[:ng], gt_I[:ng], k)),
           "recall_unrefined": strip(B.recall_block(Iu[:ng], gt_I[:ng], k)),
           "recall_ground_truth": "bench.py's exact fp32 inner-product search over the same corpus",
           "parity": parity(ref, xq, Ib, Ir, Dr, k, min(args.parity_queries, nq)),
           "build": build, "steps": args.steps, "warmup": args.warmup}
    del stores, ref
    print(json.dumps(out), flush=True)
    return 0


def stores_main(args, device):
    """All-device stores of --store-dtype and --compare-store on one index, measured one after the other."""
    import retrieval_scaling_b200 as rsb
    from retrieval_scaling_b200 import synth
    dtypes = [args.store_dtype] + [t for t in [args.compare_store] if t and t != args.store_dtype]
    need = sum(store_bytes(args, t) for t in dtypes) + args.n * (args.m + 8) + 2 * B.CHUNK_ROWS * args.d * 4
    free, _ = torch.cuda.mem_get_info(device)
    if need > 0.9 * free:
        raise SystemExit(f"the {' + '.join(dtypes)} stores of {args.n} x {args.d} and the index need ~{need} bytes, "
                         f"{free} are free on {device}; use a smaller --n or drop --compare-store")
    k, kf = args.k, args.k_factor
    kb = k * kf
    probe = synth.Corpus(d=args.d, mode="gmm", n_centres=max(16, args.nlist // 4), device=device)
    xq_all = probe.queries(args.nq)
    del probe
    n_gt = min(args.recall_queries, args.nq)
    index, corpus, _, gt_I, build = build_index(args, device, xq_all[:n_gt].contiguous())
    stores = {t: rsb.IndexRefine(index, t, kf) for t in dtypes}
    secs = fill_stores(stores, corpus, args)
    info = gpu_identity(device)
    peak, peak_src = B.measured_peak_gbs()
    strip = lambda r: {kk: vv for kk, vv in r.items() if kk != "ground_truth"}   # noqa: E731
    nqs = sorted({min(int(v), args.nq) for v in args.store_nq.split(",")}, reverse=True)
    blocks = {}
    for t, ref in stores.items():
        eb = ELEM_BYTES[t]
        per_nq = []
        for nq in nqs:
            xq = xq_all[:nq].contiguous()
            ms_unref, (Iu, _) = timed(lambda: index.search_ids(xq, k), args.steps, args.warmup)
            ms_ref, (I, D) = timed(lambda: ref.search_ids(xq, k), args.steps, args.warmup)
            Ib, _ = index.search_ids(xq, kb)
            ms_rr, (Ir, Dr) = timed(lambda: ref.rerank(xq, Ib, k), args.steps, args.warmup)
            gathered = nq * kb * args.d * eb
            per_nq.append({"nq": nq, "qps_refined": nq / (ms_ref / 1e3), "qps_unrefined": nq / (ms_unref / 1e3),
                           "ms_per_step_refined": ms_ref, "ms_per_step_unrefined": ms_unref, "rerank_kernel_ms": ms_rr,
                           "gathered_bytes": gathered, "gathered_gbs": gathered / (ms_rr / 1e3) / 1e9,
                           "valid_candidate_frac": int((Ib >= 0).sum().item()) / (nq * kb),
                           "same_result_as_two_stage": bool(torch.equal(I, Ir) and torch.equal(D, Dr))})
            if nq == nqs[0]:
                ng = min(n_gt, nq)
                top = {"recall": strip(B.recall_block(I[:ng], gt_I[:ng], k)),
                       "recall_unrefined": strip(B.recall_block(Iu[:ng], gt_I[:ng], k)), "recall_nq": ng,
                       "parity": parity(ref, xq, Ib, Ir, Dr, k, min(args.parity_queries, nq))}
        blocks[t] = {"dtype": t, "device_bytes": store_bytes(args, t), "host_bytes": 0, "build_s": secs[t],
                     "per_nq": per_nq, **top}
        if t == "sq8":
            blocks[t]["sq8_train_rows"] = min(args.n, args.sq_train_rows)
    out = {"metric": f"exact re-ranking of k x {kf} candidates, {args.n // 1_000_000}M x {args.d} IVF-PQ, "
                     f"{' vs '.join(dtypes)} store",
           "config": {**B.make_config(args, 1), "k_factor": kf, "k_base": kb}, "stores": blocks, **info,
           "peak_gbs": peak, "peak_source": peak_src,
           "gathered_bytes_rule": "nq x k' x d x element bytes (every candidate row read once per query)",
           "recall_ground_truth": "bench.py's exact fp32 inner-product search over the same corpus",
           "build": build, "steps": args.steps, "warmup": args.warmup}
    print(json.dumps(out), flush=True)
    return 0


def main():
    args = parse()
    if not torch.cuda.is_available():
        raise SystemExit("bench_refine.py needs a CUDA device: the product path has no CPU fallback")
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    if args.pq_arms:
        return arms_main(args, device)
    if args.device_rows is not None:
        return tiered_main(args, device)
    if args.store_dtype != "float16" or args.compare_store is not None:
        return stores_main(args, device)
    need = store_bytes(args) + args.n * (args.m + 8)                   # store + PQ codes + ids
    free, _ = torch.cuda.mem_get_info(device)
    if need > 0.9 * free:
        raise SystemExit(f"the fp16 store of {args.n} x {args.d} ({store_bytes(args)} bytes) and the index need ~{need} "
                         f"bytes, {free} are free on {device}; use a smaller --n")
    import retrieval_scaling_b200 as rsb
    from retrieval_scaling_b200 import synth
    k, kf = args.k, args.k_factor
    kb = k * kf
    probe = synth.Corpus(d=args.d, mode="gmm", n_centres=max(16, args.nlist // 4), device=device)
    xq = probe.queries(args.nq)
    del probe
    n_gt = min(args.recall_queries, args.nq)
    index, corpus, _, gt_I, build = build_index(args, device, xq[:n_gt].contiguous())

    t0 = time.time()
    ref = rsb.IndexRefine(index, "float16", kf)
    ref.reserve(args.n)
    for c in range((args.n + B.CHUNK_ROWS - 1) // B.CHUNK_ROWS):
        ref.add_store(corpus.chunk(c, B.CHUNK_ROWS)[: min(B.CHUNK_ROWS, args.n - c * B.CHUNK_ROWS)])
    store_s = time.time() - t0

    ms_base_k, (Iu, _) = timed(lambda: index.search_ids(xq, k), args.steps, args.warmup)
    ms_ref, (I, D) = timed(lambda: ref.search_ids(xq, k), args.steps, args.warmup)
    # the stages on their own: base search at k' -> re-rank kernel, events between them
    for _ in range(args.warmup):
        Ib, _ = index.search_ids(xq, kb)
        ref.rerank(xq, Ib, k)
    torch.cuda.synchronize()
    evs = []
    for _ in range(args.steps):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record()
        Ib, _ = index.search_ids(xq, kb)
        ev[1].record()
        Ir, Dr = ref.rerank(xq, Ib, k)
        ev[2].record()
        evs.append(ev)
    torch.cuda.synchronize()
    base_ms = float(np.mean([a.elapsed_time(b) for a, b, _ in evs]))
    refine_ms = float(np.mean([b.elapsed_time(c) for _, b, c in evs]))
    valid = int((Ib >= 0).sum().item())
    gathered = valid * args.d * 2
    peak, peak_src = B.measured_peak_gbs()
    gbs = gathered / refine_ms / 1e6
    strip = lambda r: {kk: vv for kk, vv in r.items() if kk != "ground_truth"}   # noqa: E731
    out = {"metric": f"queries/sec @ top-k={k} with exact re-ranking of k x {kf} candidates, "
                     f"{args.n // 1_000_000}M x {args.d} IVF-PQ, fp16 store",
           "config": {**B.make_config(args, 1), "k_factor": kf, "k_base": kb},
           "qps_refined": args.nq / (ms_ref / 1e3), "qps_unrefined": args.nq / (ms_base_k / 1e3),
           "ms_per_step_refined": ms_ref, "ms_per_step_unrefined": ms_base_k,
           "base_search_ms": base_ms, "refine_kernel_ms": refine_ms,
           "store": {"dtype": "float16", "bytes": store_bytes(args), "build_s": store_s},
           "gathered_bytes": gathered, "gathered_bytes_shape": args.nq * kb * args.d * 2,
           "valid_candidate_frac": valid / (args.nq * kb), "achieved_gbs": gbs, "peak_gbs": peak,
           "peak_source": peak_src, "frac_of_peak": gbs / peak, **gpu_identity(device),
           "same_result_as_two_stage": bool(torch.equal(I, Ir) and torch.equal(D, Dr)),
           "recall": strip(B.recall_block(I[:n_gt], gt_I, k)), "recall_unrefined": strip(B.recall_block(Iu[:n_gt], gt_I, k)),
           "recall_ground_truth": "bench.py's exact fp32 inner-product search over the same corpus",
           "parity": parity(ref, xq, Ib, Ir, Dr, k, min(args.parity_queries, args.nq)),
           "build": build, "steps": args.steps, "warmup": args.warmup}
    print(json.dumps(out), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())
