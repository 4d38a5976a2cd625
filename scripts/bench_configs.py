#!/usr/bin/env python
"""Side measurements for the BASELINE configurations that are parity-test cases rather than the bench line:
  C1  Flat, 100k x 768 iid fp32, 1k queries, top-10
  C2  IVF-Flat nlist=4096 nprobe=64, 10M x 768 synthetic gmm, top-100  (30.7 GB of fp32 vectors on the GPU)
  c1_large  Flat 768-d past the 8 GB limit of the 3xTF32 split, fp16 storage (tensor cores) vs fp32 (CUDA cores)
  c2_sq8    C2 as fp16 IVF-Flat and as IVF-SQ8 with / without residuals (run only when named)
Every config measures fp16 storage and fp32 storage of the same (fp16-representable) values; the card name and power
limit are part of each JSON object.  C1 alternates the arms in one loop; C2 and c1_large build one index at a time
(the two do not fit on one 80 GB card together) and compare the results of a query sample afterwards.
Prints one JSON object per config (QPS, algorithmic GB/s or TFLOP/s, CPU oracle rate on a bounded sample)."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import subprocess

import numpy as np
import torch

import retrieval_scaling_b200 as rsb
from retrieval_scaling_b200 import synth, train


def timed(fn, steps=5, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def card():
    """Name and power limit of the GPU the numbers were taken on (read-only nvidia-smi query)."""
    out = {"gpu": torch.cuda.get_device_name()}
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                            f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30)
        out["power_limit_and_max_sm_clock"] = r.stdout.strip()
    except Exception as e:          # the numbers stay usable; say why the card details are missing
        out["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return out


def c1_flat():
    from oracle import ann_oracle as O
    g = torch.Generator(device="cuda").manual_seed(1234)
    xb = torch.randn(100_000, 768, generator=g, device="cuda").half().float()       # fp16-representable: same data for all arms
    xq = torch.randn(1000, 768, generator=torch.Generator(device="cuda").manual_seed(4321), device="cuda")
    index = rsb.IndexFlatIP(768)
    index.add(xb)
    index16 = rsb.IndexFlatIP(768, dtype="float16")
    index16.add(xb.half())
    arms = (("fp16_storage_tensor_f16x2_plus_exact_rescore", index16, 1), ("tensor_3xtf32_plus_exact_rescore", index, 1),
            ("cuda_core_fp32", index, 0))
    times = {name: [] for name, _, _ in arms}
    for _ in range(3):                                    # alternate the arms
        for name, ix, opt in arms:
            if ix is index:
                ix.set_option(0, opt)
            times[name].append(timed(lambda: ix.search_ids(xq, 10)))
    out = {}
    for name, ts in times.items():
        ms = min(ts)
        out[name] = {"ms": ms, "ms_all": ts, "queries_per_s": 1000 / ms * 1e3,
                     "tflops_fp32_equiv": 2 * 1000 * 100_000 * 768 / ms / 1e9}
    index.set_option(0, 1)
    I, D = index.search_ids(xq, 10)
    I16, D16 = index16.search_ids(xq, 10)
    same16 = I16 == I
    assert torch.equal(D16[same16], D[same16])            # exact re-score: bit-equal wherever the ids agree
    t0 = time.perf_counter()
    Dr, Ir = O.flat_search(xq.cpu().numpy(), xb.cpu().numpy(), 10)
    cpu_s = time.perf_counter() - t0
    same = float((I.cpu().numpy() == Ir).mean())
    rel = float(np.abs(D.cpu().numpy() - Dr).max() / np.abs(Dr).max())
    O.assert_topk_equivalent(D16.cpu().numpy(), I16.cpu().numpy(), Dr, Ir, rtol=1e-5, atol=1e-5)
    return {"config": "C1 Flat 100k x 768 iid (fp16-representable), 1k queries, top-10", **card(), **out,
            "ids_identical_fraction": same, "fp16_ids_identical_to_fp32": float(same16.float().mean()),
            "max_rel_score_err": rel, "cpu_numpy_sgemm_queries_per_s": 1000 / cpu_s, "cpu_threads": os.cpu_count()}


def c1_large(n16=20_000_000, n32=10_000_000, d=768, k=100, nq_check=16):
    """Flat past the 8 GB cliff of the 3xTF32 split.  fp16: n16 rows (30.7 GB at 20M) on the fp16 tensor-core scorer.
    fp32: n32 rows on the CUDA-core sgemm path (rsb_finalize concatenates the add batches, so an fp32 Flat needs twice
    its payload while it is built: 20M x 768 fp32 = 61 GB does not build on an 80 GB card, 10M = 30.7 GB does).  The
    first n32 rows are the same values in both; parity: the fp16 index built from those n32 rows against the fp32 one."""
    from oracle import ann_oracle as O
    g = torch.Generator(device="cuda").manual_seed(77)
    xq_all = torch.randn(1024, d, generator=g, device="cuda")
    out = {"config": f"C1-large Flat {d}-d, top-{k}: fp16 {n16} rows, fp32 {n32} rows", **card()}

    def rows(c, m):
        return (0.05 * torch.randn(m, d, generator=torch.Generator(device="cuda").manual_seed(1000 + c), device="cuda")).half()

    def measure(ix, n, tag):
        res = {"index_gb": ix.index_bytes / 1e9}
        for nq in (1, 64, 1024):
            ms = timed(lambda: ix.search_ids(xq_all[:nq], k), steps=3, warmup=1)
            res[f"nq_{nq}"] = {"ms": ms, "queries_per_s": nq / ms * 1e3, "tflops_algorithmic": 2 * nq * n * d / ms / 1e9}
        out[tag] = res

    def build(dtype, n):
        ix = rsb.IndexFlatIP(d, dtype=dtype)
        for c in range(n // 1_000_000):
            x = rows(c, 1_000_000)
            ix.add(x if dtype == "float16" else x.float())
            del x
        ix.finalize()
        return ix

    ix = build("float16", n16)
    measure(ix, n16, "fp16_storage_tensor")
    del ix
    ix = build("float16", n32)
    I16, D16 = (t.cpu() for t in ix.search_ids(xq_all[:nq_check], k))
    del ix
    torch.cuda.empty_cache()
    ix = build("float32", n32)
    measure(ix, n32, "fp32_storage_cuda_core")
    I32, D32 = (t.cpu() for t in ix.search_ids(xq_all[:nq_check], k))
    del ix
    same = I16 == I32
    O.assert_topk_equivalent(D16.numpy(), I16.numpy(), D32.numpy(), I32.numpy(), rtol=1e-5, atol=1e-5)
    out["parity_fp16_vs_fp32_ids_identical_fraction"] = float(same.float().mean())
    out["parity_fp16_vs_fp32_max_abs_score_diff_where_ids_equal"] = float((D16[same] - D32[same]).abs().max())
    return out


def c2_ivfflat(n=10_000_000, nlist=4096, nprobe=64, k=100, nq_parity=256, dtype="float32", round_to_fp16=False):
    """BASELINE config 2.  Built entirely through librsb (k-means on the coarse quantizer kernels, list assignment by
    `index.add`); parity: GPU top-k vs the C oracle on the same exported index for `nq_parity` queries with the tie-aware
    comparison, every id mismatch re-scored in float64 from the stored vectors (BASELINE.md asks for identical ids: a
    mismatch is accepted only inside a group of scores closer than fp32 noise)."""
    from oracle import c_oracle as C
    from oracle import parity as P
    d = 768
    corpus = synth.Corpus(d=d, mode="gmm", n_centres=nlist // 4, device="cuda")
    t0 = time.time()
    cent = train.kmeans(corpus.train_sample(nlist * 64), nlist, niter=10, metric="ip", spherical=True)
    index = rsb.IndexIVFFlat(d, nlist, dtype=dtype)
    index.set_centroids(cent)
    for c in range(n // 1_000_000):
        x = corpus.chunk(c)
        if round_to_fp16 or dtype == "float16":       # the same fp16-representable values in both storage dtypes
            x = x.half() if dtype == "float16" else x.half().float()
        index.add(x, torch.arange(c * 1_000_000, (c + 1) * 1_000_000, device="cuda"))     # rsb_add: tensor-core assignment
        del x
    index.finalize()
    build_s = time.time() - t0
    index.nprobe = nprobe
    index.set_profiling(True)
    out = {"config": f"C2 IVF-Flat nlist={nlist} nprobe={nprobe}, {n} x {d} gmm, top-{k}, {dtype} storage",
           **card(), "index_gb": index.index_bytes / 1e9, "build_s": build_s}
    for nq in (1, 64, 2048):
        xq = corpus.queries(10_000)[:nq].contiguous()
        ms = timed(lambda: index.search_ids(xq, k), steps=3, warmup=1)
        p = index.profile()
        out[f"nq_{nq}"] = {"ms": ms, "queries_per_s": nq / ms * 1e3, "scan_ms": p["scan_ms"],
                           "scan_algorithmic_gbs": p["scan_bytes"] / p["scan_ms"] / 1e6 if p["scan_ms"] > 0 else None}
    # CPU oracle on a bounded sample of the same index exported to the host
    off, vecs, ids = index.export_lists()
    xq = corpus.queries(10_000)[:nq_parity].cpu().numpy()
    off, vecs, ids, cent_np = off.cpu().numpy(), np.asarray(vecs.cpu().numpy(), dtype=np.float32), ids.cpu().numpy(), cent.cpu().numpy()
    threads = C.set_num_threads()
    t0 = time.perf_counter()
    Dr, Ir = C.ivfflat_search(xq, cent_np, off, vecs, ids, nprobe, k)
    out["cpu_oracle_queries_per_s"] = nq_parity / (time.perf_counter() - t0)
    out["cpu_threads"] = threads
    I, D = index.search_ids(torch.from_numpy(xq).cuda(), k)
    I, D = I.cpu().numpy(), D.cpu().numpy()
    inv = np.empty(ids.max() + 1, dtype=np.int64)
    inv[ids] = np.arange(ids.shape[0])

    def score_of(q_idx, id_):            # float64 inner product with the stored vector of that id
        return np.einsum("ij,ij->i", xq[q_idx].astype(np.float64), vecs[inv[id_]].astype(np.float64))
    par = P.topk_parity(D, I, Dr, Ir, rtol=1e-5, atol=1e-5, score_of=score_of)
    qi = np.repeat(np.arange(nq_parity), k)
    s64 = score_of(qi, I.reshape(-1))
    par["rescore_max_rel_err"] = float((np.abs(s64 - D.reshape(-1)) / np.maximum(np.abs(s64), 1e-30)).max())
    out["parity"] = par
    out["ids_identical_fraction_vs_oracle"] = par["ids_equal_frac"]
    assert par["non_tie_mismatches"] == 0 and par["scores_out_of_tol"] == 0, par
    out["_sample"] = (I, D)
    return out


def c2_both(**kw):
    """C2 in fp16 and fp32 storage of the same fp16-representable vectors, one index at a time; the sampled results
    must be bit-identical."""
    import gc
    a = c2_ivfflat(dtype="float16", **kw)
    gc.collect()
    torch.cuda.empty_cache()          # the first index's workspace and the corpus chunks sit in torch's cache
    b = c2_ivfflat(dtype="float32", round_to_fp16=True, **kw)
    (Ia, Da), (Ib, Db) = a.pop("_sample"), b.pop("_sample")
    assert np.array_equal(Ia, Ib) and np.array_equal(Da, Db), "fp16 and fp32 IVF-Flat results differ"
    return {"config": "C2 fp16 vs fp32 storage", "fp16": a, "fp32": b, "fp16_fp32_bit_identical": True}


def c2_sq8(n=10_000_000, nlist=4096, nprobe=64, k=100, nq_parity=256):
    """C2's corpus (10M x 768 gmm, nlist 4096, nprobe 64, top-100) as fp16 IVF-Flat and as IVF-SQ8 with and without
    residuals (IndexIVFScalarQuantizer), one index at a time, all built from the same fp16 rows and centroids; the SQ8
    range is trained on the centroid-training sample.  Per arm: index GB, QPS, scan ms, algorithmic scan GB/s (bytes the
    scan must read: list length x row bytes, 1536 for fp16, 768 for SQ8), and the overlap of the top-100 with the fp16
    arm's top-100 for the same 2048 queries (recall@100 against fp16 IVF-Flat).  SQ8 arms: tie-aware parity with the
    IVF-SQ8 oracle (tests/ivfsq8_oracle.py) on nq_parity queries, every returned score re-scored in float64."""
    import gc
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from ivfsq8_oracle import ivfsq8_search
    from oracle import ann_oracle as O
    from oracle.sq8_oracle import sq8_decode
    d = 768
    corpus = synth.Corpus(d=d, mode="gmm", n_centres=nlist // 4, device="cuda")
    sample = corpus.train_sample(nlist * 64)
    cent = train.kmeans(sample, nlist, niter=10, metric="ip", spherical=True)
    xq_all = corpus.queries(10_000)[:2048].contiguous()
    out = {"config": f"C2 IVF-Flat fp16 vs IVF-SQ8, nlist={nlist} nprobe={nprobe}, {n} x {d} gmm, top-{k}", **card()}
    ref_I = None
    for arm in ("fp16_ivfflat", "sq8_by_residual", "sq8_no_residual"):
        t0 = time.time()
        if arm == "fp16_ivfflat":
            index = rsb.IndexIVFFlat(d, nlist, dtype="float16")
            index.set_centroids(cent)
        else:
            index = rsb.IndexIVFScalarQuantizer(d, nlist, by_residual=arm == "sq8_by_residual")
            index.set_centroids(cent)
            index.train_sq(sample.half())
        for c in range(n // 1_000_000):
            x = corpus.chunk(c).half()
            index.add(x, torch.arange(c * 1_000_000, (c + 1) * 1_000_000, device="cuda"))
            del x
        index.finalize()
        index.nprobe = nprobe
        index.set_profiling(True)
        res = {"index_gb": index.index_bytes / 1e9, "build_s": time.time() - t0}
        for nq in (1, 64, 2048):
            xq = xq_all[:nq]
            ms = timed(lambda: index.search_ids(xq, k), steps=5, warmup=2)
            p = index.profile()
            res[f"nq_{nq}"] = {"ms": ms, "queries_per_s": nq / ms * 1e3, "scan_ms": p["scan_ms"],
                               "scan_algorithmic_gbs": p["scan_bytes"] / p["scan_ms"] / 1e6 if p["scan_ms"] > 0 else None}
        I = index.search_ids(xq_all, k)[0].cpu().numpy()
        if ref_I is None:
            ref_I = I
        res["recall_at_100_vs_fp16_ivfflat"] = O.recall_at_k(I, ref_I)
        if arm != "fp16_ivfflat":
            xq = xq_all[:nq_parity]
            Ig, Dg = (t.cpu().numpy() for t in index.search_ids(xq, k))
            lists, coarse = (t.cpu().numpy() for t in index.coarse(xq, nprobe))
            off, codes, ids = (t.cpu().numpy() for t in index.export_lists())
            sq = torch.stack(index.sq_params).cpu().numpy()
            xq_np, cent_np = xq.cpu().numpy(), cent.cpu().numpy()
            t0 = time.perf_counter()
            Dr, Ir = ivfsq8_search(xq_np, cent_np, sq, off, codes, ids, nprobe, k, index.by_residual, lists=lists,
                                   coarse_dis=coarse)
            res["cpu_oracle_queries_per_s"] = nq_parity / (time.perf_counter() - t0)
            row_of = np.empty(int(ids.max()) + 1, dtype=np.int64)
            row_of[ids] = np.arange(ids.shape[0])
            list_of = np.repeat(np.arange(nlist), np.diff(off))

            def score_of(qi, id_):       # float64: <q, c_list> (by residual) + <q, decoded row>
                r = row_of[np.atleast_1d(id_)]
                x = sq8_decode(codes[r], sq).astype(np.float64)
                if index.by_residual:
                    x = x + cent_np[list_of[r]].astype(np.float64)
                return (x @ xq_np[qi].astype(np.float64)).squeeze()
            O.assert_topk_equivalent(Dg, Ig, Dr, Ir, score_of=score_of, rtol=1e-5, atol=1e-4)
            s64 = np.stack([score_of(qi, Ig[qi]) for qi in range(nq_parity)])
            res["parity"] = {"queries": nq_parity, "ids_equal_frac": float((Ig == Ir).mean()),
                             "rescore_max_abs_err": float(np.abs(s64 - Dg).max())}
            del codes
        out[arm] = res
        del index
        gc.collect()
        torch.cuda.empty_cache()
    return out


if __name__ == "__main__":
    which = sys.argv[1:] or ["c1", "c2", "c1_large"]
    if "c1" in which:
        print(json.dumps(c1_flat()), flush=True)
    if "c2" in which:
        print(json.dumps(c2_both()), flush=True)
    if "c1_large" in which:
        print(json.dumps(c1_large()), flush=True)
    if "c2_sq8" in which:
        print(json.dumps(c2_sq8()), flush=True)
