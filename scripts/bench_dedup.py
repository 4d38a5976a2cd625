#!/usr/bin/env python
"""MinHash de-duplication of merged retrieval results on the GPU, stage by stage, on a seeded synthetic workload:
--queries queries x --docs passages of 100-250 words (a 30k-word vocabulary), a third of them near-duplicates (0-4
word edits) of an earlier passage of the same query, and one passage per query containing the query.

Per batch of --batch-queries queries: JSONL parsing of the batch (json.loads of every line, what reading a merged
file costs), host packing (UTF-8 buffer + offsets), H2D, split + hash and signature (both in rsb_minhash_signatures),
dedup (rsb_minhash_dedup), D2H of the keep flags and applying them.  Device stages are timed with CUDA events; the
split + hash / signature split of rsb_minhash_signatures comes from a torch.profiler run over the first batch.  The
CPU oracle (the reference's per-query algorithm) runs in a multiprocessing.Pool on --oracle-queries queries.
One JSON line to stdout and to --out.
"""
import argparse
import json
import multiprocessing
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def make_batch(rng, vocab, vlen, n_queries, n_docs):
    """Examples plus (bytes of shingles hashed, SHA-1 blocks) computed from the word lengths."""
    examples, sh_bytes, blocks = [], 0, 0
    for _ in range(n_queries):
        q_idx = rng.integers(0, len(vocab), 20)
        query = " ".join(vocab[q_idx])
        docs, idxs = [], []
        for d in range(n_docs):
            if d and rng.random() < 1 / 3:
                idx = idxs[rng.integers(0, len(idxs))].copy()
                e = rng.integers(0, 5)
                idx[rng.integers(0, len(idx), e)] = rng.integers(0, len(vocab), e)
            else:
                idx = rng.integers(0, len(vocab), rng.integers(100, 251))
            if d == n_docs // 2:
                idx = np.concatenate([q_idx, idx[:100]])
            idxs.append(idx)
            docs.append(" ".join(vocab[idx]))
        for idx in idxs + [q_idx]:
            c = np.concatenate([[0], np.cumsum(vlen[idx])])
            if len(idx) >= 13:
                L = c[13:] - c[:-13] + 12
                sh_bytes += int(L.sum())
                blocks += int(((L + 8) // 64 + 1).sum())
        examples.append({"raw_query": query, "ctxs": [{"id": [0, d], "retrieval text": t, "retrieval score": "1.0"}
                                                      for d, t in enumerate(docs)]})
    return examples, sh_bytes, blocks


def _oracle_one(ex):
    from oracle import minhash_oracle as M
    return M.remove_duplicates_with_minhash(ex["ctxs"], string_for_decontamination=ex["raw_query"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=10000)
    ap.add_argument("--docs", type=int, default=1000)
    ap.add_argument("--batch-queries", type=int, default=100)
    ap.add_argument("--oracle-queries", type=int, default=64)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch
    from retrieval_scaling_b200 import dedup
    assert torch.cuda.is_available(), "bench_dedup measures the GPU path and needs cuda:0"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    rng = np.random.default_rng(a.seed)
    vocab = np.array([("".join(chr(97 + c) for c in rng.integers(0, 26, rng.integers(2, 10)))) for _ in range(30000)],
                     dtype=object)
    vlen = np.array([len(w) for w in vocab])
    dev = torch.device("cuda", 0)
    stages = {k: 0.0 for k in ("jsonl_parse", "host_pack", "h2d", "signatures", "dedup", "d2h_apply", "total")}
    counts = {"texts": 0, "text_bytes": 0, "shingle_bytes": 0, "sha1_blocks": 0, "kept": 0, "passages": 0}
    prof_split = None
    first_batch = None
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    dedup.deduplicate(make_batch(np.random.default_rng(a.seed + 1), vocab, vlen, 2, 50)[0])     # module load, warm-up
    torch.cuda.synchronize()
    done = 0
    while done < a.queries:
        nq = min(a.batch_queries, a.queries - done)
        examples, shb, blk = make_batch(rng, vocab, vlen, nq, a.docs)
        if first_batch is None:
            first_batch = json.loads(json.dumps(examples[: a.oracle_queries]))
        lines = [json.dumps(ex) for ex in examples]
        t0 = time.perf_counter()
        examples = [json.loads(x) for x in lines]
        t1 = time.perf_counter()
        torch.cuda.synchronize()
        t_start = time.perf_counter()
        batch = dedup.pack_batch(examples)
        t2 = time.perf_counter()
        ev[0].record()
        buf = torch.from_numpy(batch.buf.copy()).to(dev)
        off = torch.from_numpy(batch.text_off).to(dev)
        goff = torch.from_numpy(batch.group_off).to(dev)
        ev[1].record()
        sig, nw = dedup.signatures_device(buf, off)
        ev[2].record()
        keep_dev = dedup.keep_device(sig, nw, goff)
        ev[3].record()
        keep = keep_dev.cpu().numpy().astype(bool)
        dedup.apply_keep(examples, batch, keep)
        t3 = time.perf_counter()
        stages["jsonl_parse"] += t1 - t0
        stages["host_pack"] += t2 - t_start
        stages["h2d"] += ev[0].elapsed_time(ev[1]) / 1e3
        stages["signatures"] += ev[1].elapsed_time(ev[2]) / 1e3
        stages["dedup"] += ev[2].elapsed_time(ev[3]) / 1e3
        stages["total"] += t3 - t_start
        stages["d2h_apply"] += (t3 - t_start) - (t2 - t_start) - ev[0].elapsed_time(ev[3]) / 1e3
        counts["texts"] += len(batch.text_off) - 1
        counts["text_bytes"] += int(batch.text_off[-1])
        counts["shingle_bytes"] += shb
        counts["sha1_blocks"] += blk
        counts["kept"] += sum(len(ex["ctxs"]) for ex in examples)
        counts["passages"] += nq * a.docs
        if prof_split is None:                      # kernel split of rsb_minhash_signatures, a run of its own
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                dedup.keep_device(*dedup.signatures_device(buf, off), goff)
                torch.cuda.synchronize()
            prof_split = {}
            for e in prof.key_averages():
                for k in ("minhash_split_hash_kernel", "minhash_signature_kernel", "minhash_dedup_kernel"):
                    if k in e.key:
                        prof_split[k + "_ms"] = round(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 1e3, 3)
        done += nq

    procs = min(32, os.cpu_count() or 1)
    t0 = time.perf_counter()
    with multiprocessing.Pool(procs) as pool:
        oracle_out = pool.map(_oracle_one, first_batch)
    t_oracle = time.perf_counter() - t0
    gpu_check = dedup.deduplicate(json.loads(json.dumps(first_batch)))
    parity = [ex["ctxs"] for ex in gpu_check] == oracle_out

    sig_s = stages["signatures"]
    out = {
        "gpu": smi, "queries": a.queries, "docs": a.docs, "batch_queries": a.batch_queries,
        "stage_s": {k: round(v, 4) for k, v in stages.items()},
        "per_query_ms": {k: round(1e3 * v / a.queries, 4) for k, v in stages.items()},
        "first_batch_kernel_ms": prof_split,
        "counts": counts,
        "shingle_bytes_per_s_signatures_stage": counts["shingle_bytes"] / sig_s if sig_s else None,
        "sha1_blocks_per_s_signatures_stage": counts["sha1_blocks"] / sig_s if sig_s else None,
        "oracle_pool": {"processes": procs, "queries": len(first_batch), "per_query_ms": round(1e3 * t_oracle / len(first_batch), 2)},
        "oracle_parity_on_subset": parity,
    }
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
