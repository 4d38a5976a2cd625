#!/usr/bin/env python
"""BM25 search on one GPU: a seeded Zipf corpus at the size of a real datastore shard set, long queries of the kind the
perplexity evaluation sends (the previous window's text: a few hundred distinct terms), scored by rsb_bm25_search.

  python scripts/bench_bm25.py [--n-docs 3500000] [--nq 10000] [--k 100]

Corpus: n_docs passages of --doc-tokens tokens each, terms drawn with probability proportional to (rank + 1) ** -s
over a --vocab term vocabulary; queries of --query-tokens tokens from the same distribution.  The index is built with
the device sort of BM25Index.from_tokens (the analyzer is not timed: the corpus is term ids).  Prints one JSON line:
time per batch from CUDA events, queries/s, the postings the scorer reads per query and their bytes/s against the
3.35 TB/s HBM3 data-sheet figure, the card's name and power limit read in the same run, and the numpy oracle's time
per query on a few queries for scale.  Nothing is written to the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def zipf_tokens(n, vocab, s, gen, device):
    import torch
    p = torch.arange(1, vocab + 1, dtype=torch.float64, device=device) ** -s
    cdf = torch.cumsum(p / p.sum(), 0)
    out = torch.empty(n, dtype=torch.int32, device=device)
    step = 1 << 26
    for a in range(0, n, step):
        u = torch.rand(min(step, n - a), dtype=torch.float64, device=device, generator=gen)
        out[a:a + step] = torch.searchsorted(cdf, u).clamp_(max=vocab - 1).to(torch.int32)
    return out


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        name, power, clock = (x.strip() for x in r.stdout.strip().splitlines()[0].split(","))
        return {"gpu": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:  # noqa: BLE001
        return {"gpu": "unknown", "error": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n-docs", type=int, default=3_500_000)
    ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--doc-tokens", type=int, default=200)
    ap.add_argument("--query-tokens", type=int, default=400)
    ap.add_argument("--s", type=float, default=1.0)
    ap.add_argument("--nq", type=int, default=10_000)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--oracle-queries", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()

    import torch
    from retrieval_scaling_b200 import _lib, bm25
    from oracle import bm25_oracle as O
    if not torch.cuda.is_available():
        raise SystemExit("bench_bm25 measures the GPU scorer: no CUDA device")
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev).manual_seed(a.seed)

    t0 = time.perf_counter()
    tok = zipf_tokens(a.n_docs * a.doc_tokens, a.vocab, a.s, gen, dev)
    doc_off = np.arange(a.n_docs + 1, dtype=np.int64) * a.doc_tokens
    ix = bm25.BM25Index.from_tokens(tok, doc_off, a.vocab, sort_device=dev)
    del tok
    torch.cuda.empty_cache()
    ix.to_device(dev)
    build_s = time.perf_counter() - t0

    qtok = zipf_tokens(a.nq * a.query_tokens, a.vocab, a.s, gen, dev).view(a.nq, a.query_tokens).cpu().numpy()
    queries = []
    for row in qtok:
        ids, cnt = np.unique(row, return_counts=True)
        queries.append(ix.term_query(dict(zip(ids.tolist(), cnt.tolist()))))
    q_off, q_term, q_w = bm25.pack_queries(queries)
    postings = np.add.reduceat(ix.df[q_term], q_off[:-1]) if len(q_term) else np.zeros(a.nq)
    q_off_d, q_term_d, q_w_d = (torch.as_tensor(x, device=dev) for x in (q_off, q_term, q_w))

    L = _lib.lib()
    ws = torch.empty(L.rsb_bm25_workspace_bytes(ix.n_docs, a.nq, a.k), dtype=torch.uint8, device=dev)
    D = torch.empty((a.nq, a.k), dtype=torch.float32, device=dev)
    I = torch.empty((a.nq, a.k), dtype=torch.int64, device=dev)
    stream = torch.cuda.current_stream(dev)

    def run():
        bm25._check(L.rsb_bm25_search(ix._dev["offsets"].data_ptr(), ix._dev["post"].data_ptr(), ix.n_docs,
                                      q_off_d.data_ptr(), q_term_d.data_ptr(), q_w_d.data_ptr(), a.nq, a.k,
                                      D.data_ptr(), I.data_ptr(), ws.data_ptr(), ws.numel(), stream.cuda_stream))

    run()                                                    # warm-up: module load, shared-memory attribute
    torch.cuda.synchronize()
    times = []
    for _ in range(a.iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        run()
        e1.record(stream)
        e1.synchronize()
        times.append(e0.elapsed_time(e1) / 1e3)
    best = min(times)

    # the numpy oracle on a few queries, for scale (and a spot check of the first query)
    nor = min(a.oracle_queries, a.nq)
    t1 = time.perf_counter()
    Dh, Ih = D[:nor].cpu().numpy(), I[:nor].cpu().numpy()
    agree = True
    for q in range(nor):
        t, w = queries[q]
        cnt = np.rint(w / ix.idf[t]).astype(np.int64)
        Do, Io = O.topk(O.scores_f32(ix.offsets, ix.docs, ix.tfs, ix.norms, ix.sum_len, list(zip(t, cnt))), a.k)
        agree &= bool(np.array_equal(Io, Ih[q]) and np.array_equal(Do.view(np.uint32), Dh[q].view(np.uint32)))
    oracle_s = (time.perf_counter() - t1) / max(nor, 1)

    bytes_read = 8.0 * float(postings.sum())
    out = {
        "bench": "bm25", **card(),
        "n_docs": ix.n_docs, "vocab": a.vocab, "zipf_s": a.s, "postings": int(len(ix.docs)),
        "distinct_terms_per_doc": round(len(ix.docs) / ix.n_docs, 1),
        "index_gib": round(ix.device_bytes() / 2 ** 30, 2), "build_s": round(build_s, 1),
        "nq": a.nq, "k": a.k, "distinct_terms_per_query": round(len(q_term) / a.nq, 1),
        "batch_s": round(best, 4), "batch_s_all": [round(t, 4) for t in times], "qps": round(a.nq / best, 1),
        "postings_per_query": round(float(postings.mean())), "gb_per_query": round(8.0 * float(postings.mean()) / 1e9, 4),
        "posting_bytes_per_s": round(bytes_read / best / 1e12, 3), "posting_bytes_unit": "TB/s",
        "hbm_datasheet_tb_s": 3.35, "share_of_hbm_datasheet": round(bytes_read / best / 3.35e12, 3),
        "oracle_numpy_s_per_query": round(oracle_s, 3), "oracle_agrees": agree,
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
