#!/usr/bin/env python
"""SURVEY §8f-2 on the host: materialising nq x k passages.  Times the reference's per-passage way (`_id2psg`,
src/indicies/ivf_pq.py:209-214: open(), seek(), readline(), json.loads() for every (query, rank)) restated here against
`index_utils.fetch_passages` (group by file, sort by offset, one open() per file) on synthetic passage shards.
    python scripts/bench_passage_fetch.py"""
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from retrieval_scaling_b200.indicies import index_utils as iu  # noqa: E402


def per_passage(pos_id_map, db_ids):                       # the reference's access pattern, one file open per passage
    out = []
    for shard, chunk in db_ids:
        path, pos = pos_id_map[int(shard)][int(chunk)]
        with open(path, "r") as f:
            f.seek(pos)
            out.append(json.loads(f.readline()))
    return out


def main():
    nshards, per_shard, nq, k = 8, 50_000, 1000, 100
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as d:
        words = ["retrieval", "scaling", "datastore", "passage", "query", "index", "token", "shard"]
        for s in range(nshards):
            with open(os.path.join(d, f"raw_passages-{s}-of-{nshards}.jsonl"), "w") as f:
                for c in range(per_shard):
                    text = " ".join(words[(c + j) % len(words)] for j in range(120))
                    f.write(json.dumps({"id": f"{s}-{c}", "text": text}) + "\n")
        t0 = time.perf_counter()
        pos = iu.get_passage_pos_ids(d, os.path.join(d, "pos.pkl"))
        t_map = time.perf_counter() - t0
        ids = list(zip(rng.integers(0, nshards, nq * k).tolist(), rng.integers(0, per_shard, nq * k).tolist()))
        t0 = time.perf_counter()
        a = per_passage(pos, ids)
        t_ref = time.perf_counter() - t0
        t0 = time.perf_counter()
        b = iu.fetch_passages(pos, ids)
        t_new = time.perf_counter() - t0
        assert a == b
        print(f"# {nshards} shards x {per_shard} passages (~0.9 kB each), {nq} queries x top-{k} = {nq * k} passages, page cache warm, "
              f"{os.cpu_count()} host cores (single thread used)")
        print(f"offset map build (once per datastore): {t_map:.2f} s")
        print(f"reference pattern (open + seek + readline + json.loads per passage): {t_ref:.2f} s = {t_ref / (nq * k) * 1e6:.1f} us / passage")
        print(f"index_utils.fetch_passages (grouped by file, sorted by offset):      {t_new:.2f} s = {t_new / (nq * k) * 1e6:.1f} us / passage")
        print(f"ratio {t_ref / t_new:.2f}x; identical records")


if __name__ == "__main__":
    main()
