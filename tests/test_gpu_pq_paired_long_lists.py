"""IVF-PQ paired scan on lists longer than a candidate buffer: the look-up loop appends the vectors that pass the
quantised-table filter as pending entries, and the block re-scores them exactly when a buffer reaches its limit and
before the item's candidates are emitted.  With the forced all-survive codebook (an unused code value with a huge
table entry) every vector of a paired item is pending for both queries, so on lists of thousands of vectors the
buffers fill, and are resolved and compacted, many times within one item.  Ids and scores must be byte-identical
to the single-item scan (RSB_PQ_SINGLE_ITEMS=1, read once per process, so each mode runs in a child process)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D, NLIST, NPROBE = 128, 16, 4
KS = (1, 10, 100, 256)


def _data(M):
    rng = np.random.default_rng(1000 + M)
    centres = rng.standard_normal((NLIST, D)).astype(np.float32)
    pick = np.repeat(np.arange(NLIST), 2000 + 100 * np.arange(NLIST))   # lists of 2000 .. 3500 vectors
    xb = (centres[pick] + 0.3 * rng.standard_normal((len(pick), D))).astype(np.float32)
    cent = centres / np.linalg.norm(centres, axis=1, keepdims=True)
    cb = (0.35 * rng.standard_normal((M, 256, D // M))).astype(np.float32)
    cb[0, 255] = 1e6                                                      # never the nearest code: huge, unused
    xq = (centres[rng.integers(0, NLIST, 1000)] + 0.3 * rng.standard_normal((1000, D))).astype(np.float32)
    same = xq.copy()
    same[1::2] = same[0::2]                                               # pairs of identical queries
    return xb, cent, cb, {"distinct": xq, "same": same}


CHILD = r"""
import json, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[1] + "/tests")
import retrieval_scaling_b200 as r
from test_gpu_pq_paired_long_lists import _data, D, NLIST, NPROBE, KS

out, prof = {}, {}
for M in (16, 32, 64):
    xb, cent, cb, queries = _data(M)
    ix = r.IndexIVFPQ(D, NLIST, M)
    ix.set_centroids(cent)
    ix.set_codebook(cb)
    ix.add(xb)
    ix.nprobe = NPROBE
    ix.set_profiling(True)
    for name, xq in queries.items():
        for nq in (7, 1000):
            for k in KS:
                D_, I_ = ix.search(xq[:nq], k)
                key = f"M{M}_{name}_nq{nq}_k{k}"
                out[key + "_D"] = D_
                out[key + "_I"] = I_
                prof[key] = ix.profile()["rescored"]
np.savez(sys.argv[2], **out)
print(json.dumps(prof))
"""


def _run(tmp_path, single):
    env = dict(os.environ)
    env.pop("RSB_PQ_SINGLE_ITEMS", None)
    if single:
        env["RSB_PQ_SINGLE_ITEMS"] = "1"
    path = str(tmp_path / ("single.npz" if single else "paired.npz"))
    res = subprocess.run([sys.executable, "-c", CHILD, ROOT, path], env=env, capture_output=True, text=True,
                         timeout=1800)
    assert res.returncode == 0, res.stderr[-4000:]
    return np.load(path), json.loads(res.stdout.strip().splitlines()[-1])


def _cand_capacity(k, slack=256):
    p = 1
    while p < k + slack:
        p <<= 1
    return p


def test_paired_scan_resolves_full_buffers_mid_item_bit_identically(tmp_path):
    # every list holds more vectors than a paired item's candidate buffer (cand_capacity(k, 256) entries)
    xb, cent, _, _ = _data(16)
    lens = np.bincount(np.argmax(xb @ cent.T, axis=1), minlength=NLIST)
    cap2 = max(_cand_capacity(k) for k in KS)
    assert lens.min() > 2 * cap2, lens

    paired, prof_p = _run(tmp_path, single=False)
    single, prof_s = _run(tmp_path, single=True)
    assert sorted(paired.files) == sorted(single.files)
    for name in paired.files:
        a, b = paired[name], single[name]
        assert a.dtype == b.dtype and a.shape == b.shape, name
        assert a.tobytes() == b.tobytes(), f"{name}: {np.count_nonzero(a != b)} entries differ"
    assert all(v == 0 for v in prof_s.values())
    for M in (16, 32, 64):
        for name in ("distinct", "same"):
            for k in KS:
                # all-survive: a paired item re-scores each of its >= lens.min() vectors for both queries, more
                # than a buffer holds; 1000 queries over 16 lists always leave some item paired
                n = prof_p[f"M{M}_{name}_nq1000_k{k}"]
                assert n >= 2 * lens.min() > 2 * _cand_capacity(k), (M, name, k, n)
