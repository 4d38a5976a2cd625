"""IVF-PQ paired scan (two queries of a list per item, packed 10-bit tables, exact fp32 re-score of the survivors)
against the single-item scan, which RSB_PQ_SINGLE_ITEMS=1 selects.  The switch is read once per process, so each
mode runs in a child process on the same seeded index and queries; ids and scores must be byte-identical.

The forced all-survive index gives one sub-quantizer a code value no vector uses whose table entries are huge: the
quantisation step becomes so coarse that every vector passes the filter, so every score the search returns comes
from the per-vector exact re-score (pq_vector_score) -- for K = 1, 2, 4 -- and must equal pq_block_score's bits."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

CHILD = r"""
import json, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import retrieval_scaling_b200 as r

out, prof = {}, {}
for M in (16, 32, 64):
    for forced in (False, True):
        rng = np.random.default_rng(M + 7 * forced)
        d, nlist = 128, 160
        centres = rng.standard_normal((nlist, d)).astype(np.float32)
        pick = np.repeat(np.arange(nlist), np.arange(nlist) % 34)      # lists of 0..33 vectors
        xb = (centres[pick] + 0.3 * rng.standard_normal((len(pick), d))).astype(np.float32)
        cent = centres / np.linalg.norm(centres, axis=1, keepdims=True)
        cb = (0.35 * rng.standard_normal((M, 256, d // M))).astype(np.float32)
        if forced:
            cb[0, 255] = 1e6                                           # never the nearest code: a huge, unused entry
        ix = r.IndexIVFPQ(d, nlist, M)
        ix.set_centroids(cent)
        ix.set_codebook(cb)
        ix.add(xb)
        ix.nprobe = 16
        xq = (centres[rng.integers(0, nlist, 10000)] + 0.3 * rng.standard_normal((10000, d))).astype(np.float32)
        xq[1::2] = xq[0::2]                                            # pairs of identical queries
        ix.set_profiling(True)
        for nq in (1, 7, 1000, 10000):
            for k in (1, 10, 100, 4096):
                if k == 4096 and nq == 10000:
                    continue                                           # 490 MB of results: covered by nq = 1000
                D, I = ix.search(xq[:nq], k)
                key = f"M{M}_f{int(forced)}_nq{nq}_k{k}"
                out[key + "_D"] = D
                out[key + "_I"] = I
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


def test_paired_scan_is_bit_identical_to_single_item_scan(tmp_path):
    paired, prof_p = _run(tmp_path, single=False)
    single, prof_s = _run(tmp_path, single=True)
    assert sorted(paired.files) == sorted(single.files)
    for name in paired.files:
        a, b = paired[name], single[name]
        assert a.dtype == b.dtype and a.shape == b.shape, name
        assert a.tobytes() == b.tobytes(), f"{name}: {np.count_nonzero(a != b)} entries differ"
    # the single-item scan never re-scores; the paired scan does wherever two queries share a list
    assert all(v == 0 for v in prof_s.values())
    for M in (16, 32, 64):
        # forced all-survive: every vector of a paired item is re-scored, for each K = M / 16.  Paired items need
        # both queries' bounds, and the lists hold at most 33 vectors, so k = 1 pairs most: of 10000 queries x 16
        # lists (~260 k vectors) most are scanned in paired items, far more than the 10 000 results returned.
        assert prof_p[f"M{M}_f1_nq10000_k1"] > 10000, prof_p
        assert all(prof_p[f"M{M}_f1_nq1_k{k}"] == 0 for k in (1, 10, 100, 4096))   # one query: nothing to pair
