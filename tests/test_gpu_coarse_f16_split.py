"""The IVF coarse quantizer on the fp16 hi/lo split of queries and centroids (gemm_ip_tc_kernel<true, FUSED> with a
split B operand, rsb_tf32.cu) against the 3xTF32 scorer, which Flat search over fp32 rows still uses: the same
centroids as the rows of an fp32 IndexFlatIP give the 3xTF32 candidates and the same exact fp32 re-score.

* Probed ids and scores equal the 3xTF32 path's after the exact re-score, bit for bit; where ids differ, only because
  the float64 scores of the two ids tie within the 3xTF32 error at the nprobe boundary.
* The ids are the float64 top-nprobe up to that error.
* Shapes: d 768 and 1024; nq 1 (the score-tile form), 1250 and 10 000 (the fused form); 1100 centroids (9 column
  tiles: odd, the last 76 wide), 16 250 (127 tiles, the last 122 wide) and 16 384; d = 96, where the last 64-wide K
  step is half zeros; rows whose best centroids crowd into one tile (the exhaustive path).  The profiler confirms
  which form ran.
* rsb_add's list assignment equals the nearest centroid by the 3xTF32 path's exact scores on a fixed seed."""
import os
import re
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FUSED_F16 = re.compile(r"gemm_ip_tc_kernel<true, true>")
TILE_F16 = re.compile(r"gemm_ip_tc_kernel<true, false>")
TF32 = re.compile(r"gemm_ip_tc_kernel<false, (true|false)>")


def _data(nlist, d, nq, seed):
    rng = np.random.default_rng(seed)
    cent = rng.standard_normal((nlist, d)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    xq = rng.standard_normal((nq, d)).astype(np.float32)
    xq[::5] = 3.0 * cent[rng.integers(0, nlist, len(xq[::5]))] + 0.1 * xq[::5]
    return cent, xq


def _traced(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, [e.key for e in prof.key_averages()]


def _tol(q, cent):
    """2 x the 3xTF32 bound 2^-20 sum |q_i c_i|, the row's largest such sum (cf. test_gpu_coarse_scorer)."""
    return 2.0 * 2.0 ** -20 * (np.abs(q).astype(np.float64) @ np.abs(cent).astype(np.float64).T).max(axis=1)


def _compare(cent, xq, nprobe, what):
    import retrieval_scaling_b200 as r
    ivf = r.IndexIVFFlat(cent.shape[1], len(cent))
    ivf.set_centroids(cent)
    flat = r.IndexFlatIP(cent.shape[1])                       # fp32 rows: 3xTF32 candidates + exact fp32 re-score
    flat.add(cent)
    (L, S), names = _traced(lambda: ivf.coarse(xq, nprobe))
    L, S = L.cpu().numpy(), S.cpu().numpy()
    (D, I), tnames = _traced(lambda: flat.search(xq, nprobe))
    assert not any(TF32.search(n) for n in names), what      # the coarse stage no longer runs 3xTF32
    assert any(TF32.search(n) for n in tnames), what
    diff = L != I
    same = ~diff.any(axis=1)
    assert same.mean() > 0.99, (what, same.mean())
    assert S[same].tobytes() == D[same].tobytes(), what
    assert all(len(set(row)) == nprobe for row in L.tolist()), what
    # float64 checks on every row that differs and on a sample of up to ~1000 rows
    rows = np.union1d(np.nonzero(~same)[0], np.arange(0, len(xq), max(1, len(xq) // 1000)))
    q = xq[rows]
    s64 = q.astype(np.float64) @ cent.astype(np.float64).T
    tol = _tol(q, cent)
    Lr, Ir = L[rows], I[rows]
    for r_, c_ in zip(*np.nonzero(Lr != Ir)):                 # differing ids: float64 ties at the boundary only
        a, b = s64[r_, Lr[r_, c_]], s64[r_, Ir[r_, c_]]
        assert abs(a - b) <= tol[r_], (what, rows[r_], c_, a, b)
        assert abs(a - s64[r_, Lr[r_, nprobe - 1]]) <= tol[r_], (what, rows[r_], c_)
    kth = -np.partition(-s64, nprobe - 1, axis=1)[:, nprobe - 1]
    got = np.take_along_axis(s64, Lr, axis=1)
    assert (got >= kth[:, None] - tol[:, None]).all(), what  # the float64 top-nprobe up to the boundary error
    return names


@pytest.mark.parametrize("d", (768, 1024))
@pytest.mark.parametrize("nlist", (1100, 16250, 16384))
def test_coarse_matches_3xtf32_and_float64(d, nlist):
    cent, xq = _data(nlist, d, 10000, seed=nlist + d)
    nprobe = 8 if nlist < 2048 else 32                        # the fused filter needs nprobe + 8 <= 2 per 128 columns
    for nq in (1, 1250, 10000):
        names = _compare(cent, xq[:nq], nprobe, (d, nlist, nq))
        if nq == 1 and nlist > 8192:                          # one query, many columns: the column-split score tile
            assert any(TILE_F16.search(n) for n in names), (d, nlist, nq)
        else:
            assert any(FUSED_F16.search(n) for n in names), (d, nlist, nq)


def test_coarse_partial_k_step():
    cent, xq = _data(4000, 96, 1250, seed=96)                 # K = 96: the second 64-wide K step reads 32 zero columns
    names = _compare(cent, xq, 16, "d96")
    assert any(FUSED_F16.search(n) for n in names)


def test_coarse_concentrated_rows_take_the_exhaustive_path():
    """Half of the queries have their best 30 centroids in one 128-column tile: more than the 8 candidates a tile
    emits, so the exactness check sends those rows to exact_rows_kernel; the result still equals the 3xTF32 path's
    (test_gpu_parity's concentrated case shows that such rows take that path)."""
    rng = np.random.default_rng(5)
    d, nlist, nq = 768, 4096, 256
    cent = rng.standard_normal((nlist, d)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    hot = rng.standard_normal(d).astype(np.float32)
    hot /= np.linalg.norm(hot)
    cols = 1024 + rng.permutation(128)[:30]
    cent[cols] = hot[None, :] + 0.01 * rng.standard_normal((30, d)).astype(np.float32)
    xq = rng.standard_normal((nq, d)).astype(np.float32)
    xq[::2] = 3 * hot[None, :] + 0.05 * rng.standard_normal((nq // 2, d)).astype(np.float32)
    names = _compare(cent, xq, 24, "concentrated")
    assert any(FUSED_F16.search(n) for n in names)


def test_add_assignment_is_the_exact_nearest_centroid():
    import torch
    import retrieval_scaling_b200 as r
    cent, _ = _data(16384, 768, 1, seed=11)
    rng = np.random.default_rng(12)
    x = (cent[rng.integers(0, len(cent), 40000)] + 0.3 * rng.standard_normal((40000, 768))).astype(np.float32)
    ivf = r.IndexIVFFlat(768, len(cent))
    ivf.set_centroids(cent)
    ivf.add(x)
    off, _, ids = (t.cpu().numpy() for t in ivf.export_lists())
    got = np.empty(len(x), np.int64)
    for lst in range(len(cent)):
        got[ids[off[lst]:off[lst + 1]]] = lst
    flat = r.IndexFlatIP(768)
    flat.add(cent)
    _, I = flat.search(torch.from_numpy(x).cuda(), 1)
    want = I.cpu().numpy()[:, 0]
    diff = np.nonzero(got != want)[0]
    if len(diff):
        s64 = x[diff].astype(np.float64) @ cent.astype(np.float64).T
        tol = _tol(x[diff], cent)
    for j, i in enumerate(diff):                              # a float64 tie for the nearest centroid only
        assert abs(s64[j, got[i]] - s64[j, want[i]]) <= tol[j], (i, got[i], want[i])
    assert len(diff) <= 4, len(diff)
    assert np.array_equal(got, ivf.assign(torch.from_numpy(x).cuda()).cpu().numpy())
