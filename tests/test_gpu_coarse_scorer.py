"""The persistent 3xTF32 / fp16 coarse scorer (rsb_tf32.cu) at the tile edges.

(a) The fused path (top-9 filter straight from the accumulators) returns the same coarse ids and scores, bit for bit,
    as the score-matrix path (`RSB_NO_FUSED_COARSE=1`: every score written out, then a row select), including exact
    ties from duplicated centroids (the lower column first) and rows whose best centroids crowd into one tile.  The
    shapes include ones where the fused kernel runs with an odd number of 128-column tiles (the empty second half of
    the last 256-column group), a partial last tile, and M = 1; the profiler confirms which kernel ran.
(b) The score tile itself (the unfused form): the ids it selects are the float64 top-k up to the 3xTF32 error at the
    k boundary.  The same check holds the fused arm's coarse ids to float64, so neither arm can share a wrong mainloop.
(c) (a) for the fp16 Flat form.
The switch is read when the library loads, so each arm runs in a subprocess of its own."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MS = (1, 127, 129, 1000, 4097)
# 1100: 9 column tiles (odd), the last one 76 columns wide; 4000: 32 tiles, the last 32 wide; 16250: 127 tiles (odd),
# the last 122 wide.  Below 8192 columns the fused path runs for any M; from 8192 on, for M >= 264.
NS = (100, 300, 1100, 4000, 16250, 16384)
KCS = (8, 40, 256)
DS = (64, 768)
FUSED_KERNEL = re.compile(r"gemm_ip_tc_kernel<(true|false), true>")
TILE_KERNEL = re.compile(r"gemm_ip_tc_kernel<(true|false), false>")


def _data(n, d, seed):
    rng = np.random.default_rng(seed)
    cent = rng.standard_normal((n, d)).astype(np.float32)
    src = rng.integers(0, n, n // 8)
    dst = rng.integers(0, n, n // 8)
    cent[dst] = cent[src]                                     # exact duplicates: tied scores in both orders of columns
    xq = rng.standard_normal((max(MS), d)).astype(np.float32)
    xq[::7] = 2.0 * cent[rng.choice(dst, len(xq[::7]))]       # queries whose best centroid is duplicated
    return cent, xq


def _concentrated():
    """Half of the queries have their best 30 centroids in ONE 128-column tile (cf. test_gpu_parity's case)."""
    rng = np.random.default_rng(5)
    d, nlist, nq = 64, 4096, 64
    cent = rng.standard_normal((nlist, d)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    hot = rng.standard_normal(d).astype(np.float32)
    hot /= np.linalg.norm(hot)
    cols = 1024 + rng.permutation(128)[:30]
    cent[cols] = hot[None, :] + 0.01 * rng.standard_normal((30, d)).astype(np.float32)
    xq = rng.standard_normal((nq, d)).astype(np.float32)
    xq[::2] = 3 * hot[None, :] + 0.05 * rng.standard_normal((nq // 2, d)).astype(np.float32)
    return cent, xq, cols


def _worker(out):
    """Runs every case with the library as the environment configured it; writes the results, and which form of the
    scorer kernel each case launched, to `out` (.npz)."""
    sys.path.insert(0, ROOT)
    import torch
    from torch.profiler import ProfilerActivity, profile
    import retrieval_scaling_b200 as r
    res = {}

    def traced(key, fn):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            a, b = fn()
            torch.cuda.synchronize()
        names = [e.key for e in prof.key_averages()]
        res["fused_" + key] = np.array(any(FUSED_KERNEL.search(n) for n in names))
        res["tile_" + key] = np.array(any(TILE_KERNEL.search(n) for n in names))
        return a, b

    for d in DS:
        for n in NS:
            cent, xq = _data(n, d, seed=n * 1000 + d)
            ivf = r.IndexIVFFlat(d, n)
            ivf.set_centroids(cent)
            flat = r.IndexFlatIP(d)                           # fp32 rows: the 3xTF32 score tile
            flat.add(cent)
            half = r.IndexFlatIP(d, dtype="float16")          # fp16 rows: the hi/lo fp16 scorer
            half.add(cent.astype(np.float16))
            for m in MS:
                for kc in KCS:
                    if kc > n:
                        continue
                    key = f"{m}_{n}_{kc}_{d}"
                    L, S = traced("ivf_" + key, lambda: ivf.coarse(xq[:m], kc))
                    res["ivf_ids_" + key], res["ivf_scores_" + key] = L.cpu().numpy(), S.cpu().numpy()
                    D, I = traced("f16_" + key, lambda: half.search(xq[:m], kc))
                    res["f16_ids_" + key], res["f16_scores_" + key] = I, D
                # k + 8 candidates > 2 per 128 columns (or > 256): always the score-tile form
                key = f"{m}_{n}_{d}"
                D, I = traced("flat_" + key, lambda: flat.search(xq[:m], min(300, n // 3)))
                res["flat_ids_" + key], res["flat_scores_" + key] = I, D
            del ivf, flat, half
            torch.cuda.empty_cache()
    cent, xq, _ = _concentrated()
    ivf = r.IndexIVFFlat(xq.shape[1], cent.shape[0])
    ivf.set_centroids(cent)
    for kc in (16, 24):
        L, S = traced(f"conc_{kc}", lambda: ivf.coarse(xq, kc))
        res[f"conc_ids_{kc}"], res[f"conc_scores_{kc}"] = L.cpu().numpy(), S.cpu().numpy()
    np.savez(out, **res)


def _run(tmp_path, no_fused):
    out = str(tmp_path / ("nofused.npz" if no_fused else "fused.npz"))
    env = dict(os.environ)
    env.pop("RSB_NO_FUSED_COARSE", None)
    if no_fused:
        env["RSB_NO_FUSED_COARSE"] = "1"
    r = subprocess.run([sys.executable, os.path.abspath(__file__), out], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return dict(np.load(out))


@pytest.fixture(scope="module")
def arms(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("coarse")
    return _run(tmp, False), _run(tmp, True)


def _ids_scores(res, prefix):
    keys = sorted(k[len(prefix) + 4:] for k in res if k.startswith(prefix + "ids_"))
    assert keys
    return [(k, res[f"{prefix}ids_{k}"], res[f"{prefix}scores_{k}"]) for k in keys]


def _assert_float64_topk(ids, cent, xq, what):
    """Every returned id's float64 score is at least the float64 k-th best of its row, less twice the 3xTF32 bound
    2^-20 * sum |q_i c_i| of the row's largest such sum: ids a correct score tile may select, and no others."""
    m, k = ids.shape
    assert ((ids >= 0) & (ids < len(cent))).all(), what
    assert all(len(set(row)) == k for row in ids.tolist()), what
    c64, ca = cent.astype(np.float64), np.abs(cent)
    for q0 in range(0, m, 512):
        q = xq[q0:q0 + 512]
        s = q.astype(np.float64) @ c64.T
        tol = 2.0 * 2.0 ** -20 * (np.abs(q) @ ca.T).max(axis=1)
        kth = -np.partition(-s, k - 1, axis=1)[:, k - 1]
        got = np.take_along_axis(s, ids[q0:q0 + 512], axis=1)
        short = kth[:, None] - tol[:, None] - got
        assert (short <= 0).all(), (what, q0, float(short.max()), float(tol.max()))


def test_fused_kernel_runs_at_the_edges(arms):
    fused, plain = arms
    required = [f"{m}_1100_8_{d}" for m in MS for d in DS]                    # 9 tiles: odd, last one partial
    required += [f"{m}_4000_{kc}_{d}" for m in (1, 129) for kc in (8, 40) for d in DS]
    required += [f"{m}_16250_40_{d}" for m in (1000, 4097) for d in DS]       # 127 tiles: odd, last one partial
    required += [f"{m}_16384_{kc}_{d}" for m in (1000, 4097) for kc in (8, 40) for d in DS]
    for key in required:
        for form in ("ivf", "f16"):
            assert fused[f"fused_{form}_{key}"], (form, key)
    assert fused["fused_conc_16"] and fused["fused_conc_24"]
    assert not any(plain[k] for k in plain if k.startswith("fused_"))   # the other arm never runs it
    flat = [k for k in fused if k.startswith("tile_flat_")]
    assert flat and all(fused[k] for k in flat)


def test_fused_coarse_matches_score_matrix_bit_for_bit(arms):
    fused, plain = arms
    ties = 0
    for key, ids, scores in _ids_scores(fused, "ivf_"):
        np.testing.assert_array_equal(ids, plain["ivf_ids_" + key], err_msg=key)
        assert scores.tobytes() == plain["ivf_scores_" + key].tobytes(), key
        same = scores[:, 1:] == scores[:, :-1]
        ties += int(same.sum())
        assert (ids[:, 1:][same] > ids[:, :-1][same]).all(), key   # equal scores: the lower column first
    assert ties > 0                                           # the duplicated centroids did produce exact ties


def test_fused_coarse_concentrated_rows_bit_for_bit(arms):
    fused, plain = arms
    _, _, cols = _concentrated()
    for kc in (16, 24):
        np.testing.assert_array_equal(fused[f"conc_ids_{kc}"], plain[f"conc_ids_{kc}"])
        assert fused[f"conc_scores_{kc}"].tobytes() == plain[f"conc_scores_{kc}"].tobytes()
    assert set(fused["conc_ids_16"][0].tolist()) <= set(cols.tolist())   # the row really is concentrated


def test_f16_flat_fused_matches_score_matrix_bit_for_bit(arms):
    fused, plain = arms
    for key, ids, scores in _ids_scores(fused, "f16_"):
        np.testing.assert_array_equal(ids, plain["f16_ids_" + key], err_msg=key)
        assert scores.tobytes() == plain["f16_scores_" + key].tobytes(), key


def test_score_tile_selects_the_float64_topk(arms):
    fused, _ = arms
    for d in DS:
        for n in NS:
            cent, xq = _data(n, d, seed=n * 1000 + d)
            for m in MS:
                _assert_float64_topk(fused[f"flat_ids_{m}_{n}_{d}"], cent, xq[:m], ("flat", m, n, d))


def test_fused_coarse_selects_the_float64_topk(arms):
    fused, _ = arms
    for d in DS:
        for n in NS:
            cent, xq = _data(n, d, seed=n * 1000 + d)
            for m in MS:
                for kc in KCS:
                    if kc <= n:
                        _assert_float64_topk(fused[f"ivf_ids_{m}_{n}_{kc}_{d}"], cent, xq[:m], ("ivf", m, n, kc, d))


if __name__ == "__main__":
    _worker(sys.argv[1])
