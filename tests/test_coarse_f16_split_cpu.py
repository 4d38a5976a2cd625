"""The fp16 hi/lo split of the coarse quantizer's operands (split_f16_kernel, rsb_tf32.cu), restated in numpy, and the
per-product error bound the kernel comment states for the three-product form Al.Bh + Ah.Bl + Ah.Bh:

    x s = hi + lo + e,  |lo| <= u (1 + u) |x s| + d,  |e| <= u^2 |x s| + d          (u = 2^-11, d = 2^-25)
    |a b - (Ah Bh + Ah Bl + Al Bh)| <= (3 u^2 + 2 u^3 + 2 u^4) |a b| + d (1 + u + 2 u^2) (|a| + |b|) + 2 d^2

in scaled units, checked in float64 on random and adversarial rows: a wide dynamic range, one large element, all
zeros, and values at the fp16 subnormal edge after scaling.  The last test restates the candidate argument: the exact
top-nprobe is inside the approximate top-(nprobe + 8) whenever ranks nprobe and nprobe + 8 are more than twice the
row's error bound apart."""
import numpy as np
import pytest

U = 2.0 ** -11
DSUB = 2.0 ** -25


def split_f16(x):
    """split_f16_kernel: per row s = 2^(15 - e) with max |x| = f 2^e, f in [0.5, 1) (clamped to 2^+-126; 1 for a zero
    or non-finite maximum), hi = fp16(x s), lo = fp16(x s - hi) (the difference is exact in fp32)."""
    x = np.asarray(x, dtype=np.float32)
    m = np.abs(x).max(axis=1)
    _, e = np.frexp(m)
    sh = np.where((m > 0) & np.isfinite(m), np.clip(15 - e, -126, 126), 0)
    s = np.ldexp(np.float32(1), sh).astype(np.float32)
    v = x * s[:, None]                                        # exact: a power of two, no overflow below 2^15
    hi = v.astype(np.float16)
    lo = (v - hi.astype(np.float32)).astype(np.float16)
    inv = np.ldexp(np.float32(1), -sh).astype(np.float32)
    return v.astype(np.float64), hi, lo, inv


def product_bound(a, b):
    """Per-product bound of the kernel comment, a and b scaled (float64 arrays, broadcast)."""
    aa, ab = np.abs(a), np.abs(b)
    return (3 * U**2 + 2 * U**3 + 2 * U**4) * aa * ab + DSUB * (1 + U + 2 * U**2) * (aa + ab) + 2 * DSUB**2


def _rows(kind, rng, n=64, d=768):
    if kind == "normal":
        return rng.standard_normal((n, d)).astype(np.float32)
    if kind == "unit":                                        # normalised centroids, as the IVF indexes keep them
        x = rng.standard_normal((n, d))
        return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)
    if kind == "wide":                                        # magnitudes from 2^-40 to 2^10 in one row
        return (rng.choice([-1.0, 1.0], (n, d)) * 2.0 ** rng.uniform(-40, 10, (n, d))).astype(np.float32)
    if kind == "spike":                                       # one large element, the rest tiny: lo goes subnormal
        x = (1e-6 * rng.standard_normal((n, d))).astype(np.float32)
        x[np.arange(n), rng.integers(0, d, n)] = 1e3
        return x
    if kind == "zeros":
        return np.zeros((n, d), np.float32)
    if kind == "subnormal_edge":                              # x s around 2^-14 .. 2^-26: hi and lo subnormal
        x = (rng.choice([-1.0, 1.0], (n, d)) * 2.0 ** rng.uniform(-30, -12, (n, d))).astype(np.float32)
        x[:, 0] = 2.0 ** 14.5                                 # scale 1: the row maximum already in [2^14, 2^15)
        return x
    if kind == "tiny_rows":                                   # whole rows near the fp32 subnormal range
        return (1e-30 * rng.standard_normal((n, d))).astype(np.float32)
    raise ValueError(kind)


KINDS = ("normal", "unit", "wide", "spike", "zeros", "subnormal_edge", "tiny_rows")


@pytest.mark.parametrize("kind", KINDS)
def test_split_rule_and_element_bounds(kind):
    x = _rows(kind, np.random.default_rng(KINDS.index(kind)))
    v, hi, lo, inv = split_f16(x)
    assert np.isfinite(hi).all() and np.isfinite(lo).all()
    m = np.abs(v).max(axis=1)
    live = m > 0
    assert ((m[live] >= 2.0 ** 14) & (m[live] < 2.0 ** 15)).all()   # the row maximum lands just below the fp16 range
    assert (inv[~live] == 1).all()
    h64, l64 = hi.astype(np.float64), lo.astype(np.float64)
    e = v - h64 - l64
    assert (np.abs(l64) <= U * (1 + U) * np.abs(v) + DSUB).all()
    assert (np.abs(e) <= U * U * np.abs(v) + DSUB).all()
    np.testing.assert_array_equal(v * inv[:, None].astype(np.float64), x.astype(np.float64))   # the scale undoes exactly


@pytest.mark.parametrize("kind_a", KINDS)
@pytest.mark.parametrize("kind_b", ("normal", "unit", "wide", "spike", "subnormal_edge"))
def test_three_product_error_bound(kind_a, kind_b):
    rng = np.random.default_rng(100 + 10 * KINDS.index(kind_a) + KINDS.index(kind_b))
    a, ah, al, _ = split_f16(_rows(kind_a, rng, n=32))
    b, bh, bl, _ = split_f16(_rows(kind_b, rng, n=32))
    ah, al, bh, bl = (t.astype(np.float64) for t in (ah, al, bh, bl))
    # every (row of a, row of b) pair, element by element: the three products in float64 (each is exact in fp32)
    got = ah[:, None, :] * bh[None] + ah[:, None, :] * bl[None] + al[:, None, :] * bh[None]
    exact = a[:, None, :] * b[None]
    err = np.abs(exact - got)
    bound = product_bound(a[:, None, :], b[None])
    assert (err <= bound).all(), float((err - bound).max())
    # the bound is tight to within a small factor on the relative term where nothing is subnormal
    if kind_a == kind_b == "normal":
        rel = err / np.maximum(np.abs(exact), 1e-300)
        assert rel.max() > 0.25 * U * U


def test_row_bound_relative_to_row_maxima():
    """Summed over a row the absolute term is below 2^-39 of the two row maxima products: negligible next to 3 u^2."""
    rng = np.random.default_rng(7)
    a, *_ = split_f16(_rows("unit", rng, n=16))
    b, *_ = split_f16(_rows("unit", rng, n=16))
    ma, mb = np.abs(a).max(axis=1), np.abs(b).max(axis=1)
    abs_term = (DSUB * (1 + U + 2 * U**2) * (np.abs(a)[:, None, :] + np.abs(b)[None])).sum(axis=2)
    assert (abs_term <= 2.0 ** -39 * a.shape[1] * (ma[:, None] * mb[None]) * 2).all()


@pytest.mark.parametrize("seed", range(4))
def test_candidates_hold_the_exact_topk(seed):
    """Scores from the split operands (float64 sums of the three products, unscaled by inv_a inv_b), top kc =
    nprobe + 8 of them, exact re-score: the exact top-nprobe whenever the exact gap between ranks nprobe and
    nprobe + 8 exceeds twice the row's summed bound."""
    rng = np.random.default_rng(seed)
    nprobe, kc = 32, 40
    c = _rows("unit", rng, n=2048, d=128)
    q = rng.standard_normal((64, 128)).astype(np.float32)
    q[::4] = 2.0 * c[rng.integers(0, len(c), 16)]             # queries sitting on a centroid: a dominant first score
    a, ah, al, ia = split_f16(q)
    b, bh, bl, ib = split_f16(c)
    ah, al, bh, bl = (t.astype(np.float64) for t in (ah, al, bh, bl))
    approx = (ah @ bh.T + ah @ bl.T + al @ bh.T) * ia[:, None] * ib[None]
    exact = q.astype(np.float64) @ c.astype(np.float64).T
    eps = (product_bound(a[:, None, :], b[None]).sum(axis=2) * ia[:, None] * ib[None]).max(axis=1)
    assert (np.abs(approx - exact).max(axis=1) <= eps).all()
    cand = np.argsort(-approx, axis=1, kind="stable")[:, :kc]
    order = np.argsort(-exact, axis=1, kind="stable")
    srt = np.take_along_axis(exact, order, axis=1)
    for r in range(len(q)):
        if srt[r, nprobe - 1] - srt[r, kc - 1] <= 2 * eps[r]:
            continue                                          # the boundary caveat: not claimed
        rescored = cand[r][np.argsort(-exact[r, cand[r]], kind="stable")][:nprobe]
        np.testing.assert_array_equal(np.sort(rescored), np.sort(order[r, :nprobe]))
