"""CPU restatement of the IVF-PQ paired scan's quantised tables (pq_lut_quant_kernel) and of the fp32 summation
order of the scan (pq_pass + pq_block_score): the fp32 score s of every vector satisfies
    s <= dis0 + base + delta * S + err + gamma * (|dis0| + amax)
for the integer sum S of its quantised entries, so the S >= S_min filter never drops a vector the exact rule keeps."""
import numpy as np
import pytest

GAMMA = 70.0 / 2.0 ** 24
F32 = np.float32


def quantise(T):
    """T [M, 256] fp32 -> (Q [M, 256] int, base, delta, err, amax) exactly as pq_lut_quant_kernel computes them."""
    lo = T.min(axis=1)
    hi = T.max(axis=1)
    rng = (hi - lo).astype(F32).max()
    delta = F32(rng / F32(1023)) if rng > 0 else F32(1)
    q = np.rint(((T - lo[:, None]).astype(F32) / delta).astype(F32))
    q = np.clip(q, 0, 1023).astype(F32)
    resid = np.abs(T.astype(np.float64) - (lo[:, None].astype(np.float64) + np.float64(delta) * q.astype(np.float64)))
    return (q.astype(np.int64), float(lo.astype(np.float64).sum()), float(delta), float(resid.max(axis=1).sum()),
            float(np.abs(T).max(axis=1).astype(np.float64).sum()))


def kernel_score(T, code, dis0, v):
    """fp32 score of block-local vector v in the scan kernel's order: K = M / 16 lanes of group g = v // K; pass
    t = v % K of lane rank r sums sub-quantizers r + K * ((g + s) & 15), s = 0..15, in two chains (even / odd s); the
    partials combine as the shuffle tree does.  The rotation by g makes the order depend on v."""
    M = T.shape[0]
    K = M // 16
    g, t = v // K, v % K
    p = []
    for r in range(K):
        s0 = s1 = None
        for s in range(16):
            m = r + K * ((g + s) & 15)
            e = T[m, code[m]]
            if s % 2 == 0:
                s0 = e if s0 is None else F32(s0 + e)
            else:
                s1 = e if s1 is None else F32(s1 + e)
        p.append(F32(s0 + s1))
    if K == 4:
        tot = F32(F32(p[t] + p[t ^ 2]) + F32(p[t ^ 1] + p[t ^ 3]))
    elif K == 2:
        tot = F32(p[t] + p[t ^ 1])
    else:
        tot = p[0]
    return F32(F32(dis0) + tot)


def check_bound(T, codes, dis0s):
    """returns the largest fp32 rounding error seen, in units of 2^-24 * (|dis0| + amax)"""
    T = T.astype(F32)
    Q, base, delta, err, amax = quantise(T)
    M = T.shape[0]
    assert Q.max() <= 1023 and M * 1023 < 2 ** 16
    worst = 0.0
    for i, (code, dis0) in enumerate(zip(codes, dis0s)):
        s = kernel_score(T, code, dis0, i % 32)
        exact = float(dis0) + float(T[np.arange(M), code].astype(np.float64).sum())
        scale = abs(float(dis0)) + amax
        if scale > 0:
            worst = max(worst, abs(float(s) - exact) / (2.0 ** -24 * scale))
        S = int(Q[np.arange(M), code].sum())
        bound = float(dis0) + base + delta * S + err + GAMMA * (abs(float(dis0)) + amax)
        assert float(s) <= bound, (float(s), bound)
        # the threshold rule: any tau the exact score reaches is reached by S >= S_min
        c0 = float(dis0) + base + err + GAMMA * (abs(float(dis0)) + amax)
        smin = max(0, int(np.floor((float(s) - c0) * (1.0 / delta)) - 1))
        assert S >= smin
    return worst


def _codes(rng, M, n):
    return rng.integers(0, 256, (n, M))


@pytest.mark.parametrize("M", [16, 32, 64])
def test_bound_random_tables(M):
    rng = np.random.default_rng(M)
    for _ in range(5):
        T = rng.standard_normal((M, 256)).astype(F32) * F32(rng.uniform(1e-3, 1e3))
        check_bound(T, _codes(rng, M, 200), rng.standard_normal(200).astype(F32))


@pytest.mark.parametrize("M", [16, 64])
def test_bound_huge_dynamic_range(M):
    rng = np.random.default_rng(100 + M)
    T = (rng.standard_normal((M, 256)) * 10.0 ** rng.uniform(-30, 30, (M, 256))).astype(F32)
    check_bound(T, _codes(rng, M, 200), (rng.standard_normal(200) * 1e20).astype(F32))


@pytest.mark.parametrize("M", [16, 32, 64])
def test_bound_constant_columns(M):
    rng = np.random.default_rng(200 + M)
    T = np.repeat(rng.standard_normal((M, 1)).astype(F32), 256, axis=1)        # R = 0
    check_bound(T, _codes(rng, M, 50), rng.standard_normal(50).astype(F32))
    T[: M // 2] = F32(-3.5)                                                    # mixed constant and varying rows
    T[M // 2:] = rng.standard_normal((M - M // 2, 256)).astype(F32)
    check_bound(T, _codes(rng, M, 50), rng.standard_normal(50).astype(F32))


@pytest.mark.parametrize("M", [32, 64])
def test_bound_negative_and_tiny_values(M):
    rng = np.random.default_rng(300 + M)
    T = -np.abs(rng.standard_normal((M, 256))).astype(F32) * F32(1e-38)      # subnormal range
    check_bound(T, _codes(rng, M, 100), (rng.standard_normal(100) * 1e-38).astype(F32))
    T = -np.abs(rng.standard_normal((M, 256))).astype(F32) - F32(1e6)
    check_bound(T, _codes(rng, M, 100), rng.standard_normal(100).astype(F32))


@pytest.mark.parametrize("M", [16, 64])
def test_bound_entries_on_rounding_boundaries(M):
    """entries at lo + (i + 1/2) * delta (and their fp32 neighbours), where rint of the fp32 quotient decides"""
    rng = np.random.default_rng(400 + M)
    lo = rng.standard_normal(M).astype(F32)
    T = np.empty((M, 256), F32)
    T[:, 0] = lo
    T[:, 1] = lo + F32(1.0)                        # range 1 => delta = 1 / 1023
    delta = F32(F32(1.0) / F32(1023))
    i = rng.integers(0, 1022, (M, 254))
    half = (lo[:, None].astype(np.float64) + (i + 0.5) * np.float64(delta)).astype(F32)
    nudge = rng.integers(-1, 2, (M, 254))
    T[:, 2:] = np.where(nudge < 0, np.nextafter(half, F32(-np.inf)), np.where(nudge > 0, np.nextafter(half, F32(np.inf)), half))
    check_bound(T, _codes(rng, M, 300), rng.standard_normal(300).astype(F32))


def test_packed_sum_has_no_carry():
    """two 16-bit lanes of M <= 64 entries of at most 1023 never carry into each other"""
    a = np.full(64, 1023, np.uint32)
    packed = (a | (a << 16)).sum(dtype=np.uint32)
    assert packed & 0xFFFF == 64 * 1023 and packed >> 16 == 64 * 1023


@pytest.mark.parametrize("M", [16, 32, 64])
def test_rounding_error_of_same_sign_sums(M):
    """Many same-sign entries near amax and a large |dis0|: the fp32 rounding of the kernel's order, measured against
    the fp64 sum, must reach a sizeable part of 2^-24 * (|dis0| + amax) (the tables do exercise the rounding term) and
    stay inside gamma.  The order's depth is ~12 additions, so the worst case is a few units; gamma = 70 units."""
    rng = np.random.default_rng(500 + M)
    worst = 0.0
    for _ in range(4):
        T = (1.0 + rng.uniform(0, 2.0 ** -10, (M, 256))).astype(F32) * F32(rng.uniform(0.5, 2))
        dis0s = (rng.uniform(0.9, 1.1, 400) * float(T.sum(axis=1).mean())).astype(F32)
        worst = max(worst, check_bound(T, _codes(rng, M, 400), dis0s))
    assert 0.5 < worst < GAMMA * 2.0 ** 24, worst


def test_residual_can_exceed_half_step():
    """rint of the fp32 quotient (T - lo) / delta can land on the far side of a half step: the measured residual,
    not delta / 2, bounds the quantisation error."""
    rng = np.random.default_rng(600)
    over = 0
    for _ in range(20):
        T = rng.standard_normal((64, 256)).astype(F32)
        lo = T.min(axis=1)
        rng_ = (T.max(axis=1) - lo).astype(F32).max()
        delta = F32(rng_ / F32(1023))
        q = np.clip(np.rint(((T - lo[:, None]).astype(F32) / delta).astype(F32)), 0, 1023)
        resid = np.abs(T.astype(np.float64) - (lo[:, None].astype(np.float64) + np.float64(delta) * q))
        over += int((resid > np.float64(delta) / 2).sum())
    assert over > 0
