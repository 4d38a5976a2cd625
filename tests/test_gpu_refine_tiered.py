"""Tiered re-rank store on the GPU (IndexRefine(device_rows=...), rsb_refine / rsb_search_refine with n_dev < ntotal):
results byte-identical to the all-device store for every split of the rows, the host-row de-duplication counts, ragged
query chunks, padding and out-of-range candidates, refusal of host tiers a kernel cannot read, parity with the CPU
oracle, and the Indexer(cfg) integration with `refine_device_rows`."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from oracle import ann_oracle as O
from oracle import refine_oracle as R

pytestmark = pytest.mark.gpu
N, NLIST, NQ = 6000, 16, 1000
M_OF = {64: 16, 768: 64}
SPLITS = ("0", "1", "half", "n-1", "n")


def _n_dev(split):
    return {"0": 0, "1": 1, "half": N // 2, "n-1": N - 1, "n": N}[split]


_DATA, _FULL, _TIER = {}, {}, {}


def _data(d):
    if d not in _DATA:
        rng = np.random.default_rng(d)
        centres = rng.standard_normal((NLIST, d)).astype(np.float32)
        xb = (centres[rng.integers(0, NLIST, N)] + 0.5 * rng.standard_normal((N, d))).astype(np.float16)
        xq = (centres[rng.integers(0, NLIST, NQ)] + 0.5 * rng.standard_normal((NQ, d))).astype(np.float32)
        cent = centres / np.linalg.norm(centres, axis=1, keepdims=True)
        cb = (0.5 * rng.standard_normal((M_OF[d], 256, d // M_OF[d]))).astype(np.float32)
        _DATA[d] = (xb, xq, cent, cb)
    return _DATA[d]


def _base(d):
    import retrieval_scaling_b200 as rsb
    key = ("base", d)
    if key not in _FULL:
        xb, _, cent, cb = _data(d)
        base = rsb.IndexIVFPQ(d, NLIST, M_OF[d], 8)
        base.set_centroids(cent)
        base.set_codebook(cb)
        base.add(xb.astype(np.float32))
        base.nprobe = 8
        _FULL[key] = base
    return _FULL[key]


def _full(d, dtype):
    import retrieval_scaling_b200 as rsb
    if (d, dtype) not in _FULL:
        ref = rsb.IndexRefine(_base(d), store_dtype=dtype)
        ref.add_store(_data(d)[0])
        _FULL[(d, dtype)] = ref
    return _FULL[(d, dtype)]


def _tier(d, dtype, n_dev):
    import retrieval_scaling_b200 as rsb
    if (d, dtype, n_dev) not in _TIER:
        ref = rsb.IndexRefine(_base(d), store_dtype=dtype, device_rows=n_dev)
        ref.add_store(_data(d)[0])
        assert ref.n_dev == n_dev and ref.host_store.shape[0] == N - n_dev
        _TIER[(d, dtype, n_dev)] = ref
    return _TIER[(d, dtype, n_dev)]


def _per_query(ref, k_base):
    return k_base * ref.d * ref._store.element_size()


def _same(a, b):
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize("split", SPLITS)
@pytest.mark.parametrize("k,k_factor", [(1, 1), (10, 8), (100, 8), (100, 40)])
@pytest.mark.parametrize("nq", [1, 7, 1000])
@pytest.mark.parametrize("d", [64, 768])
@pytest.mark.parametrize("dtype", ["float16", "float32"])
def test_tiered_is_byte_identical_to_the_device_store(dtype, d, nq, k, k_factor, split):
    full, tier = _full(d, dtype), _tier(d, dtype, _n_dev(split))
    q = torch.from_numpy(_data(d)[1][:nq]).cuda()
    _same(full.search_ids(q, k, k_factor=k_factor), tier.search_ids(q, k, k_factor=k_factor))
    Ib, _ = full.base.search_ids(q, k * k_factor)
    want = full.rerank(q, Ib, k)
    _same(want, tier.rerank(q, Ib, k))
    _same(want, tier.rerank(q, Ib, k, staging_bytes=3 * _per_query(tier, k * k_factor)))     # ragged chunks


def test_duplicates_cross_pcie_once_per_chunk():
    """Every query gets the same k' host-tier candidates: one chunk gathers k' rows, one query per chunk nq * k'."""
    tier, full = _tier(768, "float16", N // 2), _full(768, "float16")
    nq, kb, k = 7, 800, 100
    rng = np.random.default_rng(5)
    cand = torch.from_numpy(np.tile(rng.choice(np.arange(N // 2, N), kb, replace=False), (nq, 1))).cuda()
    q = torch.from_numpy(_data(768)[1][:nq]).cuda()
    for staging, want_rows in ((nq * _per_query(tier, kb), kb), (_per_query(tier, kb), nq * kb)):
        rows = torch.zeros(1, dtype=torch.int64, device="cuda")
        _same(full.rerank(q, cand, k), tier.rerank(q, cand, k, staging_bytes=staging, host_rows=rows))
        assert int(rows.item()) == want_rows
    rows = torch.zeros(1, dtype=torch.int64, device="cuda")
    tier.search_ids(q, 10, k_factor=8, host_rows=rows)
    torch.cuda.synchronize()
    assert 0 < int(rows.item()) <= nq * 80


def test_straddling_padding_and_out_of_range_candidates():
    """Candidates on both sides of n_dev, ids -1 and >= ntotal, a row of padding only; staging of exactly one query
    and of three queries with nq = 7 (ragged last chunk)."""
    tier, full = _tier(64, "float32", N // 2), _full(64, "float32")
    nq, kb, k = 7, 64, 10
    rng = np.random.default_rng(9)
    c = rng.integers(N // 2 - 40, N // 2 + 40, (nq, kb))                  # straddles n_dev, with repeats
    c[0, ::5] = -1
    c[1, ::7] = N + rng.integers(0, 1000, c[1, ::7].shape)                 # ids >= ntotal are skipped
    c[2, :] = -1                                                           # padding only
    c[3, kb // 2:] = -1
    cand = torch.from_numpy(c).cuda()
    q = torch.from_numpy(_data(64)[1][:nq]).cuda()
    want = full.rerank(q, cand, k)
    assert (want[0][2] == -1).all() and (want[1][2] == np.finfo(np.float32).min).all()
    host = {int(x) for x in c.ravel() if N // 2 <= x < N}
    for staging in (_per_query(tier, kb), 3 * _per_query(tier, kb), 64 << 20):
        rows = torch.zeros(1, dtype=torch.int64, device="cuda")
        _same(want, tier.rerank(q, cand, k, staging_bytes=staging, host_rows=rows))
        if staging == 64 << 20:
            assert int(rows.item()) == len(host)
    with pytest.raises(ValueError, match="staging_bytes"):
        tier.rerank(q, cand, k, staging_bytes=_per_query(tier, kb) - 16)


def test_rsb_refine_refuses_unreadable_host_tiers_before_any_launch():
    from retrieval_scaling_b200 import _lib
    from retrieval_scaling_b200.index import _ptr, _stream
    L = _lib.lib()
    d, nq, kb, k = 64, 4, 32, 8
    full = _full(d, "float32")
    q = torch.from_numpy(_data(d)[1][:nq]).cuda()
    cand = torch.arange(nq * kb, dtype=torch.int64, device="cuda").reshape(nq, kb)
    D = torch.full((nq, k), 7.0, device="cuda")
    I = torch.full((nq, k), 7, dtype=torch.int64, device="cuda")
    rows = torch.zeros(1, dtype=torch.int64, device="cuda")
    ws = torch.empty(L.rsb_refine_workspace_bytes(nq, kb, k, d, _lib.RSB_DTYPE_F32, 0, N, 1 << 20), dtype=torch.uint8,
                     device="cuda")
    pageable = np.zeros((N, d), np.float32)
    device_mem = torch.zeros((N, d), device="cuda")
    for host in (ctypes.c_void_p(pageable.ctypes.data), _ptr(device_mem)):
        rc = L.rsb_refine(_ptr(q), nq, None, 0, host, _lib.RSB_DTYPE_F32, None, d, N, _ptr(cand), kb, k, _ptr(D), _ptr(I),
                          _ptr(ws), ws.numel(), 1 << 20, _ptr(rows), _stream())
        assert rc == _lib.RSB_ERR_INVALID, L.rsb_last_error()
        assert b"host tier" in L.rsb_last_error()
    torch.cuda.synchronize()
    assert (D == 7.0).all() and (I == 7).all() and int(rows.item()) == 0            # no kernel ran
    _same(full.rerank(q, cand, k), _tier(d, "float32", 0).rerank(q, cand, k))       # and the library still works


@pytest.mark.parametrize("split", ["0", "half"])
@pytest.mark.parametrize("dtype", ["float16", "float32"])
def test_oracle_parity_through_store_rows(dtype, split):
    d, nq, k, kf = 768, 64, 20, 8
    tier = _tier(d, dtype, _n_dev(split))
    xb, xq, _, _ = _data(d)
    rows = tier.store_rows(np.arange(N)).cpu().numpy()
    assert np.array_equal(rows.astype(np.float32), xb.astype(np.float32))      # both tiers hold the added rows
    q = torch.from_numpy(xq[:nq]).cuda()
    I, Dd = tier.search_ids(q, k, k_factor=kf)
    Ib, _ = tier.base.search_ids(q, k * kf)
    Do, Io = R.refine_candidates(xq[:nq], rows, Ib.cpu().numpy(), k, dtype=np.float64)
    score_of = lambda qi, i: float(rows[i].astype(np.float64) @ xq[qi].astype(np.float64))   # noqa: E731
    O.assert_topk_equivalent(Dd.cpu().numpy(), I.cpu().numpy(), Do, Io, score_of=score_of, rtol=1e-5, atol=1e-5)


def test_store_growth_and_the_store_views():
    import retrieval_scaling_b200 as rsb
    xb = _data(64)[0]
    ref = rsb.IndexRefine(_base(64), store_dtype="float16", device_rows=1000)
    for a in range(0, N, 1700):                                            # grows both tiers several times
        ref.add_store(xb[a:a + 1700])
    assert ref.n_dev == 1000 and ref.host_store.shape == (N - 1000, 64) and ref.host_store.device.type == "cpu"
    assert torch.equal(ref.device_store.cpu(), torch.from_numpy(xb[:1000]))
    assert torch.equal(ref.host_store, torch.from_numpy(xb[1000:]))
    with pytest.raises(ValueError, match="tiered"):
        ref.store
    with pytest.raises(IndexError):
        ref.store_rows([N])
    q = torch.from_numpy(_data(64)[1][:100]).cuda()
    _same(_full(64, "float16").search_ids(q, 10, k_factor=8), ref.search_ids(q, 10, k_factor=8))


def test_indexer_refine_device_rows(tmp_path):
    """Indexer(cfg) over two fp16 shards: refine_device_rows = 0 and = half the rows give the results of no key."""
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_gpu_indexer import _cfg, _make_datastore
    from retrieval_scaling_b200.indicies.base import Indexer
    _, q = _make_datastore(str(tmp_path))
    base = ["+datastore.index.refine_k_factor=8", "datastore.index.probe=4"]
    want = Indexer(_cfg(str(tmp_path), "IVFPQ", "[0,1]", base))
    s0, _, ids0 = want.search(q, 5)
    i0, d0 = want.search_ids(q.astype(np.float32), 5)
    for rows in (0, 3000):
        ix = Indexer(_cfg(str(tmp_path), "IVFPQ", "[0,1]", base + [f"+datastore.index.refine_device_rows={rows}"]))
        ref = ix.datastore.index
        assert ref.tiered and ref.n_dev == rows and ref.host_store.shape[0] == 6000 - rows
        s, _, ids = ix.search(q, 5)
        assert ids == ids0 and np.array_equal(np.asarray(s), np.asarray(s0))
        i, dd = ix.search_ids(q.astype(np.float32), 5)
        assert torch.equal(i, i0) and torch.equal(dd, d0)
