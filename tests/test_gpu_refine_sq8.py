"""SQ8 re-rank store on the GPU (IndexRefine(store_dtype="sq8"), rsb_sq8_train / rsb_sq8_encode / rsb_refine /
rsb_search_refine with RSB_DTYPE_SQ8): training and encoding equal to the CPU oracle bit for bit (every code occurs in
every dimension, so the decode is checked exhaustively), results byte-identical to an fp32 store holding the decoded
rows for the split-query and direct paths, k' up to 4096, padding and out-of-range candidates, every tier split, the
all-device workspace, the oracle, the IxRF + IxSQ round trip, and the Indexer(cfg) integration with
`refine_dtype=sq8`."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import ann_oracle as O
from oracle import refine_oracle as R
from oracle import sq8_oracle as S

pytestmark = pytest.mark.gpu
N, NLIST, NQ = 6000, 16, 1000
M_OF = {64: 16, 768: 64}

_DATA, _IDX = {}, {}


def _data(d):
    """Rows in a per-dimension range [lo, hi]: row 0 is lo, row 1 is hi, rows 2 .. 257 hold the middle of code
    (r + j) % 256's bin in dimension j (hi for code 255), the rest are clustered values clipped to the range."""
    if d not in _DATA:
        rng = np.random.default_rng(100 + d)
        centres = rng.standard_normal((NLIST, d)).astype(np.float32)
        xb = centres[rng.integers(0, NLIST, N)] + 0.5 * rng.standard_normal((N, d))
        lo = rng.uniform(-3.0, -1.0, d)
        hi = rng.uniform(1.0, 3.0, d)
        xb = np.clip(xb, lo, hi)
        xb[0], xb[1] = lo, hi
        c = (np.arange(256)[:, None] + np.arange(d)[None, :]) % 256
        xb[2:258] = np.where(c == 255, hi, lo + ((c + 0.5) / 255.0) * (hi - lo))
        xb = xb.astype(np.float32)
        xq = (centres[rng.integers(0, NLIST, NQ)] + 0.5 * rng.standard_normal((NQ, d))).astype(np.float32)
        cent = centres / np.linalg.norm(centres, axis=1, keepdims=True)
        cb = (0.5 * rng.standard_normal((M_OF[d], 256, d // M_OF[d]))).astype(np.float32)
        _DATA[d] = (xb, xq, cent, cb)
    return _DATA[d]


def _base(d):
    import retrieval_scaling_b200 as rsb
    if ("base", d) not in _IDX:
        xb, _, cent, cb = _data(d)
        base = rsb.IndexIVFPQ(d, NLIST, M_OF[d], 8)
        base.set_centroids(cent)
        base.set_codebook(cb)
        base.add(xb)
        base.nprobe = 8
        _IDX[("base", d)] = base
    return _IDX[("base", d)]


def _sq8(d, device_rows=None):
    import retrieval_scaling_b200 as rsb
    key = ("sq8", d, device_rows)
    if key not in _IDX:
        ref = rsb.IndexRefine(_base(d), store_dtype="sq8", device_rows=device_rows)
        ref.train_store(_data(d)[0])
        ref.add_store(_data(d)[0])
        _IDX[key] = ref
    return _IDX[key]


def _oracle_store(d):
    xb = _data(d)[0]
    sq = S.sq8_train(xb)
    return sq, S.sq8_encode(xb, sq)


def _decoded_f32(d):
    """An fp32 store holding the oracle-decoded rows: the reference every SQ8 result must equal byte for byte."""
    import retrieval_scaling_b200 as rsb
    if ("dec", d) not in _IDX:
        sq, codes = _oracle_store(d)
        ref = rsb.IndexRefine(_base(d), store_dtype="float32")
        ref.add_store(S.sq8_decode(codes, sq))
        _IDX[("dec", d)] = ref
    return _IDX[("dec", d)]


def _same(a, b):
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


@pytest.mark.parametrize("d", [64, 768])
@pytest.mark.parametrize("dtype", ["float32", "float16"])
def test_train_and_encode_equal_the_oracle(dtype, d):
    import retrieval_scaling_b200 as rsb
    x = _data(d)[0].astype(dtype)
    ref = rsb.IndexRefine(_base(d), store_dtype="sq8")
    with pytest.raises(ValueError, match="not trained"):
        ref.add_store(x[:10])
    ref.train_store(torch.from_numpy(x))
    ref.add_store(x)
    sq = S.sq8_train(x)
    vmin, vdiff = ref.sq_params
    assert np.array_equal(vmin.cpu().numpy(), sq[0]) and np.array_equal(vdiff.cpu().numpy(), sq[1])
    codes = S.sq8_encode(x, sq)
    assert all(len(np.unique(codes[:, j])) == 256 for j in range(d))        # every code in every dimension
    got = ref.store.cpu().numpy()
    assert got.dtype == np.uint8 and np.array_equal(got, codes)


@pytest.mark.parametrize("k,k_factor", [(1, 1), (10, 8), (100, 8), (100, 40), (64, 64)])
@pytest.mark.parametrize("nq", [1, 7, 1000])
@pytest.mark.parametrize("d", [64, 768])
def test_byte_identical_to_the_decoded_fp32_store(d, nq, k, k_factor):
    sq8, f32 = _sq8(d), _decoded_f32(d)
    q = torch.from_numpy(_data(d)[1][:nq]).cuda()
    _same(f32.search_ids(q, k, k_factor=k_factor), sq8.search_ids(q, k, k_factor=k_factor))
    Ib, _ = f32.base.search_ids(q, k * k_factor)
    _same(f32.rerank(q, Ib, k), sq8.rerank(q, Ib, k))


@pytest.mark.parametrize("n_dev", [0, N // 2, N])
@pytest.mark.parametrize("d", [64, 768])
def test_tiered_is_byte_identical_to_all_device(d, n_dev):
    full, tier = _sq8(d), _sq8(d, n_dev)
    assert tier.n_dev == n_dev and tier.host_store.shape[0] == N - n_dev and tier.host_store.dtype == torch.uint8
    assert np.array_equal(tier.store_rows(np.arange(N)).cpu().numpy(), full.store.cpu().numpy())
    for nq, k, kf in ((1, 10, 8), (7, 100, 8), (1000, 100, 40)):
        q = torch.from_numpy(_data(d)[1][:nq]).cuda()
        _same(full.search_ids(q, k, k_factor=kf), tier.search_ids(q, k, k_factor=kf))
        Ib, _ = full.base.search_ids(q, k * kf)
        want = full.rerank(q, Ib, k)
        _same(want, tier.rerank(q, Ib, k))
        _same(want, tier.rerank(q, Ib, k, staging_bytes=3 * k * kf * d))               # ragged chunks


def test_padding_out_of_range_and_host_rows():
    d, nq, kb, k = 64, 7, 64, 10
    full, tier, f32 = _sq8(d), _sq8(d, N // 2), _decoded_f32(d)
    rng = np.random.default_rng(9)
    c = rng.integers(N // 2 - 40, N // 2 + 40, (nq, kb))                  # straddles n_dev, with repeats
    c[0, ::5] = -1
    c[1, ::7] = N + rng.integers(0, 1000, c[1, ::7].shape)                 # ids >= ntotal are skipped
    c[2, :] = -1                                                           # padding only
    c[3, kb // 2:] = -1
    cand = torch.from_numpy(c).cuda()
    q = torch.from_numpy(_data(d)[1][:nq]).cuda()
    want = f32.rerank(q, cand, k)
    assert (want[0][2] == -1).all() and (want[1][2] == np.finfo(np.float32).min).all()
    _same(want, full.rerank(q, cand, k))
    host = {int(x) for x in c.ravel() if N // 2 <= x < N}
    for staging in (kb * d, 3 * kb * d, 64 << 20):
        rows = torch.zeros(1, dtype=torch.int64, device="cuda")
        _same(want, tier.rerank(q, cand, k, staging_bytes=staging, host_rows=rows))
        if staging == 64 << 20:
            assert int(rows.item()) == len(host)
    with pytest.raises(ValueError, match="staging_bytes"):
        tier.rerank(q, cand, k, staging_bytes=kb * d - 16)


def test_oracle_parity():
    d, nq, k, kf = 768, 64, 20, 8
    sq8 = _sq8(d)
    sq, codes = _oracle_store(d)
    dec = S.sq8_decode(codes, sq)
    xq = _data(d)[1][:nq]
    q = torch.from_numpy(xq).cuda()
    I, D = sq8.search_ids(q, k, k_factor=kf)
    Ib, _ = sq8.base.search_ids(q, k * kf)
    Do, Io = R.refine_candidates(xq, dec, Ib.cpu().numpy(), k, dtype=np.float64)
    score_of = lambda qi, i: float(dec[i].astype(np.float64) @ xq[qi].astype(np.float64))   # noqa: E731
    O.assert_topk_equivalent(D.cpu().numpy(), I.cpu().numpy(), Do, Io, score_of=score_of, rtol=1e-5, atol=1e-5)


def test_sq8_store_without_range_is_refused_before_any_launch():
    from retrieval_scaling_b200 import _lib
    from retrieval_scaling_b200.index import _ptr, _stream
    L = _lib.lib()
    sq8 = _sq8(64)
    nq, k, kf = 4, 8, 4
    q = torch.from_numpy(_data(64)[1][:nq]).cuda()
    D = torch.full((nq, k), 7.0, device="cuda")
    I = torch.full((nq, k), 7, dtype=torch.int64, device="cuda")
    ws = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
    h, st, SQ8 = sq8.base._h, _stream(), _lib.RSB_DTYPE_SQ8
    # all-device, then tiered (the host tier pointer is never read: the range is checked first)
    rcs = [L.rsb_search_refine(h, _ptr(q), nq, k, kf, 8, _ptr(sq8._store), N, None, SQ8, None, N, _ptr(D), _ptr(I),
                               _ptr(ws), ws.numel(), 0, None, st),
           L.rsb_search_refine(h, _ptr(q), nq, k, kf, 8, _ptr(sq8._store), N // 2, _ptr(sq8._store[N // 2:]), SQ8, None,
                               N, _ptr(D), _ptr(I), _ptr(ws), ws.numel(), 1 << 20, None, st)]
    for rc in rcs:
        assert rc == _lib.RSB_ERR_INVALID and b"sq_dev" in L.rsb_last_error()
    torch.cuda.synchronize()
    assert (D == 7.0).all() and (I == 7).all()


def _refine_plan_bytes(nq, k_base, k):
    """The all-device re-rank's workspace restated: partial keys and counts when a query's candidates are split over
    several CTAs (at least 256 candidates each, about four CTAs per SM in all)."""
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    nchunks = max(1, min(max(1, k_base // 256), (4 * sms + nq - 1) // nq))
    chunk = (k_base + nchunks - 1) // nchunks
    nchunks = (k_base + chunk - 1) // chunk
    return nq * nchunks * (min(k, chunk) * 8 + 4) + 16 if nchunks > 1 else 0


def test_all_device_workspace_holds_no_staging_buffer():
    """n_dev = ntotal: the SQ8 and fp16 workspace queries agree, do not depend on staging_bytes, and equal the plain
    re-rank's size (a staging buffer and its sort buffers are reserved for a tiered store only)."""
    from retrieval_scaling_b200 import _lib
    L = _lib.lib()
    F16, SQ8 = _lib.RSB_DTYPE_F16, _lib.RSB_DTYPE_SQ8
    al = lambda x: (x + 255) // 256 * 256                                  # noqa: E731
    for d in (64, 768):
        h = _base(d)._h
        for nq, k, kf in ((1, 10, 8), (64, 100, 8), (10000, 100, 8)):
            kb = k * kf
            want_search = (al(L.rsb_workspace_bytes(h, nq, kb, 8)) + al(nq * kb * 4) + al(nq * kb * 8)
                           + al(_refine_plan_bytes(nq, kb, k)))
            for sb in (0, 1 << 20, 512 << 20):
                for dt in (F16, SQ8):
                    assert L.rsb_refine_workspace_bytes(nq, kb, k, d, dt, N, N, sb) == _refine_plan_bytes(nq, kb, k)
                    assert L.rsb_search_refine_workspace_bytes(h, nq, k, kf, 8, dt, N, N, sb) == want_search
        tiered = [L.rsb_search_refine_workspace_bytes(h, 10000, 100, 8, 8, SQ8, 0, N, sb) for sb in (1 << 20, 512 << 20)]
        assert want_search < tiered[0] < tiered[1]                         # the tiered store sizes its staging buffer


def test_write_read_round_trip(tmp_path):
    import retrieval_scaling_b200 as rsb
    for rows in (None, N // 2):
        sq8 = _sq8(768, rows)
        path = str(tmp_path / f"refine_{rows}.faiss")
        rsb.write_index(sq8, path)
        back = rsb.read_index(path)
        assert back.store_dtype == "sq8" and back.k_factor == sq8.k_factor and not back.tiered
        assert torch.equal(torch.stack(back.sq_params), torch.stack(sq8.sq_params))
        assert torch.equal(back.store, _sq8(768).store)
        q = torch.from_numpy(_data(768)[1][:100]).cuda()
        _same(sq8.search_ids(q, 10), back.search_ids(q, 10))
        for dtype in ("float16", "float32"):
            with pytest.raises(ValueError, match="sq8"):
                rsb.read_index(path, refine_dtype=dtype)


def test_indexer_refine_dtype_sq8(tmp_path):
    """Indexer(cfg) over two fp16 shards with refine_dtype=sq8: the quantizer is trained on the first
    sample_train_size rows in id order; with and without refine_device_rows, and on a reload, the ids are the same."""
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_gpu_indexer import _cfg, _make_datastore
    from retrieval_scaling_b200.indicies.base import Indexer
    _, q = _make_datastore(str(tmp_path))
    base = ["+datastore.index.refine_k_factor=8", "datastore.index.probe=4", "+datastore.index.refine_dtype=sq8"]
    ix = Indexer(_cfg(str(tmp_path), "IVFPQ", "[0,1]", base))
    ref = ix.datastore.index
    assert ref.store_dtype == "sq8" and ref.store.shape[0] == ref.ntotal
    s0, _, ids0 = ix.search(q, 5)
    i0, d0 = ix.search_ids(q.astype(np.float32), 5)
    for extra in ([], ["+datastore.index.refine_device_rows=0"], ["+datastore.index.refine_device_rows=3000"]):
        again = Indexer(_cfg(str(tmp_path), "IVFPQ", "[0,1]", base + extra))          # reloads .faiss + .meta
        r = again.datastore.index
        assert torch.equal(torch.stack(r.sq_params), torch.stack(ref.sq_params))
        s, _, ids = again.search(q, 5)
        assert ids == ids0 and np.array_equal(np.asarray(s), np.asarray(s0))
        i, dd = again.search_ids(q.astype(np.float32), 5)
        assert torch.equal(i, i0) and torch.equal(dd, d0)
