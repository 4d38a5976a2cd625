"""IVF-SQ8 on the GPU (faiss IndexIVFScalarQuantizer, QT_8bit; rsb_ivfflat_create with RSB_DTYPE_SQ8):
  * without residuals, ids and scores are torch.equal to an fp32 IndexIVFFlat holding the decoded rows in the same lists;
  * device encoding and training equal the oracle's sq8_encode / sq8_train of the rows or residuals, byte for byte, and
    the lists are the ones IVF-Flat assigns;
  * with residuals, every score is fl32(coarse + s) with s the score of a twin without residuals holding the same codes;
  * persistence (faiss IwSq and RSB1), Indexer(storage_dtype=sq8), scan bytes, refusals.
The test codes are chosen so that every code occurs in every dimension."""
import ctypes
import os

import numpy as np
import pytest
import torch

import retrieval_scaling_b200 as rsb
from ivfsq8_oracle import ivfsq8_encode, ivfsq8_search
from oracle import ann_oracle as O
from oracle.sq8_oracle import sq8_decode, sq8_train
from retrieval_scaling_b200 import _lib

pytestmark = pytest.mark.gpu
F32 = np.float32


def _range(d, rng):
    return np.stack([rng.standard_normal(d), rng.random(d) * 2 + 0.1]).astype(F32)


def _codes(n, d, rng):
    """[n, d] uint8 codes in which every code 0..255 occurs in every dimension (n >= 256)."""
    c = rng.integers(0, 256, (n, d)).astype(np.uint8)
    for j in range(d):
        c[:256, j] = rng.permutation(256)
    return c[rng.permutation(n)]


def _lists(n, nlist, rng, empty=()):
    keep = np.array([l for l in range(nlist) if l not in empty])
    return keep[rng.integers(0, len(keep), n)].astype(np.int32)


@pytest.mark.parametrize("d,nlist,nprobe,empty", [(128, 16, 4, (3, 7)), (768, 64, 16, (0, 5, 63)), (768, 8, 8, ())])
def test_no_residual_is_bit_identical_to_fp32_ivfflat_of_the_decoded_rows(d, nlist, nprobe, empty):
    rng = np.random.default_rng(d + nlist)
    n = 6000
    sq, codes = _range(d, rng), _codes(n, d, rng)
    lists = _lists(n, nlist, rng, empty)
    ids = rng.permutation(10 * n)[:n].astype(np.int64)
    cent = rng.standard_normal((nlist, d)).astype(F32)
    ix = rsb.IndexIVFScalarQuantizer(d, nlist, by_residual=False)
    assert not ix.by_residual and not ix.is_trained
    ix.set_centroids(cent)
    assert not ix.is_trained                                   # the range is missing
    ix.sq_params = sq
    assert ix.is_trained
    ix.add_codes(codes, lists, ids)
    twin = rsb.IndexIVFFlat(d, nlist)
    twin.set_centroids(cent)
    twin.add_preassigned(sq8_decode(codes, sq), lists, ids)
    off, got_codes, got_ids = (t.cpu().numpy() for t in ix.export_lists())
    assert got_codes.dtype == np.uint8 and got_codes.shape == (n, d)
    off32, _, ids32 = (t.cpu().numpy() for t in twin.export_lists())
    assert np.array_equal(off, off32) and np.array_equal(got_ids, ids32)
    for l in empty:
        assert off[l] == off[l + 1]
    xq_all = torch.from_numpy(rng.standard_normal((1000, d)).astype(F32)).cuda()
    for nq in (1, 7, 1000):
        for k in (1, 100, 1000, 4096):
            I, D = ix.search_ids(xq_all[:nq], k, nprobe=nprobe)
            It, Dt = twin.search_ids(xq_all[:nq], k, nprobe=nprobe)
            assert torch.equal(I, It) and torch.equal(D, Dt), (nq, k)


@pytest.mark.parametrize("by_residual", [False, True])
@pytest.mark.parametrize("x_dtype", [np.float32, np.float16])
def test_device_encode_training_and_lists(by_residual, x_dtype):
    rng = np.random.default_rng(7)
    d, nlist, n = 128, 32, 5000
    cent = rng.standard_normal((nlist, d)).astype(F32)
    x = (cent[rng.integers(0, nlist, n)] + 0.5 * rng.standard_normal((n, d))).astype(x_dtype)
    ix = rsb.IndexIVFScalarQuantizer(d, nlist, by_residual=by_residual)
    ix.set_centroids(cent)
    with pytest.raises(_lib.RsbError):                          # the range is not set yet: RSB_ERR_STATE
        ix.add(x)
    ix.train_sq(x)
    flat = rsb.IndexIVFFlat(d, nlist)
    flat.set_centroids(cent)
    flat.add(x.astype(F32))
    off_f, _, ids_f = (t.cpu().numpy() for t in flat.export_lists())
    assign = np.repeat(np.arange(nlist), np.diff(off_f))[np.argsort(ids_f)]       # list of row i
    xf = x.astype(F32)
    rows = xf - cent[assign] if by_residual else xf
    sq = torch.stack(ix.sq_params).cpu().numpy()
    assert np.array_equal(sq, sq8_train(rows))                   # bit for bit
    ix.add(x)
    off, codes, ids = (t.cpu().numpy() for t in ix.export_lists())
    assert np.array_equal(off, off_f) and np.array_equal(ids, ids_f)              # the lists IVF-Flat assigns
    want = ivfsq8_encode(xf, cent, sq, assign, by_residual)
    assert np.array_equal(codes, want[ids])
    # add_preassigned encodes with the given lists
    pre = rsb.IndexIVFScalarQuantizer(d, nlist, by_residual=by_residual)
    pre.set_centroids(cent)
    pre.sq_params = sq
    pre.add_preassigned(x, assign)
    _, codes2, ids2 = (t.cpu().numpy() for t in pre.export_lists())
    assert np.array_equal(codes2, want[ids2])


def test_train_uses_the_lists_add_assigns():
    rng = np.random.default_rng(11)
    d, nlist, n = 64, 16, 4000
    x = rng.standard_normal((n, d)).astype(F32)
    ix = rsb.IndexIVFScalarQuantizer(d, nlist)
    assert ix.by_residual
    ix.train(x)
    assert ix.is_trained
    cent = ix.get_centroids().cpu().numpy()
    a = ix.assign(x).cpu().numpy()
    sq = torch.stack(ix.sq_params).cpu().numpy()
    assert np.array_equal(sq, sq8_train(x - cent[a]))


def _residual_pair(d=128, nlist=16, n=4000, seed=5):
    rng = np.random.default_rng(seed)
    cent = (2 * rng.standard_normal((nlist, d))).astype(F32)
    x = (cent[rng.integers(0, nlist, n)] + 0.7 * rng.standard_normal((n, d))).astype(F32)
    ix = rsb.IndexIVFScalarQuantizer(d, nlist, by_residual=True)
    ix.set_centroids(cent)
    ix.train_sq(x)
    ix.add(x)
    off, codes, ids = (t.cpu().numpy() for t in ix.export_lists())
    twin = rsb.IndexIVFScalarQuantizer(d, nlist, by_residual=False)
    twin.set_centroids(cent)
    twin.sq_params = ix.sq_params
    twin.add_codes(codes, np.repeat(np.arange(nlist), np.diff(off)), ids)
    return rng, cent, ix, twin, off, codes, ids


def test_residual_scores_are_coarse_plus_the_twin_score():
    rng, cent, ix, twin, off, codes, ids = _residual_pair()
    nq = 200
    q = torch.from_numpy(rng.standard_normal((nq, cent.shape[1])).astype(F32)).cuda()
    lists, coarse = ix.coarse(q, 1)
    k = int(np.diff(off).max())
    I, D = ix.search_preassigned(q, k, lists, coarse)
    It, Dt = twin.search_preassigned(q, k, lists, torch.zeros_like(coarse))
    I, D, It, Dt, coarse = (t.cpu().numpy() for t in (I, D, It, Dt, coarse))
    for i in range(nq):
        s_twin = {int(a): b for a, b in zip(It[i], Dt[i]) if a >= 0}
        got = {int(a): b for a, b in zip(I[i], D[i]) if a >= 0}
        assert set(got) == set(s_twin) and len(got) == off[lists[i, 0].item() + 1] - off[lists[i, 0].item()]
        for a, s in got.items():
            assert F32(s) == F32(F32(coarse[i, 0]) + F32(s_twin[a]))


def test_residual_search_matches_the_oracle():
    rng, cent, ix, twin, off, codes, ids = _residual_pair(seed=9)
    nq, k, nprobe = 1000, 100, 4
    xq = rng.standard_normal((nq, cent.shape[1])).astype(F32)
    q = torch.from_numpy(xq).cuda()
    ix.nprobe = nprobe
    I, D = (t.cpu().numpy() for t in ix.search_ids(q, k))
    lists, coarse = (t.cpu().numpy() for t in ix.coarse(q, nprobe))     # the coarse step the search runs
    sq = torch.stack(ix.sq_params).cpu().numpy()
    Dr, Ir = ivfsq8_search(xq, cent, sq, off, codes, ids, nprobe, k, True, lists=lists, coarse_dis=coarse)
    dec = sq8_decode(codes, sq).astype(np.float64)
    row_of = {int(i): r for r, i in enumerate(ids)}
    list_of = np.repeat(np.arange(cent.shape[0]), np.diff(off))

    def score_of(qi, id_):
        r = row_of[int(id_)]
        return float(xq[qi].astype(np.float64) @ (cent[list_of[r]].astype(np.float64) + dec[r]))
    O.assert_topk_equivalent(D, I, Dr, Ir, score_of=score_of, rtol=1e-5, atol=5e-4)
    for qi in range(nq):
        for j in range(k):
            if I[qi, j] >= 0:
                s64 = score_of(qi, I[qi, j])
                assert abs(D[qi, j] - s64) <= 5e-4 + 1e-5 * abs(s64)


def test_persistence_round_trips(tmp_path):
    rng, cent, ix, twin, off, codes, ids = _residual_pair(seed=13)
    ix.nprobe = 3
    q = torch.from_numpy(rng.standard_normal((50, cent.shape[1])).astype(F32)).cuda()
    I, D = ix.search_ids(q, 20)
    for fmt in ("faiss", "rsb1"):
        path = os.path.join(str(tmp_path), f"ix.{fmt}")
        rsb.write_index(ix, path, fmt=fmt)
        if fmt == "faiss":
            assert open(path, "rb").read(4) == b"IwSq"
        back = rsb.read_index(path)
        assert isinstance(back, rsb.IndexIVFScalarQuantizer) and back.by_residual and back.nprobe == 3
        I2, D2 = back.search_ids(q, 20)
        assert torch.equal(I, I2) and torch.equal(D, D2), fmt
        assert rsb.read_index(path, storage_dtype="sq8").ntotal == ix.ntotal
        for bad in ("float16", "float32"):
            with pytest.raises(ValueError, match="sq8"):
                rsb.read_index(path, storage_dtype=bad)
    flat = rsb.IndexIVFFlat(cent.shape[1], cent.shape[0])
    flat.set_centroids(cent)
    p = os.path.join(str(tmp_path), "flat.faiss")
    rsb.write_index(flat, p)
    with pytest.raises(ValueError, match="IVF-SQ8"):
        rsb.read_index(p, storage_dtype="sq8")


def test_indexer_storage_dtype_sq8(tmp_path):
    from test_gpu_indexer import _cfg, _make_datastore
    from retrieval_scaling_b200.indicies.base import Indexer
    embs, q = _make_datastore(str(tmp_path))
    key = ["+datastore.index.storage_dtype=sq8"]
    index = Indexer(_cfg(str(tmp_path), "IVFFlat", "[0,1]", key))
    ix = index.datastore.index
    assert isinstance(ix, rsb.IndexIVFScalarQuantizer) and ix.by_residual and ix.ntotal == sum(len(e) for e in embs)
    path = index.datastore.index_path
    assert open(path, "rb").read(4) == b"IwSq" and os.path.exists(path + ".meta") and os.path.exists(index.datastore.trained_index_path)
    qt = torch.from_numpy(q.astype(F32)).cuda()
    I, D = index.search_ids(qt, 20)
    again = Indexer(_cfg(str(tmp_path), "IVFFlat", "[0,1]", key))
    I2, D2 = again.search_ids(qt, 20)
    assert torch.equal(I, I2) and torch.equal(D, D2)
    scores, passages, db_ids = again.search(q, 5)
    assert len(scores) == len(q) and all(len(s) == 5 for s in scores)
    # probe = ncentroids: the SQ8 ranking agrees with the exact one on most of the top 5
    _, If = O.flat_search(q.astype(F32), np.concatenate(embs).astype(F32), 5)
    got = np.array([[s * 3000 + c for s, c in row] for row in db_ids])
    assert O.recall_at_k(got, If) >= 0.8


def test_scan_bytes_are_half_of_fp16_and_refusals():
    rng = np.random.default_rng(17)
    d, nlist, n = 256, 16, 3000
    cent = rng.standard_normal((nlist, d)).astype(F32)
    x = (cent[rng.integers(0, nlist, n)] + rng.standard_normal((n, d))).astype(np.float16)
    ix = rsb.IndexIVFScalarQuantizer(d, nlist, by_residual=False)
    ix.set_centroids(cent)
    ix.train_sq(x)
    ix.add(x)
    h16 = rsb.IndexIVFFlat(d, nlist, dtype="float16")
    h16.set_centroids(cent)
    h16.add(x)
    q = torch.from_numpy(rng.standard_normal((32, d)).astype(F32)).cuda()
    for i in (ix, h16):
        i.set_profiling(True)
        i.search_ids(q, 10, nprobe=4)
    p8, p16 = ix.profile(), h16.profile()
    assert p8["scan_bytes"] > 0 and p8["scan_bytes"] * 2 == p16["scan_bytes"]
    assert ix.index_bytes < h16.index_bytes
    # by_residual cannot change once rows exist; the range neither
    with pytest.raises(_lib.RsbError):
        ix.set_option(_lib.OPT_BY_RESIDUAL, 1)
    with pytest.raises(_lib.RsbError):
        ix.sq_params = ix.sq_params
    # the option and the range belong to SQ8 IVF handles only
    with pytest.raises(ValueError):
        h16.set_option(_lib.OPT_BY_RESIDUAL, 1)
    L = _lib.lib()
    buf = torch.empty((2, d), dtype=torch.float32, device="cuda")
    assert L.rsb_get_sq_range(h16._h, ctypes.c_void_p(buf.data_ptr()), None) == _lib.RSB_ERR_INVALID
    out = ctypes.c_int64(-1)
    assert L.rsb_info(ix._h, _lib.INFO_DTYPE, ctypes.byref(out)) == 0 and out.value == _lib.RSB_DTYPE_SQ8
    # search before the range is set
    empty = rsb.IndexIVFScalarQuantizer(d, nlist)
    empty.set_centroids(cent)
    with pytest.raises(_lib.RsbError):
        empty.search_ids(q, 10)
    with pytest.raises(ValueError):
        rsb.IndexIVFScalarQuantizer(72, nlist)
    from retrieval_scaling_b200.dist import ShardedSearcher
    with pytest.raises(NotImplementedError):
        ShardedSearcher(ix, world=2, rank=0)
