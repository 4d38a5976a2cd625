"""IVF-Flat / IVF-SQ8 tiered by list (list_device_rows: lists [0, L_dev) in device memory, the rest in pinned host
memory, probed host lists copied per query batch).  The bar is torch.equal ids and scores against the all-device index
built from the same lists: every (query, list) pair is scanned once, by the same kernel on the same bytes, and merged by
the same merge.  The data are random floats, so no query has an exact score tie at its k-th place.  Also: the CPU
oracles, the build (several add batches, rsb_add's own assignment), export, files, Indexer and the refusals."""
import os
from functools import lru_cache

import numpy as np
import pytest
import torch

import retrieval_scaling_b200 as rsb
from ivfsq8_oracle import ivfsq8_search, ivfsq8_train
from oracle import ann_oracle as O
from retrieval_scaling_b200 import _lib

pytestmark = pytest.mark.gpu
F32 = np.float32
KINDS = ["float32", "float16", "sq8_res", "sq8_plain"]
N, NLIST, EMPTY = 20000, 64, (0, 5, 17, 63)
# (nq, k, nprobe); 20 000 queries span two 16 384-query batches
QUERIES = [(1, 1, 1), (7, 100, 16), (1000, 100, NLIST), (7, 4096, NLIST), (1, 4096, 16), (20000, 100, 16)]


@lru_cache(maxsize=None)
def _data(d):
    rng = np.random.default_rng(d)
    cent = rng.standard_normal((NLIST, d)).astype(F32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    keep = np.array([l for l in range(NLIST) if l not in EMPTY])
    lists = keep[rng.integers(0, len(keep), N)].astype(np.int32)
    xb = (cent[lists] + 0.3 * rng.standard_normal((N, d))).astype(np.float16)     # fp16-representable rows
    ids = rng.permutation(10 * N)[:N].astype(np.int64)
    q = (cent[rng.integers(0, NLIST, 20000)] + 0.3 * rng.standard_normal((20000, d))).astype(F32)
    return cent, lists, xb, ids, q


def _sq(kind, d):
    cent, lists, xb, _, _ = _data(d)
    return ivfsq8_train(xb, cent, lists, kind == "sq8_res")


def _make(kind, d, **tier):
    cent = _data(d)[0]
    if kind.startswith("sq8"):
        ix = rsb.IndexIVFScalarQuantizer(d, NLIST, by_residual=kind == "sq8_res", **tier)
        ix.set_centroids(cent)
        ix.sq_params = _sq(kind, d)
    else:
        ix = rsb.IndexIVFFlat(d, NLIST, dtype=kind, **tier)
        ix.set_centroids(cent)
    return ix


def _rows(kind, d):
    xb = _data(d)[2]
    return xb.astype(F32) if kind == "float32" else xb


@lru_cache(maxsize=None)
def _ref(kind, d):
    cent, lists, xb, ids, _ = _data(d)
    ix = _make(kind, d)
    ix.add_preassigned(_rows(kind, d), lists, ids)
    ix.finalize()
    return ix


def _offsets(d):
    sizes = np.bincount(_data(d)[1], minlength=NLIST)
    off = np.zeros(NLIST + 1, np.int64)
    np.cumsum(sizes, out=off[1:])
    return sizes, off


def _r_values(d):
    sizes, off = _offsets(d)
    return {"zero": 0, "mid_list": int(off[10] + sizes[10] // 2), "boundary": int(off[20]), "ntotal": N,
            "above": N + 1000}


@lru_cache(maxsize=None)
def _tiered(kind, d, R, staging=None, batches=3):
    """The same rows as _ref, added in `batches` consecutive batches (each spans the lists in random order)."""
    _, lists, xb, ids, _ = _data(d)
    ix = _make(kind, d, list_device_rows=R, staging_bytes=staging)
    ix.reserve_lists(_offsets(d)[0])
    rows = _rows(kind, d)
    for s in np.array_split(np.arange(N), batches):
        ix.add_preassigned(rows[s], lists[s], ids[s])
    return ix


def _assert_same(a, b, q, k, nprobe):
    qt = torch.from_numpy(q).cuda()
    Ia, Da = a.search_ids(qt, k, nprobe)
    Ib, Db = b.search_ids(qt, k, nprobe)
    assert torch.equal(Ia, Ib) and torch.equal(Da, Db)
    return Ia, Da


@pytest.mark.parametrize("d", [128, 768])
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("rname", ["zero", "mid_list", "boundary", "ntotal", "above"])
def test_search_equals_the_all_device_index(kind, d, rname):
    R = _r_values(d)[rname]
    t, ref = _tiered(kind, d, R), _ref(kind, d)
    sizes, off = _offsets(d)
    l_dev = int(np.searchsorted(off, R, side="right")) - 1
    assert t.ntotal == N and t.n_dev == off[l_dev] <= R
    rb = d * {"float32": 4, "float16": 2}.get(kind, 1)
    assert t.host_bytes == (N - off[l_dev]) * rb and t.index_bytes == off[l_dev] * rb + N * 8
    q = _data(d)[4]
    for nq, k, nprobe in QUERIES:
        _assert_same(t, ref, q[:nq], k, nprobe)


@pytest.mark.parametrize("kind", KINDS)
def test_staging_smaller_than_a_list_and_many_chunks(kind):
    d = 128
    ref = _ref(kind, d)
    rb = d * {"float32": 4, "float16": 2}.get(kind, 1)
    largest = int(_offsets(d)[0].max())
    q = _data(d)[4]
    for staging in (1, 3 * largest * rb // 2, 5 * largest * rb):       # 1: raised to the largest list
        t = _tiered(kind, d, 0, staging)
        for nq, k, nprobe in ((7, 100, NLIST), (1000, 100, 16), (1, 4096, NLIST)):
            _assert_same(t, ref, q[:nq], k, nprobe)


@pytest.mark.parametrize("kind", KINDS)
def test_against_the_cpu_oracle(kind):
    d, nq, k, nprobe = 128, 64, 100, 16
    t = _tiered(kind, d, _r_values(d)["mid_list"])
    q = _data(d)[4][:nq]
    I, D = t.search_ids(torch.from_numpy(q).cuda(), k, nprobe)
    off, payload, ids = (x.cpu().numpy() for x in t.export_lists())
    cent = _data(d)[0]
    if kind.startswith("sq8"):           # the GPU's coarse lists, so that both score the same (query, list) pairs
        lists, cdis = t.coarse(torch.from_numpy(q).cuda(), nprobe)
        Dr, Ir = ivfsq8_search(q, cent, _sq(kind, d), off, payload, ids, nprobe, k, kind == "sq8_res",
                               lists=lists.cpu().numpy(), coarse_dis=cdis.cpu().numpy())
    else:
        Dr, Ir = O.ivfflat_search(q, cent, off, payload.astype(F32), ids, nprobe, k)
    O.assert_topk_equivalent(D.cpu().numpy(), I.cpu().numpy(), Dr, Ir)


@pytest.mark.parametrize("kind", KINDS)
def test_search_preassigned(kind):
    d = 128
    t, ref = _tiered(kind, d, _r_values(d)["boundary"]), _ref(kind, d)
    q = torch.from_numpy(_data(d)[4][:500]).cuda()
    lists, cdis = ref.coarse(q, 16)
    lists[::7, 3] = -1                                                   # skipped probes
    Ia, Da = t.search_preassigned(q, 100, lists, cdis)
    Ib, Db = ref.search_preassigned(q, 100, lists, cdis)
    assert torch.equal(Ia, Ib) and torch.equal(Da, Db)


@pytest.mark.parametrize("kind", KINDS)
def test_export_and_files_equal_the_all_device_index(kind, tmp_path):
    d = 128
    R = _r_values(d)["mid_list"]
    t, ref = _tiered(kind, d, R, None, 5), _ref(kind, d)
    for x, y in zip(t.export_lists(), ref.export_lists()):
        assert torch.equal(x.cpu(), y.cpu())
    n_dev = t.n_dev
    for r0, n in ((0, N), (n_dev - 5, 10), (n_dev, 7), (N - 3, 3)):
        a, b = t.export_rows(r0, n), ref.export_rows(r0, n)
        assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
    assert torch.equal(t.export_rows(1, 9, out=torch.empty_like(t.export_rows(1, 9)).cuda()).cpu(), ref.export_rows(1, 9))
    pa, pb = str(tmp_path / "t.faiss"), str(tmp_path / "r.faiss")
    rsb.write_index(t, pa)
    rsb.write_index(ref, pb)
    assert open(pa, "rb").read() == open(pb, "rb").read()
    dt = "sq8" if kind.startswith("sq8") else kind
    back = rsb.read_index(pa, storage_dtype=dt, list_device_rows=R)
    assert back.tiered and back.n_dev == t.n_dev and back.host_bytes == t.host_bytes
    q = _data(d)[4]
    for nq, k, nprobe in ((7, 100, 16), (1000, 100, NLIST)):
        _assert_same(back, ref, q[:nq], k, nprobe)
    with pytest.raises(NotImplementedError, match="faiss format"):
        rsb.write_index(t, str(tmp_path / "t.rsb1"), fmt="rsb1")


@pytest.mark.parametrize("kind", ["float32", "float16", "sq8_res"])
def test_rsb_add_assigns_and_places(kind):
    """rsb_add on a reserved index assigns (and encodes) on the device as today, then places each row."""
    d = 128
    _, _, xb, ids, q = _data(d)
    rows = _rows(kind, d)
    ref = _make(kind, d)
    ref.add(rows, ids)
    lists = torch.cat([ref.assign(rows[a:a + 5000]) for a in range(0, N, 5000)]).cpu().numpy()
    t = _make(kind, d, list_device_rows=int(N * 0.4))
    t.reserve_lists(np.bincount(lists, minlength=NLIST))
    for s in np.array_split(np.arange(N), 4):
        t.add(rows[s], ids[s])
    for nq, k, nprobe in ((7, 100, 16), (1000, 100, NLIST)):
        _assert_same(t, ref, q[:nq], k, nprobe)


def test_refusals():
    d = 128
    _, lists, xb, ids, q = _data(d)
    sizes = _offsets(d)[0]
    qt = torch.from_numpy(q[:4]).cuda()
    t = _make("float16", d, list_device_rows=1000)
    with pytest.raises(ValueError, match="reserve_lists"):                       # add without a reservation
        t.add_preassigned(xb[:10], lists[:10])
    with pytest.raises(ValueError, match="negative"):
        t.reserve_lists(np.full(NLIST, -1))
    t.reserve_lists(sizes)
    with pytest.raises(_lib.RsbError, match="already reserved"):                 # a second reservation
        t.reserve_lists(sizes)
    over = np.full(int(sizes[1]) + 1, 1, np.int32)
    with pytest.raises(_lib.RsbError, match="nothing of the batch"):             # an overflowing add is refused whole
        t.add_preassigned(xb[:len(over)], over)
    assert t.ntotal == 0
    t.add_preassigned(xb[:100], lists[:100], ids[:100])
    with pytest.raises(_lib.RsbError, match=f"100 of the {N} reserved rows"):    # search before the rows have arrived
        t.search_ids(qt, 10, 4)
    with pytest.raises(_lib.RsbError, match="reserved rows"):
        t.export_lists()
    with pytest.raises(_lib.RsbError, match="reserved rows"):
        t.export_rows(0, 1)
    t2 = _tiered("float16", d, 1000)
    lt, cd = t2.coarse(qt, 4)
    tau = torch.zeros(4, dtype=torch.int32, device="cuda")
    tab = torch.tensor([tau.data_ptr()], dtype=torch.int64, device="cuda")
    with pytest.raises(NotImplementedError, match="shared thresholds"):
        t2.search_preassigned(qt, 10, lt, cd, shared_tau=(tau, tab, 1))
    from retrieval_scaling_b200.dist import ShardedSearcher
    with pytest.raises(NotImplementedError, match="tiered IVF"):
        ShardedSearcher(t2, world=1)
    pq = rsb.IndexIVFPQ(d, 16, 16)
    L = _lib.lib()
    arr = np.zeros(16, np.int64)
    assert L.rsb_reserve_lists(pq._h, arr.ctypes.data_as(__import__("ctypes").c_void_p), 0, 0, None) == _lib.RSB_ERR_INVALID
    flat = rsb.IndexFlatIP(d)
    assert L.rsb_reserve_lists(flat._h, arr.ctypes.data_as(__import__("ctypes").c_void_p), 0, 0, None) == _lib.RSB_ERR_INVALID
    untrained = rsb.IndexIVFFlat(d, NLIST, list_device_rows=0)
    with pytest.raises(_lib.RsbError, match="not trained"):
        untrained.reserve_lists(sizes)
    filled = _make("float32", d)
    filled.add_preassigned(xb[:10].astype(F32), lists[:10])
    filled.list_device_rows = 0
    with pytest.raises(_lib.RsbError, match="already added"):
        filled.reserve_lists(sizes)
    # the existing knobs still refuse IVF
    with pytest.raises(ValueError, match="Flat index"):
        t2.set_option(_lib.OPT_DEVICE_ROWS, 10)
    with pytest.raises(ValueError, match="Flat index"):
        t2.set_option(_lib.OPT_STAGING_BYTES, 1 << 20)


@pytest.mark.parametrize("dtype", ["float16", "sq8"])
def test_indexer_list_device_rows(tmp_path, dtype):
    from test_gpu_indexer import _cfg, _make_datastore
    from retrieval_scaling_b200.indicies.base import Indexer
    ra, rb = str(tmp_path / "a"), str(tmp_path / "b")
    os.makedirs(ra); os.makedirs(rb)
    _make_datastore(ra)
    _, q = _make_datastore(rb)
    key = [f"+datastore.index.storage_dtype={dtype}"]
    plain = Indexer(_cfg(ra, "IVFFlat", "[0,1]", key))
    tiered = Indexer(_cfg(rb, "IVFFlat", "[0,1]", key + ["+datastore.index.list_device_rows=2500"]))
    ix = tiered.datastore.index
    assert ix.tiered and 0 < ix.n_dev <= 2500 and ix.host_bytes > 0 and ix.ntotal == 6000
    qt = torch.from_numpy(q.astype(F32)).cuda()
    Ia, Da = plain.search_ids(qt, 20)
    Ib, Db = tiered.search_ids(qt, 20)
    assert torch.equal(Ia, Ib) and torch.equal(Da, Db)
    assert plain.search(q, 5) == tiered.search(q, 5)
    pa, pb = plain.datastore.index_path, tiered.datastore.index_path
    assert open(pa, "rb").read() == open(pb, "rb").read()
    assert open(pa + ".meta", "rb").read() == open(pb + ".meta", "rb").read()
    again = Indexer(_cfg(rb, "IVFFlat", "[0,1]", key + ["+datastore.index.list_device_rows=2500"]))
    assert again.datastore.index.tiered
    Ic, Dc = again.search_ids(qt, 20)
    assert torch.equal(Ia, Ic) and torch.equal(Da, Dc)
