"""fp16 vector storage for Flat and IVF-Flat on the GPU (dtype="float16", datastore.index.storage_dtype):

  * IVF-Flat: ids AND scores bit-identical to the fp32 index holding the same (fp16-valued) vectors, and oracle parity;
  * Flat: the fp16 tensor-core scorer + exact fp32 re-score against the oracle, and scores bit-equal to the fp32 index
    wherever both return the same id (including the exhaustive path of the fused filter and last-bit near-duplicates);
  * past the 8 GB fp32 cliff (6M x 768) the fp16 Flat index still scores on tensor cores;
  * index_bytes, persistence (byte-identical .faiss files, read_index(storage_dtype=...), RSB1), and Indexer(cfg)."""
import os
import pickle

import numpy as np
import pytest
import torch

from oracle import ann_oracle as O

pytestmark = pytest.mark.gpu


def _rsb():
    import retrieval_scaling_b200 as rsb
    return rsb


def _fp16_data(n, d, nq, seed, ncentres=32):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((ncentres, d)).astype(np.float32)
    xb = (0.3 * (centres[rng.integers(0, ncentres, n)] + 0.5 * rng.standard_normal((n, d)))).astype(np.float16)
    xq = (centres[rng.integers(0, ncentres, nq)] + 0.5 * rng.standard_normal((nq, d))).astype(np.float32)
    return rng, xb, xq, centres


def _score_of(xq, xb):
    q64, x64 = xq.astype(np.float64), xb.astype(np.float64)
    return lambda qi, i: float(x64[i] @ q64[qi])


# ---------------------------------------------------------------------------------------------------------------
# IVF-Flat: fp16 vs fp32 on the same values
# ---------------------------------------------------------------------------------------------------------------
IVF_D, IVF_N = 128, 30000
_IVF = {}


def _ivf_pair(nlist, mode):
    """(fp16 index, fp32 index, xb, xq, centroids, ids).  mode "add": three add batches (numpy fp16, CUDA fp16, numpy
    fp32 of the same values), custom ids; mode "preassigned": add_preassigned onto the even lists only (odd lists
    stay empty), sequential ids."""
    key = (nlist, mode)
    if key not in _IVF:
        rsb = _rsb()
        rng, xb, xq, centres = _fp16_data(IVF_N, IVF_D, 1000, seed=nlist)
        cent = rng.standard_normal((nlist, IVF_D)).astype(np.float32)
        cent /= np.linalg.norm(cent, axis=1, keepdims=True)
        a = rsb.IndexIVFFlat(IVF_D, nlist, dtype="float16")
        b = rsb.IndexIVFFlat(IVF_D, nlist)
        assert a.dtype == "float16" and b.dtype == "float32"
        for ix in (a, b):
            ix.set_centroids(cent)
        if mode == "add":
            ids = (rng.permutation(IVF_N) * 3 + 7).astype(np.int64)
            cuts = [0, 9000, 21000, IVF_N]
            a.add(xb[cuts[0]:cuts[1]], ids[cuts[0]:cuts[1]])
            a.add(torch.from_numpy(xb[cuts[1]:cuts[2]]).cuda(), ids[cuts[1]:cuts[2]])
            a.add(xb[cuts[2]:].astype(np.float32), ids[cuts[2]:])                  # fp32 input, rounded exactly
            for i in range(3):
                b.add(xb[cuts[i]:cuts[i + 1]].astype(np.float32), ids[cuts[i]:cuts[i + 1]])
        else:
            ids = np.arange(IVF_N, dtype=np.int64)
            lists = (2 * rng.integers(0, nlist // 2, IVF_N)).astype(np.int32)
            a.add_preassigned(xb, lists)
            b.add_preassigned(xb.astype(np.float32), lists)
            assert (a.list_sizes().cpu().numpy()[1::2] == 0).all()
        a.finalize(); b.finalize()
        _IVF[key] = (a, b, xb, xq, cent, ids)
    return _IVF[key]


@pytest.mark.parametrize("mode", ["add", "preassigned"])
@pytest.mark.parametrize("nlist,nprobe", [(16, 4), (64, 8), (64, 64)])
@pytest.mark.parametrize("k", [1, 100, 1000, 4096])
@pytest.mark.parametrize("nq", [1, 7, 1000])
def test_ivfflat_fp16_is_bit_identical_to_fp32(mode, nlist, nprobe, k, nq):
    a, b, xb, xq, cent, ids = _ivf_pair(nlist, mode)
    q = torch.from_numpy(xq[:nq]).cuda()
    Ia, Da = a.search_ids(q, k, nprobe)
    Ib, Db = b.search_ids(q, k, nprobe)
    assert torch.equal(Ia, Ib) and torch.equal(Da, Db)
    if nq == 1000 and k in (100, 4096):               # oracle parity on the exported (natural CSR) lists
        off, vecs, eids = (t.cpu().numpy() for t in a.export_lists())
        assert vecs.dtype == np.float16
        Dr, Ir = O.ivfflat_search(xq[:nq], cent, off, vecs.astype(np.float32), eids, nprobe, k)
        pos = np.empty(int(ids.max()) + 1, dtype=np.int64)
        pos[ids] = np.arange(len(ids))
        x64 = xb.astype(np.float64)
        score_of = lambda qi, i: float(x64[pos[i]] @ xq[qi].astype(np.float64))  # noqa: E731
        O.assert_topk_equivalent(Da.cpu().numpy(), Ia.cpu().numpy(), Dr, Ir, score_of=score_of, rtol=1e-5, atol=1e-5)


def test_ivfflat_fp16_assignment_and_scan_bytes():
    """fp16 rows get the lists the fp32 quantizer assigns to their upcast values; the profiled scan counts 2-byte
    elements."""
    a, b, *_ = _ivf_pair(64, "add")
    assert torch.equal(a.list_sizes(), b.list_sizes())
    oa, _, ia = a.export_lists()
    ob, _, ib = b.export_lists()
    assert torch.equal(oa, ob) and torch.equal(ia, ib)
    q = torch.from_numpy(_ivf_pair(64, "add")[3][:64]).cuda()
    prof = {}
    for name, ix in (("a", a), ("b", b)):
        ix.set_profiling(True)
        ix.search_ids(q, 10, 8)
        prof[name] = ix.profile()
        ix.set_profiling(False)
    assert prof["a"]["scan_bytes"] > 0 and prof["a"]["scan_bytes"] * 2 == prof["b"]["scan_bytes"]


# ---------------------------------------------------------------------------------------------------------------
# Flat: fp16 tensor-core scorer
# ---------------------------------------------------------------------------------------------------------------
_FLAT = {}


def _flat_pair(n, d):
    key = (n, d)
    if key not in _FLAT:
        rsb = _rsb()
        _, xb, xq, _ = _fp16_data(n, d, 1000, seed=n + d)
        a = rsb.IndexFlatIP(d, dtype="float16")
        a.add(xb)
        b = rsb.IndexFlatIP(d)
        b.add(xb.astype(np.float32))
        Dr, Ir = O.flat_search(xq, xb.astype(np.float32), 4096)
        _FLAT[key] = (a, b, xb, xq, Dr, Ir)
    return _FLAT[key]


def _check_flat(Da, Ia, Db, Ib, k, score_of=None):
    """fp16 vs fp32 Flat on the same values: ids equal up to tie permutations, scores bit-equal where ids are equal
    (both re-score their candidates with the same fmaf sequence; the fp32 index does so for k + 8 <= 4096)."""
    O.assert_topk_equivalent(Da, Ia, Db, Ib, score_of=score_of, rtol=1e-5,
                             atol=1e-5 if k + 8 <= 4096 else 2e-5 * float(np.abs(Db[:, 0]).max()))
    same = Ia == Ib
    if k + 8 <= 4096:
        assert np.array_equal(Da[same], Db[same])


@pytest.mark.parametrize("n", [1000, 100_000])
@pytest.mark.parametrize("d", [64, 768])
@pytest.mark.parametrize("nq", [1, 7, 1000])
@pytest.mark.parametrize("k", [1, 10, 100, 1000, 4096])
def test_flat_fp16_matches_oracle_and_fp32(n, d, nq, k):
    a, b, xb, xq, Dr, Ir = _flat_pair(n, d)
    q = torch.from_numpy(xq[:nq]).cuda()
    Ia, Da = (t.cpu().numpy() for t in a.search_ids(q, k))
    Ib, Db = (t.cpu().numpy() for t in b.search_ids(q, k))
    # the oracle's BLAS adds the d products in another order than the GPU's fmaf chain: near-zero scores deep in the
    # list differ by the fp32 rounding of the large terms, so the absolute tolerance scales with the largest score
    atol = 2e-5 * float(np.abs(Dr[:nq, 0]).max())
    O.assert_topk_equivalent(Da, Ia, Dr[:nq, :k], Ir[:nq, :k], score_of=_score_of(xq, xb), rtol=1e-5, atol=atol)
    if k > n:                                                # padding
        assert (Ia[:, n:] == -1).all() and (Da[:, n:] == np.finfo(np.float32).min).all()
    _check_flat(Da, Ia, Db, Ib, k, _score_of(xq, xb))


def test_flat_fp16_concentrated_rows_take_the_exhaustive_path():
    """fp16 counterpart of the fused-filter adversarial layout: 30 near-duplicate best rows inside ONE 128-column half
    tile, so the top 8 of that half tile cannot hold the row's top 24 -- the bound check flags those rows and the fp16
    exact_rows kernel re-does them."""
    rsb = _rsb()
    rng = np.random.default_rng(5)
    d, n, nq, k = 64, 4096, 64, 16
    xb = rng.standard_normal((n, d)).astype(np.float32)
    xb /= np.linalg.norm(xb, axis=1, keepdims=True)
    hot = rng.standard_normal(d).astype(np.float32)
    hot /= np.linalg.norm(hot)
    cols = 1024 + rng.permutation(128)[:30]
    xb[cols] = hot[None, :] + 0.01 * rng.standard_normal((30, d)).astype(np.float32)
    xb = xb.astype(np.float16)
    xq = rng.standard_normal((nq, d)).astype(np.float32)
    xq[::2] = 3 * hot[None, :] + 0.05 * rng.standard_normal((nq // 2, d)).astype(np.float32)
    a = rsb.IndexFlatIP(d, dtype="float16")
    a.add(xb)
    b = rsb.IndexFlatIP(d)
    b.add(xb.astype(np.float32))
    Ia, Da = (t.cpu().numpy() for t in a.search_ids(torch.from_numpy(xq).cuda(), k))
    Ib, Db = (t.cpu().numpy() for t in b.search_ids(torch.from_numpy(xq).cuda(), k))
    Dr, Ir = O.flat_search(xq, xb.astype(np.float32), k)
    O.assert_topk_equivalent(Da, Ia, Dr, Ir, score_of=_score_of(xq, xb), rtol=1e-5, atol=1e-5)
    assert set(Ia[0].tolist()) <= set(cols.tolist())
    _check_flat(Da, Ia, Db, Ib, k)


def test_flat_fp16_near_duplicates_differing_in_the_last_bit():
    rsb = _rsb()
    rng = np.random.default_rng(9)
    d, n = 768, 5000
    xb = (0.05 * rng.standard_normal((n, d))).astype(np.float16)
    src = rng.choice(n, 200, replace=False)
    dst = (src + 1) % n
    xb[dst] = xb[src]
    col = rng.integers(0, d, 200)
    xb[dst, col] = np.nextafter(xb[dst, col], np.float16(np.inf))      # one fp16 ulp apart
    xq = xb[src[:100]].astype(np.float32)
    a = rsb.IndexFlatIP(d, dtype="float16")
    a.add(xb)
    b = rsb.IndexFlatIP(d)
    b.add(xb.astype(np.float32))
    for k in (2, 50):
        Ia, Da = (t.cpu().numpy() for t in a.search_ids(torch.from_numpy(xq).cuda(), k))
        Ib, Db = (t.cpu().numpy() for t in b.search_ids(torch.from_numpy(xq).cuda(), k))
        Dr, Ir = O.flat_search(xq, xb.astype(np.float32), k)
        O.assert_topk_equivalent(Da, Ia, Dr, Ir, score_of=_score_of(xq, xb), rtol=1e-6, atol=1e-7)
        _check_flat(Da, Ia, Db, Ib, k)


def test_flat_fp16_option_and_d_checks():
    rsb = _rsb()
    a = rsb.IndexFlatIP(768, dtype="float16")
    with pytest.raises(NotImplementedError):
        a.set_option(0, 0)                   # RSB_OPT_COARSE_TENSOR = 0: no CUDA-core fp16 path
    a.set_option(0, 1)
    with pytest.raises(NotImplementedError):
        rsb.IndexFlatIP(72, dtype="float16")
    with pytest.raises(ValueError):
        rsb.IndexFlatIP(768, dtype="bfloat16")
    e = rsb.IndexFlatIP(768, dtype="float16")                          # empty index: all padding
    I, D = e.search_ids(torch.zeros((3, 768), device="cuda"), 5)
    assert (I == -1).all()


def test_flat_fp16_past_the_fp32_cliff():
    """6M x 768: the fp32 payload (18.4 GB) is past the 8 GB limit of the 3xTF32 split, the fp16 one (9.2 GB) is the
    tensor-core operand as stored.  Launches of one search = query split + (scorer + select) + merge + re-score = 5
    (the CUDA-core form has no split and no re-score: 3).  Results match an fp64 exhaustive search on 16 queries."""
    rsb = _rsb()
    n, d, nq, k = 6_000_000, 768, 16, 100
    g = torch.Generator(device="cuda")
    g.manual_seed(3)
    a = rsb.IndexFlatIP(d, dtype="float16")
    for r0 in range(0, n, 1_000_000):
        a.add((0.05 * torch.randn((1_000_000, d), generator=g, device="cuda")).half())
    a.finalize()
    assert n * d * 4 > (8 << 30) and a.index_bytes == n * d * 2 + n * 8
    xb = a.export_lists()[1]
    q = xb[torch.arange(nq, device="cuda") * 374_999].float() + 0.01 * torch.randn((nq, d), generator=g, device="cuda")
    a.set_profiling(True)
    I, D = a.search_ids(q, k)
    prof = a.profile()
    a.set_profiling(False)
    assert prof["launches"] == 5
    S = torch.empty((nq, n), dtype=torch.float64, device="cuda")
    for r0 in range(0, n, 1_000_000):
        S[:, r0:r0 + 1_000_000] = q.double() @ xb[r0:r0 + 1_000_000].double().T
    Dr, Ir = torch.topk(S, k, dim=1)
    Sn = S.cpu().numpy()
    O.assert_topk_equivalent(D.cpu().numpy(), I.cpu().numpy(), Dr.float().cpu().numpy(), Ir.cpu().numpy(),
                             score_of=lambda qi, i: float(Sn[qi, i]), rtol=1e-5, atol=1e-5)


# ---------------------------------------------------------------------------------------------------------------
# footprint and persistence
# ---------------------------------------------------------------------------------------------------------------
def test_index_bytes_halve_the_payload():
    rsb = _rsb()
    _, xb, _, _ = _fp16_data(10000, 128, 1, seed=1)
    a = rsb.IndexFlatIP(128, dtype="float16"); a.add(xb); a.finalize()
    b = rsb.IndexFlatIP(128); b.add(xb); b.finalize()
    assert b.index_bytes == 10000 * 128 * 4 + 10000 * 8 and a.index_bytes == 10000 * 128 * 2 + 10000 * 8
    c, e, *_ = _ivf_pair(16, "add")
    assert c.index_bytes == IVF_N * IVF_D * 2 + IVF_N * 8 and e.index_bytes == IVF_N * IVF_D * 4 + IVF_N * 8


def test_persistence(tmp_path):
    rsb = _rsb()
    c, e, xb, xq, cent, ids = _ivf_pair(16, "preassigned")      # sequential ids: both index kinds have a faiss form
    a = rsb.IndexFlatIP(IVF_D, dtype="float16"); a.add(xb)
    b = rsb.IndexFlatIP(IVF_D); b.add(xb.astype(np.float32))
    q = torch.from_numpy(xq[:100]).cuda()
    for name, (ix16, ix32) in {"flat": (a, b), "ivf": (c, e)}.items():
        ix16.nprobe = ix32.nprobe = 4
        p16, p32 = (os.path.join(str(tmp_path), f"{name}_{t}.faiss") for t in ("16", "32"))
        rsb.write_index(ix16, p16)
        rsb.write_index(ix32, p32)
        assert open(p16, "rb").read() == open(p32, "rb").read()          # upcast to fp32: the fp32 index's file
        back = rsb.read_index(p32, storage_dtype="float16")
        assert back.dtype == "float16" and back.ntotal == ix16.ntotal
        I0, D0 = ix16.search_ids(q, 50)
        I1, D1 = back.search_ids(q, 50)
        assert torch.equal(I0, I1) and torch.equal(D0, D1)
        assert rsb.read_index(p16).dtype == "float32"                    # a faiss file is fp32 unless asked
        pr = os.path.join(str(tmp_path), f"{name}.rsb1")
        rsb.write_index(ix16, pr, fmt="rsb1")
        with open(pr, "rb") as f:
            assert pickle.load(f)["payload"].dtype == np.float16       # kept as stored
        back = rsb.read_index(pr)
        assert back.dtype == "float16"
        I1, D1 = back.search_ids(q, 50)
        assert torch.equal(I0, I1) and torch.equal(D0, D1)
    # a file whose values are not fp16-representable is refused
    f32 = rsb.IndexFlatIP(IVF_D)
    f32.add(np.random.default_rng(0).standard_normal((50, IVF_D)).astype(np.float32))
    path = os.path.join(str(tmp_path), "f32.faiss")
    rsb.write_index(f32, path)
    with pytest.raises(ValueError, match="float16"):
        rsb.read_index(path, storage_dtype="float16")
    rsb.write_index(f32, path + ".rsb1", fmt="rsb1")
    with pytest.raises(ValueError, match="float16"):
        rsb.read_index(path + ".rsb1", storage_dtype="float16")


# ---------------------------------------------------------------------------------------------------------------
# drop-in boundary
# ---------------------------------------------------------------------------------------------------------------
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IDX_D = 64


def _datastore(root, n=3000, fp32_noise=False):
    rng = np.random.default_rng(0)
    centres = rng.standard_normal((8, IDX_D)).astype(np.float32)
    emb_dir = os.path.join(root, "embeddings", "enc", "dom", "2-shards")
    psg_dir = os.path.join(root, "passages", "dom", "2-shards")
    os.makedirs(emb_dir); os.makedirs(psg_dir)
    for s in range(2):
        e = ((centres[rng.integers(0, 8, n)] + 0.3 * rng.standard_normal((n, IDX_D))) / 8.0).astype(np.float16)
        if fp32_noise and s == 1:
            e = e.astype(np.float32) + np.float32(1e-6)              # no longer fp16-representable
        with open(os.path.join(emb_dir, f"passages_{s:02d}.pkl"), "wb") as f:
            pickle.dump((list(range(n)), e), f)
        with open(os.path.join(psg_dir, f"raw_passages-{s}-of-2.jsonl"), "w") as f:
            for c in range(n):
                f.write('{"text": "p%d_%d"}\n' % (s, c))
    return ((centres[rng.integers(0, 8, 12)] + 0.3 * rng.standard_normal((12, IDX_D))) / 8.0).astype(np.float32)


def _cfg(root, index_type, extra=()):
    from retrieval_scaling_b200 import config as C
    ov = [f"datastore.datastore_root_dir={root}", "datastore.domain=dom", "model.datastore_encoder=enc",
          "datastore.embedding.num_shards=2", f"datastore.index.index_type={index_type}",
          "datastore.index.index_shard_ids=[0,1]", f"datastore.index.projection_size={IDX_D}",
          "datastore.index.ncentroids=16", "datastore.index.probe=4", "datastore.index.sample_train_size=4000",
          "evaluation.search.n_docs=5"] + list(extra)
    return C.load_config("default", os.path.join(ROOT, "ric", "conf"), ov)


@pytest.mark.parametrize("index_type", ["Flat", "IVFFlat"])
def test_indexer_storage_dtype(tmp_path, index_type):
    from retrieval_scaling_b200.indicies.base import Indexer
    r32, r16 = os.path.join(str(tmp_path), "a"), os.path.join(str(tmp_path), "b")
    q = _datastore(r32)
    _datastore(r16)
    i32 = Indexer(_cfg(r32, index_type))
    key = ["+datastore.index.storage_dtype=float16"]
    i16 = Indexer(_cfg(r16, index_type, key))
    assert i16.datastore.index.dtype == "float16" and i32.datastore.index.dtype == "float32"
    qt = torch.from_numpy(q).cuda()
    I32, D32 = (t.cpu().numpy() for t in i32.search_ids(qt, 50))
    I16, D16 = (t.cpu().numpy() for t in i16.search_ids(qt, 50))
    if index_type == "IVFFlat":
        assert np.array_equal(I16, I32) and np.array_equal(D16, D32)
    else:
        _check_flat(D16, I16, D32, I32, 50)
    p32, p16 = i32.datastore.index_path, i16.datastore.index_path
    assert open(p32, "rb").read() == open(p16, "rb").read()
    again = Indexer(_cfg(r16, index_type, key))                         # the .faiss artefact reloads into fp16
    assert again.datastore.index.dtype == "float16"
    I2, D2 = (t.cpu().numpy() for t in again.search_ids(qt, 50))
    assert np.array_equal(I2, I16) and np.array_equal(D2, D16)
    s16 = i16.search(q, 5)
    s32 = i32.search(q, 5)
    assert s16[0] == s32[0] or index_type == "Flat"
    bad = os.path.join(str(tmp_path), "c")
    _datastore(bad, fp32_noise=True)
    with pytest.raises(ValueError, match="passages_01"):
        Indexer(_cfg(bad, index_type, key))
