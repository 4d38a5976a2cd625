"""GPU parity tests proper: the CUDA path (through the C-ABI, via the ctypes wrapper) against the CPU oracle on
the same seeded inputs.  Integer / index results must agree exactly (modulo fp32 near-ties, see
`assert_topk_equivalent`); float scores within 1e-5 relative (the north star allows 1e-4)."""
import numpy as np
import pytest
import torch

from oracle import ann_oracle as O
from oracle import c_oracle as C

pytestmark = pytest.mark.gpu

NEG = np.finfo(np.float32).min
RTOL, ATOL = 1e-5, 1e-5


def _rsb():
    import retrieval_scaling_b200 as r
    return r


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ------------------------------------------------------------------------------------------------------------
# Flat
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,d,nq,k", [(5000, 64, 33, 10), (20000, 768, 64, 10), (1000, 128, 7, 1), (300, 32, 5, 100)])
def test_flat_matches_oracle(n, d, nq, k):
    r = _rsb()
    rng = np.random.default_rng(n + d)
    xb = rng.standard_normal((n, d)).astype(np.float32)
    xq = rng.standard_normal((nq, d)).astype(np.float32)
    index = r.IndexFlatIP(d)
    index.add(xb[: n // 2])
    index.add(xb[n // 2:])               # two adds -> segment concat path
    assert index.ntotal == n
    D, I = index.search(xq, k)
    Dr, Ir = C.flat_search(xq, xb, k)
    xb64, xq64 = xb.astype(np.float64), xq.astype(np.float64)
    O.assert_topk_equivalent(D, I, Dr, Ir, score_of=lambda q, i: xb64[i] @ xq64[q], rtol=RTOL, atol=ATOL * np.sqrt(d))


def test_flat_c1_config_ids_identical():
    """BASELINE config 1: Flat, 100k x 768 fp32, 1k queries, k = 10 (numpy/OpenBLAS sgemm oracle)."""
    r = _rsb()
    rng = np.random.default_rng(1234)
    xb = rng.standard_normal((100_000, 768)).astype(np.float32)
    xq = rng.standard_normal((1000, 768)).astype(np.float32)
    index = r.IndexFlatIP(768)
    index.add(xb)
    D, I = index.search(xq, 10)
    Dr, Ir = O.flat_search(xq, xb, 10)
    xb64, xq64 = xb.astype(np.float64), xq.astype(np.float64)
    O.assert_topk_equivalent(D, I, Dr, Ir, score_of=lambda q, i: xb64[i] @ xq64[q], rtol=RTOL, atol=3e-4)
    assert (I == Ir).mean() > 0.9999      # near-ties are the only allowed differences and are very rare
    rel = np.abs(D - Dr) / np.maximum(np.abs(Dr), 1e-6)
    assert rel.max() < 1e-4


def test_flat_padding_duplicates_and_empty():
    r = _rsb()
    index = r.IndexFlatIP(8)
    D, I = index.search(np.ones((2, 8), np.float32), 3)        # empty index
    assert (I == -1).all() and (D == NEG).all()
    xb = np.tile(np.arange(8, dtype=np.float32)[None], (6, 1))  # 6 identical rows
    index.add(xb)
    D, I = index.search(np.ones((1, 8), np.float32), 10)        # k > ntotal
    assert I[0, :6].tolist() == [0, 1, 2, 3, 4, 5] and (I[0, 6:] == -1).all()
    assert (D[0, :6] == 28).all() and (D[0, 6:] == NEG).all()
    D, I = index.search(np.ones((0, 8), np.float32), 4)
    assert D.shape == (0, 4) and I.shape == (0, 4)


def test_flat_large_k_and_custom_ids():
    r = _rsb()
    rng = np.random.default_rng(7)
    xb = rng.standard_normal((9000, 64)).astype(np.float32)
    xq = rng.standard_normal((5, 64)).astype(np.float32)
    ids = (np.arange(9000, dtype=np.int64) * 7 + 3)
    index = r.IndexFlatIP(64)
    index.add(xb, ids)
    for k in (1000, 4096):
        D, I = index.search(xq, k)
        Dr, Ir = C.flat_search(xq, xb, k)
        O.assert_topk_equivalent(D, (I - 3) // 7, Dr, Ir, rtol=RTOL, atol=1e-4)
    with pytest.raises(NotImplementedError):
        index.search(xq, 5000)


# ------------------------------------------------------------------------------------------------------------
# layout round trip / encode
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M", [16, 32, 64, 24, 96])
def test_pq_layout_roundtrip(M):
    r = _rsb()
    rng = np.random.default_rng(M)
    d, nlist, n = M * 4, 37, 5003
    index = r.IndexIVFPQ(d, nlist, M)
    index.set_centroids(rng.standard_normal((nlist, d)).astype(np.float32))
    index.set_codebook(rng.standard_normal((M, 256, 4)).astype(np.float32))
    codes = rng.integers(0, 256, (n, M), dtype=np.uint8)
    lists = rng.integers(0, nlist, n).astype(np.int32)
    lists[lists == 5] = 6                                       # list 5 stays empty
    ids = rng.permutation(n).astype(np.int64) + 1000
    index.add_codes(codes[:2000], lists[:2000], ids[:2000])
    index.add_codes(codes[2000:], lists[2000:], ids[2000:])
    off, payload, eids = index.export_lists()
    roff, perm, rids = O.build_csr(lists.astype(np.int64), nlist, ids)
    assert np.array_equal(off.cpu().numpy(), roff)
    assert np.array_equal(eids.cpu().numpy(), rids)
    assert np.array_equal(payload.cpu().numpy(), codes[perm])
    assert np.array_equal(index.list_sizes().cpu().numpy(), np.diff(roff))
    # adding after finalize re-merges the existing layout with the new rows
    extra = rng.integers(0, 256, (77, M), dtype=np.uint8)
    index.add_codes(extra, np.full(77, 5, np.int32), np.arange(77, dtype=np.int64))
    off2, payload2, eids2 = index.export_lists()
    lists2 = np.concatenate([lists, np.full(77, 5, np.int32)])
    roff2, perm2, rids2 = O.build_csr(lists2.astype(np.int64), nlist, np.concatenate([ids, np.arange(77)]))
    assert np.array_equal(off2.cpu().numpy(), roff2)
    assert np.array_equal(payload2.cpu().numpy(), np.concatenate([codes, extra])[perm2])
    assert np.array_equal(eids2.cpu().numpy(), rids2)


@pytest.mark.parametrize("d,M", [(768, 64), (768, 16), (192, 32), (96, 16)])
def test_assign_and_encode_match_oracle(d, M):
    r = _rsb()
    rng = np.random.default_rng(d + M)
    nlist, n = 50, 3000
    cent = rng.standard_normal((nlist, d)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    cb = (0.3 * rng.standard_normal((M, 256, d // M))).astype(np.float32)
    xb = (cent[rng.integers(0, nlist, n)] * 3 + 0.5 * rng.standard_normal((n, d))).astype(np.float32)
    index = r.IndexIVFPQ(d, nlist, M)
    index.set_centroids(cent)
    index.set_codebook(cb)
    index.add(xb)
    off, payload, eids = index.export_lists()
    off, payload, eids = off.cpu().numpy(), payload.cpu().numpy(), eids.cpu().numpy()
    ra, rcodes = O.ivfpq_encode(xb, cent, cb)
    gpu_assign = np.empty(n, np.int64)
    gpu_assign[eids] = np.repeat(np.arange(nlist), np.diff(off))
    agree = gpu_assign == ra
    assert agree.mean() > 0.999                    # argmax near-ties may differ in fp32
    gcodes = np.empty((n, M), np.uint8)
    gcodes[eids] = payload
    same = (gcodes[agree] == rcodes[agree]).mean()
    assert same > 0.999, same                      # argmin near-ties only


# ------------------------------------------------------------------------------------------------------------
# IVF-Flat
# ------------------------------------------------------------------------------------------------------------
def _clustered(rng, n, d, ncl, noise=0.35):
    centres = rng.standard_normal((ncl, d)).astype(np.float32)
    return (centres[rng.integers(0, ncl, n)] + noise * rng.standard_normal((n, d))).astype(np.float32), centres


@pytest.mark.parametrize("n,d,nlist,nprobe,k,nq", [(20000, 768, 64, 8, 100, 40), (6000, 128, 32, 32, 10, 9),
                                                  (3000, 100, 16, 3, 1, 1)])
def test_ivfflat_matches_oracle(n, d, nlist, nprobe, k, nq):
    r = _rsb()
    rng = np.random.default_rng(n)
    xb, centres = _clustered(rng, n, d, nlist)
    xq, _ = _clustered(rng, nq, d, nlist)
    xq = (centres[rng.integers(0, nlist, nq)] + 0.35 * rng.standard_normal((nq, d))).astype(np.float32)
    cent = centres / np.linalg.norm(centres, axis=1, keepdims=True)
    index = r.IndexIVFFlat(d, nlist)
    index.set_centroids(cent)
    index.add(xb)
    index.nprobe = nprobe
    D, I = index.search(xq, k)
    off, vecs, ids = (t.cpu().numpy() for t in index.export_lists())
    Dr, Ir = C.ivfflat_search(xq, cent, off, vecs, ids, nprobe, k)
    xb64, xq64 = xb.astype(np.float64), xq.astype(np.float64)
    O.assert_topk_equivalent(D, I, Dr, Ir, score_of=lambda q, i: xb64[i] @ xq64[q], rtol=RTOL, atol=1e-4)
    if nprobe == nlist:   # full probe == Flat
        Df, If = C.flat_search(xq, xb, k)
        O.assert_topk_equivalent(D, I, Df, If, score_of=lambda q, i: xb64[i] @ xq64[q], rtol=RTOL, atol=1e-4)


def test_ivfflat_empty_lists_padding_and_nprobe_clamp():
    r = _rsb()
    rng = np.random.default_rng(3)
    d, nlist = 32, 8
    cent = rng.standard_normal((nlist, d)).astype(np.float32)
    xb = rng.standard_normal((40, d)).astype(np.float32)
    lists = np.array([0] * 10 + [7] * 30, dtype=np.int32)        # lists 1..6 empty
    index = r.IndexIVFFlat(d, nlist)
    index.set_centroids(cent)
    index.add_preassigned(xb, lists)
    xq = rng.standard_normal((6, d)).astype(np.float32)
    for nprobe in (1, 3, 8, 50):                                   # 50 > nlist -> clamped like faiss
        index.nprobe = nprobe
        D, I = index.search(xq, 60)
        off, vecs, ids = (t.cpu().numpy() for t in index.export_lists())
        Dr, Ir = C.ivfflat_search(xq, cent, off, vecs, ids, min(nprobe, nlist), 60)
        O.assert_topk_equivalent(D, I, Dr, Ir, rtol=RTOL, atol=1e-4)
        assert ((I == -1) == (D == NEG)).all()


# ------------------------------------------------------------------------------------------------------------
# IVF-PQ
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,M,nlist,nprobe,k,n,nq", [
    (768, 64, 64, 8, 100, 30000, 50),      # C3-shaped (M=64, dsub=12)
    (768, 16, 32, 32, 10, 8000, 17),       # repo default n_subquantizers=16, full probe
    (192, 32, 16, 4, 33, 5000, 8),
    (64, 16, 4, 2, 1, 500, 1),
    (768, 48, 32, 8, 100, 12000, 21),      # generic-M path: sub-quantizer counts the tuned layout does not cover
    (768, 96, 16, 16, 10, 6000, 9),
    (96, 24, 8, 3, 50, 3000, 5),
])
def test_ivfpq_matches_oracle(d, M, nlist, nprobe, k, n, nq):
    r = _rsb()
    rng = np.random.default_rng(d * M + n)
    xb, centres = _clustered(rng, n, d, nlist)
    xq = (centres[rng.integers(0, nlist, nq)] + 0.35 * rng.standard_normal((nq, d))).astype(np.float32)
    cent = centres / np.linalg.norm(centres, axis=1, keepdims=True)
    cb = (0.35 * rng.standard_normal((M, 256, d // M))).astype(np.float32)
    index = r.IndexIVFPQ(d, nlist, M)
    index.set_centroids(cent)
    index.set_codebook(cb)
    index.add(xb[: n // 3])
    index.add(xb[n // 3:])
    index.nprobe = nprobe
    D, I = index.search(xq, k)
    off, codes, ids = (t.cpu().numpy() for t in index.export_lists())
    Dr, Ir = C.ivfpq_search(xq, cent, cb, off, codes, ids, nprobe, k)
    # fp64 re-score of a (query, id) pair for boundary near-ties
    pos_of = np.empty(n, np.int64); pos_of[ids] = np.arange(n)
    list_of = np.repeat(np.arange(nlist), np.diff(off))
    rec = O.pq_decode(codes, cb).astype(np.float64)
    def score_of(q, i):
        p = pos_of[i]
        return (cent[list_of[p]].astype(np.float64) + rec[p]) @ xq[q].astype(np.float64)
    O.assert_topk_equivalent(D, I, Dr, Ir, score_of=score_of, rtol=RTOL, atol=2e-4)


def test_tensor_core_coarse_matches_cuda_core_coarse():
    """3xTF32 (wgmma) coarse quantizer == fp32 CUDA-core coarse quantizer == oracle, on a C3-shaped problem."""
    r = _rsb()
    rng = np.random.default_rng(29)
    d, nlist, nq, nprobe = 768, 1000, 300, 32
    cent = rng.standard_normal((nlist, d)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    xq = (cent[rng.integers(0, nlist, nq)] * 3 + 0.7 * rng.standard_normal((nq, d))).astype(np.float32)
    index = r.IndexIVFFlat(d, nlist)
    index.set_centroids(cent)
    Lt, St = index.coarse(xq, nprobe)                    # tensor-core path (default)
    index.set_option(0, 0)
    Lc, Sc = index.coarse(xq, nprobe)                    # CUDA-core fp32 path
    Sr, Lr = O.coarse_probe(xq, cent, nprobe)
    c64, q64 = cent.astype(np.float64), xq.astype(np.float64)
    for L, S in ((Lt, St), (Lc, Sc)):
        O.assert_topk_equivalent(S.cpu().numpy(), L.cpu().numpy(), Sr, Lr, score_of=lambda q, i: c64[i] @ q64[q],
                                 rtol=RTOL, atol=1e-5)
    assert (Lt == Lc).float().mean().item() > 0.9999     # exact fp32 re-score makes the two paths agree
    assert (St - Sc).abs().max().item() < 1e-5


@pytest.mark.parametrize("d,nlist,nq,nprobe", [(768, 16384, 700, 32), (64, 4096, 300, 8), (128, 5000, 129, 1)])
def test_fused_coarse_scorer_matches_oracle(d, nlist, nq, nprobe):
    """The fused 3xTF32 scorer + per-half-tile top-8 filter (no score matrix in HBM) + exact re-score returns the same
    top-nprobe lists as the oracle's IndexFlatIP quantizer and as the score-matrix path (RSB_OPT_COARSE_TENSOR = 0),
    including ragged shapes (nq % 128 != 0, nlist % 256 != 0)."""
    r = _rsb()
    rng = np.random.default_rng(d + nlist)
    cent = rng.standard_normal((nlist, d)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    xq = (cent[rng.integers(0, nlist, nq)] * 2 + 0.8 * rng.standard_normal((nq, d))).astype(np.float32)
    index = r.IndexIVFFlat(d, nlist)
    index.set_centroids(cent)
    Lt, St = index.coarse(xq, nprobe)
    Sr, Lr = O.coarse_probe(xq, cent, nprobe)
    c64, q64 = cent.astype(np.float64), xq.astype(np.float64)
    O.assert_topk_equivalent(St.cpu().numpy(), Lt.cpu().numpy(), Sr, Lr, score_of=lambda q, i: c64[i] @ q64[q],
                             rtol=RTOL, atol=1e-5)
    index.set_option(0, 0)
    Lc, Sc = index.coarse(xq, nprobe)
    assert (Lt == Lc).float().mean().item() > 0.9999 and (St - Sc).abs().max().item() < 1e-5


def test_fused_coarse_scorer_concentrated_rows_take_the_exhaustive_path():
    """Adversarial layout for the per-half-tile filter: for half of the queries, 30 near-duplicate best centroids sit in
    ONE 128-column half tile, so the top 8 of that half tile cannot contain the row's top 24 -- the bound check must
    flag those rows and the exhaustive fp32 pass must still return exactly the oracle's lists."""
    r = _rsb()
    rng = np.random.default_rng(5)
    d, nlist, nq, nprobe = 64, 4096, 64, 16
    cent = rng.standard_normal((nlist, d)).astype(np.float32)
    cent /= np.linalg.norm(cent, axis=1, keepdims=True)
    hot = rng.standard_normal(d).astype(np.float32)
    hot /= np.linalg.norm(hot)
    cols = 1024 + rng.permutation(128)[:30]                   # all inside columns [1024, 1152): one half tile
    cent[cols] = hot[None, :] + 0.01 * rng.standard_normal((30, d)).astype(np.float32)
    xq = rng.standard_normal((nq, d)).astype(np.float32)
    xq[::2] = 3 * hot[None, :] + 0.05 * rng.standard_normal((nq // 2, d)).astype(np.float32)
    index = r.IndexIVFFlat(d, nlist)
    index.set_centroids(cent)
    L, S = index.coarse(xq, nprobe)
    Sr, Lr = O.coarse_probe(xq, cent, nprobe)
    c64, q64 = cent.astype(np.float64), xq.astype(np.float64)
    O.assert_topk_equivalent(S.cpu().numpy(), L.cpu().numpy(), Sr, Lr, score_of=lambda q, i: c64[i] @ q64[q],
                             rtol=RTOL, atol=1e-5)
    assert set(L[0].tolist()) <= set(cols.tolist())           # the concentrated row really has its top 16 in that half tile


def test_ivfpq_edge_cases():
    r = _rsb()
    rng = np.random.default_rng(11)
    d, M, nlist = 64, 16, 6
    cent = rng.standard_normal((nlist, d)).astype(np.float32)
    cb = rng.standard_normal((M, 256, d // M)).astype(np.float32)
    index = r.IndexIVFPQ(d, nlist, M)
    with pytest.raises(RuntimeError):
        index.add(rng.standard_normal((4, d)).astype(np.float32))   # not trained
    index.set_centroids(cent)
    index.set_codebook(cb)
    assert index.is_trained and index.ntotal == 0
    D, I = index.search(rng.standard_normal((3, d)).astype(np.float32), 5)
    assert (I == -1).all() and (D == NEG).all()
    # one list with exactly 32, one with 33, one with 1 vector, others empty (block-padding boundaries)
    codes = rng.integers(0, 256, (66, M), dtype=np.uint8)
    lists = np.array([1] * 32 + [3] * 33 + [4], dtype=np.int32)
    index.add_codes(codes, lists)
    xq = rng.standard_normal((5, d)).astype(np.float32)
    for nprobe, k in ((1, 5), (6, 66), (6, 100), (2, 40)):
        index.nprobe = nprobe
        D, I = index.search(xq, k)
        off, cc, ids = (t.cpu().numpy() for t in index.export_lists())
        Dr, Ir = C.ivfpq_search(xq, cent, cb, off, cc, ids, nprobe, k)
        O.assert_topk_equivalent(D, I, Dr, Ir, rtol=RTOL, atol=2e-4)


def test_ivfpq_large_k_and_many_probes():
    r = _rsb()
    rng = np.random.default_rng(13)
    d, M, nlist, n = 128, 32, 128, 40000
    xb, centres = _clustered(rng, n, d, nlist)
    cent = centres / np.linalg.norm(centres, axis=1, keepdims=True)
    cb = (0.35 * rng.standard_normal((M, 256, d // M))).astype(np.float32)
    index = r.IndexIVFPQ(d, nlist, M)
    index.set_centroids(cent)
    index.set_codebook(cb)
    index.add(xb)
    xq = rng.standard_normal((6, d)).astype(np.float32)
    off, codes, ids = (t.cpu().numpy() for t in index.export_lists())
    for nprobe, k in ((128, 1000), (64, 2048), (16, 600)):
        index.nprobe = nprobe
        D, I = index.search(xq, k)
        Dr, Ir = C.ivfpq_search(xq, cent, cb, off, codes, ids, nprobe, k)
        O.assert_topk_equivalent(D, I, Dr, Ir, rtol=RTOL, atol=2e-4)


def test_train_build_search_recall_and_persistence(tmp_path):
    """End-to-end on the GPU: k-means + PQ training, add, search; IVF-PQ recall against exact Flat and a
    write_index/read_index round trip (same results after reload)."""
    r = _rsb()
    rng = np.random.default_rng(17)
    d, n, nlist, M = 128, 60000, 64, 32
    xb, centres = _clustered(rng, n, d, 16)
    xq = (centres[rng.integers(0, 16, 64)] + 0.35 * rng.standard_normal((64, d))).astype(np.float32)
    flat = r.IndexFlatIP(d); flat.add(xb)
    Df, If = flat.search(xq, 10)
    ivf = r.IndexIVFFlat(d, nlist); ivf.train(xb); ivf.add(xb); ivf.nprobe = 16
    D1, I1 = ivf.search(xq, 10)
    assert O.recall_at_k(I1, If) > 0.9
    pq = r.IndexIVFPQ(d, nlist, M); pq.train(xb); pq.add(xb); pq.nprobe = 16
    D2, I2 = pq.search(xq, 10)
    D2w, I2w = pq.search(xq, 100)
    # PQ is lossy (dsub = 4 on isotropic within-cluster noise): demand that most true top-10 neighbours are
    # inside the PQ top-100, and that the GPU result equals the oracle's on the trained index.
    hit = np.mean([len(set(If[q].tolist()) & set(I2w[q].tolist())) / 10.0 for q in range(xq.shape[0])])
    assert hit > 0.6, hit
    off, codes, ids = (t.cpu().numpy() for t in pq.export_lists())
    Dr, Ir = C.ivfpq_search(xq, pq.get_centroids().cpu().numpy(), pq.get_codebook().cpu().numpy(), off, codes, ids, 16, 10)
    O.assert_topk_equivalent(D2, I2, Dr, Ir, rtol=RTOL, atol=2e-4)
    path = str(tmp_path / "index_IVFPQ.faiss")
    r.write_index(pq, path)
    pq2 = r.read_index(path)
    assert pq2.ntotal == n and pq2.nprobe == 16
    D3, I3 = pq2.search(xq, 10)
    assert np.array_equal(I3, I2) and np.allclose(D3, D2, rtol=1e-6, atol=1e-6)


# ------------------------------------------------------------------------------------------------------------
# merge + properties at scale
# ------------------------------------------------------------------------------------------------------------
def test_merge_topk_matches_reference_semantics():
    r = _rsb()
    rng = np.random.default_rng(19)
    nshards, nq, k = 8, 33, 100
    D = np.sort(rng.standard_normal((nshards, nq, k)).astype(np.float32), axis=2)[:, :, ::-1].copy()
    I = rng.integers(0, 1 << 40, (nshards, nq, k))
    D[3, :, 50:] = NEG; I[3, :, 50:] = -1                   # a short shard
    D[1, 0, 0] = D[0, 0, 0]                                 # exact tie across shards -> lower shard first
    Dm, Im = r.merge_topk(_cuda(D), _cuda(I))
    Dr, Ir = O.merge_topk(list(D), list(I), k)
    assert np.array_equal(Im.cpu().numpy(), Ir) and np.array_equal(Dm.cpu().numpy(), Dr)
    Dm, Im = r.merge_topk(_cuda(D[:, :, :3]), _cuda(I[:, :, :3]), k_out=40)   # fewer than k_out candidates
    Dr, Ir = O.merge_topk(list(D[:, :, :3]), list(I[:, :, :3]), 40)
    assert np.array_equal(Im.cpu().numpy(), Ir) and np.array_equal(Dm.cpu().numpy(), Dr)


def test_sharded_search_equals_single_index():
    """Static datastore partition + merge == one index (SURVEY §8e): ids identical, 1 GPU standing in for G."""
    r = _rsb()
    rng = np.random.default_rng(23)
    d, M, nlist, n, G = 128, 32, 32, 24000, 4
    xb, centres = _clustered(rng, n, d, nlist)
    cent = centres / np.linalg.norm(centres, axis=1, keepdims=True)
    cb = (0.35 * rng.standard_normal((M, 256, d // M))).astype(np.float32)
    xq = rng.standard_normal((20, d)).astype(np.float32)
    def make(rows):
        ix = r.IndexIVFPQ(d, nlist, M); ix.set_centroids(cent); ix.set_codebook(cb)
        ix.add(xb[rows], np.asarray(rows, dtype=np.int64)); ix.nprobe = 8
        return ix
    full = make(np.arange(n))
    Dfull, Ifull = full.search(xq, 50)
    Ds, Is = [], []
    for g in range(G):
        Dg, Ig = make(np.arange(g, n, G)).search(xq, 50)
        Ds.append(Dg); Is.append(Ig)
    Dm, Im = r.merge_topk(_cuda(np.stack(Ds)), _cuda(np.stack(Is)))
    O.assert_topk_equivalent(Dm.cpu().numpy(), Im.cpu().numpy(), Dfull, Ifull, rtol=1e-6, atol=1e-5)


def test_properties_at_scale_ivf_full_probe_equals_flat():
    """Size-independent property at a size the CPU oracle would not finish quickly: IVF-Flat with
    nprobe = nlist must return Flat's answer (GPU vs GPU), 200k x 768."""
    r = _rsb()
    g = torch.Generator(device="cuda").manual_seed(5)
    xb = torch.randn(200_000, 768, generator=g, device="cuda")
    xq = torch.randn(32, 768, generator=g, device="cuda")
    cent = torch.nn.functional.normalize(torch.randn(256, 768, generator=g, device="cuda"), dim=1)
    flat = r.IndexFlatIP(768); flat.add(xb)
    ivf = r.IndexIVFFlat(768, 256); ivf.set_centroids(cent); ivf.add(xb); ivf.nprobe = 256
    Df, If = flat.search(xq, 100)
    Di, Ii = ivf.search(xq, 100)
    O.assert_topk_equivalent(Di.cpu().numpy(), Ii.cpu().numpy(), Df.cpu().numpy(), If.cpu().numpy(), rtol=1e-5, atol=3e-4)
    assert int(ivf.list_sizes().sum()) == 200_000


def test_faiss_format_files_round_trip_on_gpu(tmp_path):
    """write_index(fmt="faiss") / read_index auto-detection: same search results after a trip through the faiss
    binary layout (retrieval_scaling_b200/faiss_io.py), for all three index kinds."""
    r = _rsb()
    rng = np.random.default_rng(31)
    d, nlist, M, n = 64, 8, 16, 3000
    xb, centres = _clustered(rng, n, d, nlist)
    cent = centres / np.linalg.norm(centres, axis=1, keepdims=True)
    xq = rng.standard_normal((9, d)).astype(np.float32)
    flat = r.IndexFlatIP(d); flat.add(xb)
    ivf = r.IndexIVFFlat(d, nlist); ivf.set_centroids(cent); ivf.add(xb); ivf.nprobe = 3
    pq = r.IndexIVFPQ(d, nlist, M); pq.set_centroids(cent)
    pq.set_codebook((0.35 * rng.standard_normal((M, 256, d // M))).astype(np.float32)); pq.add(xb); pq.nprobe = 4
    for name, ix in (("flat", flat), ("ivf", ivf), ("pq", pq)):
        path = str(tmp_path / f"{name}.faiss")
        r.write_index(ix, path, fmt="faiss")
        assert open(path, "rb").read(4) in (b"IxFI", b"IwFl", b"IwPQ")
        ix2 = r.read_index(path)
        assert ix2.ntotal == n and ix2.nprobe == ix.nprobe
        D1, I1 = ix.search(xq, 10)
        D2, I2 = ix2.search(xq, 10)
        assert np.array_equal(I1, I2) and np.allclose(D1, D2, rtol=1e-6, atol=1e-6)


def test_host_pipeline_overlapped_transfers_return_the_same_rows():
    """dist.HostPipeline: batches stream host -> device -> host with the copies of neighbouring batches overlapping the
    search; every batch's host result must equal the direct search of that batch (different queries per batch, so a
    buffer that is reused too early would show up)."""
    r = _rsb()
    from retrieval_scaling_b200.dist import HostPipeline, ShardedSearcher
    rng = np.random.default_rng(3)
    d, M, nlist, n, nq, k = 128, 32, 32, 20000, 300, 20
    xb, centres = _clustered(rng, n, d, nlist)
    cent = centres / np.linalg.norm(centres, axis=1, keepdims=True)
    index = r.IndexIVFPQ(d, nlist, M)
    index.set_centroids(cent)
    index.set_codebook((0.35 * rng.standard_normal((M, 256, d // M))).astype(np.float32))
    index.add(xb)
    index.nprobe = 8
    batches = [torch.from_numpy((centres[rng.integers(0, nlist, nq)] + 0.35 * rng.standard_normal((nq, d))).astype(np.float32)).pin_memory()
               for _ in range(7)]
    outs = [(torch.empty((nq, k), dtype=torch.int64).pin_memory(), torch.empty((nq, k), dtype=torch.float32).pin_memory())
            for _ in range(7)]
    pipe = HostPipeline(ShardedSearcher(index, 1, 0), "cuda")
    for qh, o in zip(batches, outs):
        pipe.submit(qh, k, o)
    pipe.drain()
    for qh, (Ih, Dh) in zip(batches, outs):
        I, D = index.search_ids(qh.cuda(), k)
        assert torch.equal(Ih, I.cpu()) and torch.equal(Dh, D.cpu())


# ------------------------------------------------------------------------------------------------------------
# training: member sums are reproducible (fixed summation order), so index.train gives the same index every run
# ------------------------------------------------------------------------------------------------------------
def test_training_sums_match_float64_and_are_reproducible():
    from retrieval_scaling_b200 import train
    ops = train.default_ops()
    g = torch.Generator(device="cuda").manual_seed(11)
    n, d, k, M = 20000, 96, 300, 8
    x = torch.randn(n, d, generator=g, device="cuda")
    a = torch.randint(-1, k + 1, (n,), generator=g, device="cuda")          # -1 and k: out of range, ignored
    sums, counts = ops.accumulate(x, a, k)
    an, xn = a.cpu().numpy(), x.cpu().numpy().astype(np.float64)
    ok = (an >= 0) & (an < k)
    ref = np.zeros((k, d))
    np.add.at(ref, an[ok], xn[ok])
    assert np.array_equal(counts.cpu().numpy(), np.bincount(an[ok], minlength=k).astype(np.float32))
    assert np.abs(sums.cpu().numpy() - ref).max() < 1e-4
    for _ in range(3):
        s2, c2 = ops.accumulate(x, a, k)
        assert torch.equal(s2, sums) and torch.equal(c2, counts)

    codes = torch.randint(0, 256, (n, M), generator=g, device="cuda", dtype=torch.uint8)
    psums, pcounts = ops.pq_accumulate(x, codes, M, 256)
    cn = codes.cpu().numpy().astype(np.int64)
    dsub = d // M
    pref = np.zeros((M, 256, dsub))
    for m in range(M):
        np.add.at(pref[m], cn[:, m], xn[:, m * dsub:(m + 1) * dsub])
        assert np.array_equal(pcounts[m].cpu().numpy(), np.bincount(cn[:, m], minlength=256).astype(np.float32))
    assert np.abs(psums.cpu().numpy() - pref).max() < 1e-4
    s2, c2 = ops.pq_accumulate(x, codes, M, 256)
    assert torch.equal(s2, psums) and torch.equal(c2, pcounts)

    xs = torch.nn.functional.normalize(x, dim=1)
    c1 = train.kmeans(xs, 64, niter=5, metric="ip", spherical=True, seed=3)
    assert torch.equal(c1, train.kmeans(xs, 64, niter=5, metric="ip", spherical=True, seed=3))
    cb1 = train.train_pq(x, M, 256, niter=4, seed=3)
    assert torch.equal(cb1, train.train_pq(x, M, 256, niter=4, seed=3))
