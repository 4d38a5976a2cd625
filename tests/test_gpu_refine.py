"""Exact re-ranking on the GPU (IndexRefine, rsb_search_refine / rsb_refine): parity with the CPU oracle (faiss
IndexRefine::search restated in oracle/refine_oracle.py), the k' = k * k_factor limit, padding, store dtypes, the
Indexer(cfg) integration with two embedding shards, and the IndexRefineFlat (IxRF) file round trip."""
import os
import sys

import numpy as np
import pytest
import torch

from oracle import ann_oracle as O
from oracle import refine_oracle as R

pytestmark = pytest.mark.gpu
D = 192                    # divisible by M = 16, 32, 64 and by the generic M = 24
NLIST, N = 32, 20000


def _data(seed=0, n=N, nq=1000):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((NLIST, D)).astype(np.float32)
    xb = (centres[rng.integers(0, NLIST, n)] + 0.5 * rng.standard_normal((n, D))).astype(np.float16)   # fp16 like the pickles
    xq = (centres[rng.integers(0, NLIST, nq)] + 0.5 * rng.standard_normal((nq, D))).astype(np.float32)
    cent = centres / np.linalg.norm(centres, axis=1, keepdims=True)
    return rng, xb, xq, cent


_CACHE = {}


def _index(M, store_dtype="float16"):
    key = (M, store_dtype)
    if key not in _CACHE:
        import retrieval_scaling_b200 as rsb
        rng, xb, xq, cent = _data()
        cb = (0.5 * rng.standard_normal((M, 256, D // M))).astype(np.float32)
        base = rsb.IndexIVFPQ(D, NLIST, M, 8)
        base.set_centroids(cent)
        base.set_codebook(cb)
        ref = rsb.IndexRefine(base, store_dtype=store_dtype)
        ref.add(xb.astype(np.float32))
        ref.nprobe = 4
        _CACHE[key] = (ref, xb, xq, cent, cb)
    return _CACHE[key]


def _exact(xq, xb, I):
    """float64 <q, x_id> for every returned pair (NaN for padding)."""
    out = np.full(I.shape, np.nan)
    for i in range(I.shape[0]):
        v = I[i] >= 0
        out[i, v] = xb[I[i, v]].astype(np.float64) @ xq[i].astype(np.float64)
    return out


@pytest.mark.parametrize("M", [16, 32, 64, 24])
def test_base_candidates_match_the_oracle(M):
    """The re-rank's input: the GPU base search at k' equals the C oracle's IVF-PQ search on the same index."""
    from oracle import c_oracle as CO
    ref, xb, xq, cent, cb = _index(M)
    q = xq[:64]
    Ib, Db = ref.base.search_ids(torch.from_numpy(q).cuda(), 400)
    off, codes, ids = (t.cpu().numpy() for t in ref.base.export_lists())
    Dr, Ir = CO.ivfpq_search(q, cent, cb, off, codes, ids, 4, 400)
    O.assert_topk_equivalent(Db.cpu().numpy(), Ib.cpu().numpy(), Dr, Ir, rtol=1e-5, atol=2e-4)


@pytest.mark.parametrize("M", [16, 32, 64, 24])
@pytest.mark.parametrize("k", [1, 10, 100])
@pytest.mark.parametrize("k_factor", [1, 4, 16])
@pytest.mark.parametrize("nq", [1, 7, 1000])
def test_parity_with_oracle(M, k, k_factor, nq):
    ref, xb, xq, _, _ = _index(M)
    q = torch.from_numpy(xq[:nq]).cuda()
    I, Dd = ref.search_ids(q, k, k_factor=k_factor)
    Ib, _ = ref.base.search_ids(q, k * k_factor)
    Do, Io = R.refine_candidates(xq[:nq], xb, Ib.cpu().numpy(), k)
    I, Dd = I.cpu().numpy(), Dd.cpu().numpy()
    score_of = lambda qi, i: float(xb[i].astype(np.float64) @ xq[qi].astype(np.float64))   # noqa: E731
    O.assert_topk_equivalent(Dd, I, Do, Io, score_of=score_of, rtol=1e-5, atol=1e-5)
    # the standalone re-rank entry on the same candidates gives the same answer
    I2, D2 = ref.rerank(q, Ib, k)
    assert np.array_equal(I2.cpu().numpy(), I) and np.array_equal(D2.cpu().numpy(), Dd)
    # every returned score is the exact inner product with the store row of the returned id
    ex = _exact(xq[:nq], xb, I)
    v = I >= 0
    assert np.allclose(Dd[v], ex[v], rtol=1e-5, atol=1e-5)
    # re-ranking never makes a rank worse: refined exact >= exact scores of the unrefined result, rank by rank
    Iu, _ = ref.base.search_ids(q, k)
    exu = _exact(xq[:nq], xb, Iu.cpu().numpy())
    exu = -np.sort(-np.where(np.isnan(exu), -np.inf, exu), axis=1)
    both = v & np.isfinite(exu)
    assert (Dd[both] >= exu[both] - 1e-5 * np.abs(exu[both]) - 1e-5).all()
    if k_factor == 1:            # the base's id set, re-ordered by exact score
        Iu = Iu.cpu().numpy()
        assert all(set(a[a >= 0]) == set(b[b >= 0]) for a, b in zip(I, Iu))
        assert (np.diff(np.where(v, Dd, -np.inf), axis=1) <= 0).all()


def test_largest_k_prime_and_the_limit():
    ref, xb, xq, _, _ = _index(16)
    q = torch.from_numpy(xq[:7]).cuda()
    I, Dd = ref.search_ids(q, 256, k_factor=16, nprobe=32)          # k' = 4096
    Ib, _ = ref.base.search_ids(q, 4096, nprobe=32)
    Do, Io = R.refine_candidates(xq[:7], xb, Ib.cpu().numpy(), 256)
    O.assert_topk_equivalent(Dd.cpu().numpy(), I.cpu().numpy(), Do, Io, rtol=1e-5, atol=1e-5)
    with pytest.raises(NotImplementedError, match="4096"):
        ref.search_ids(q, 241, k_factor=17)                            # k' = 4097
    with pytest.raises(NotImplementedError):
        ref.rerank(q, torch.zeros((7, 4097), dtype=torch.int64, device="cuda"), 10)


def test_short_lists_pad_like_the_oracle():
    ref, xb, xq, _, _ = _index(32)
    q = torch.from_numpy(xq[:50]).cuda()
    I, Dd = ref.search_ids(q, 1000, k_factor=4, nprobe=1)              # one list holds ~600 vectors < k'
    Ib, _ = ref.base.search_ids(q, 4000, nprobe=1)
    Do, Io = R.refine_candidates(xq[:50], xb, Ib.cpu().numpy(), 1000)
    I, Dd = I.cpu().numpy(), Dd.cpu().numpy()
    assert (Io == -1).any()
    O.assert_topk_equivalent(Dd, I, Do, Io, rtol=1e-5, atol=1e-5)
    assert (Dd[I < 0] == np.finfo(np.float32).min).all()


def test_fp16_and_fp32_stores_agree_bit_for_bit():
    ref16, xb, xq, _, _ = _index(64, "float16")
    ref32, _, _, _, _ = _index(64, "float32")
    q = torch.from_numpy(xq[:300]).cuda()
    for kf in (1, 8):
        a, b = ref16.search_ids(q, 50, k_factor=kf), ref32.search_ids(q, 50, k_factor=kf)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_refine_needs_ivfpq_and_sequential_ids(tmp_path):
    import retrieval_scaling_b200 as rsb
    with pytest.raises(ValueError):
        rsb.IndexRefine(rsb.IndexFlatIP(D))
    with pytest.raises(ValueError):
        rsb.IndexRefine(rsb.IndexIVFFlat(D, 4))
    ref, xb, _, _, _ = _index(16)
    with pytest.raises(ValueError, match="custom ids"):
        ref.add(xb[:10].astype(np.float32), ids=np.arange(10) + 10 ** 6)
    free, _ = torch.cuda.mem_get_info()
    with pytest.raises(MemoryError, match="bytes"):
        rsb.IndexRefine(ref.base, "float32").reserve(free // (D * 4) + 1)


def test_ixrf_reload_searches_identically(tmp_path):
    import retrieval_scaling_b200 as rsb
    ref, xb, xq, _, _ = _index(24)
    ref.k_factor = 8
    path = str(tmp_path / "refine.faiss")
    rsb.write_index(ref, path)
    with open(path, "rb") as f:
        assert f.read(4) == b"IxRF"
    back = rsb.read_index(path, refine_dtype="float16")              # written upcast to fp32, every value round-trips
    assert isinstance(back, rsb.IndexRefine) and back.k_factor == 8 and back.store_dtype == "float16"
    assert torch.equal(back.store, ref.store)
    back.nprobe = ref.nprobe
    q = torch.from_numpy(xq[:100]).cuda()
    a, b = ref.search_ids(q, 20), back.search_ids(q, 20)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    ref.k_factor = 1


def test_indexer_store_follows_meta_order(tmp_path):
    """Indexer(cfg) with refine_k_factor over two fp16 embedding shards: each returned score is <q, embedding of
    its [shard, chunk]>; search and search_ids agree; ShardedSearcher refuses to partition a refined index."""
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_gpu_indexer import _cfg, _make_datastore
    from retrieval_scaling_b200.indicies.base import Indexer
    import retrieval_scaling_b200 as rsb
    embs, q = _make_datastore(str(tmp_path))
    cfg = _cfg(str(tmp_path), "IVFPQ", "[0,1]", ["+datastore.index.refine_k_factor=8", "datastore.index.probe=4"])
    ix = Indexer(cfg)
    assert isinstance(ix.datastore.index, rsb.IndexRefine) and ix.datastore.index.store_dtype == "float16"
    scores, passages, db_ids = ix.search(q, 5)
    qf = q.astype(np.float64)
    for i in range(len(q)):
        assert len(db_ids[i]) == 5
        for (s, c), sc in zip(db_ids[i], scores[i]):
            assert np.isclose(sc, embs[s][c].astype(np.float64) @ qf[i], rtol=1e-5, atol=1e-6)
    ids, sc = ix.search_ids(q.astype(np.float32), 5)
    assert np.allclose(sc.cpu().numpy(), np.asarray(scores, np.float32), rtol=0, atol=0)
    names = os.listdir(os.path.join(cfg.datastore.embedding.embedding_dir, "index_IVFPQ", "0_1"))
    faiss_file = [n for n in names if n.endswith(".faiss")][0]
    with open(os.path.join(cfg.datastore.embedding.embedding_dir, "index_IVFPQ", "0_1", faiss_file), "rb") as f:
        assert f.read(4) == b"IwPQ"                                   # the artefact stays the plain IVF-PQ base
    ix2 = Indexer(cfg)                                                # reload from disk + store rebuilt from pickles
    assert ix2.search(q, 5)[2] == db_ids
    from retrieval_scaling_b200.dist import ShardedSearcher
    with pytest.raises(NotImplementedError):
        ShardedSearcher(ix.datastore.index, 2, 0)
