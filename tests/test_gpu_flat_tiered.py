"""Tiered fp16 Flat index on the GPU (IndexFlatIP(dtype="float16", device_rows=n), RSB_OPT_DEVICE_ROWS): rows [0, n)
in device memory, the rest in pinned host memory streamed through staging buffers by every search.

  * ids tie-equivalent to the oracle, scores bit-equal to the all-device index wherever both return the same id, and
    n >= ntotal identical (torch.equal) to a plain fp16 Flat index, over n, d, nq, k and n_dev, with staging buffers
    small enough for >= 3 chunks, a partial last chunk, and chunks crossing add-batch / host-block boundaries;
  * the exhaustive path of the fused filter inside a host chunk, custom ids, pageable / pinned / device adds, tier
    byte counts, a search on a side stream, refusals, persistence and Indexer(cfg)."""
import os
import pickle

import numpy as np
import pytest
import torch

from oracle import ann_oracle as O

pytestmark = pytest.mark.gpu

NQ_ORACLE = 1000
NQ_BIG = 16400            # > 16384 queries per batch: the host tier is streamed once per query batch


def _rsb():
    import retrieval_scaling_b200 as rsb
    return rsb


def _score_of(xq, xb):
    q64, x64 = xq.astype(np.float64), xb.astype(np.float64)
    return lambda qi, i: float(x64[i] @ q64[qi])


def _check_same_index(Da, Ia, Db, Ib, k, score_of):
    """tiered vs all-device on the same rows: ids equal up to tie permutations, scores bit-equal where ids are equal"""
    atol = 1e-5 if k + 8 <= 4096 else 2e-5 * float(np.abs(Db[:, 0]).max())   # no spare candidates at k = 4096
    O.assert_topk_equivalent(Da, Ia, Db, Ib, score_of=score_of, rtol=1e-5, atol=atol)
    same = Ia == Ib
    assert np.array_equal(Da[same], Db[same])


_DATA = {}


def _data(n, d):
    """(xb fp16 [n, d], xq fp32 [NQ_BIG, d], plain fp16 Flat index, oracle (D, I) of the first NQ_ORACLE queries)"""
    if (n, d) not in _DATA:
        _DATA.clear()                        # one (n, d) at a time: the tiered indexes below hold pinned memory
        rng = np.random.default_rng(n + d)
        centres = rng.standard_normal((32, d)).astype(np.float32)
        xb = (0.3 * (centres[rng.integers(0, 32, n)] + 0.5 * rng.standard_normal((n, d)))).astype(np.float16)
        xq = (centres[rng.integers(0, 32, NQ_BIG)] + 0.5 * rng.standard_normal((NQ_BIG, d))).astype(np.float32)
        plain = _rsb().IndexFlatIP(d, dtype="float16")
        plain.add(xb)
        plain.finalize()
        Dr, Ir = O.flat_search(xq[:NQ_ORACLE], xb.astype(np.float32), min(4096, n))
        _DATA[(n, d)] = {"xb": xb, "xq": xq, "plain": plain, "Dr": Dr, "Ir": Ir, "tiered": {}}
    return _DATA[(n, d)]


def _n_dev_cases(n):
    return {"0": 0, "1": 1, "third": n // 3, "n-1": n - 1, "n": n, "n+5": n + 5}


def _tiered(n, d, case):
    """A tiered copy of _data(n, d)'s rows, added in three batches (pageable numpy, pinned CPU tensor, CUDA tensor)
    whose cuts do not line up with the chunks; the staging buffers hold 2/7 of the host tier, so it is streamed in 4
    chunks, the last one partial."""
    D = _data(n, d)
    if case not in D["tiered"]:
        xb = D["xb"]
        n_dev = _n_dev_cases(n)[case]
        n_host = max(0, n - n_dev)
        chunk_rows = max(1, (2 * n_host) // 7)
        ix = _rsb().IndexFlatIP(d, dtype="float16", device_rows=n_dev, staging_bytes=chunk_rows * d * 2)
        cuts = [0, (2 * n) // 7 + 3, (5 * n) // 7 + 1, n]
        ix.add(xb[cuts[0]:cuts[1]])
        ix.add(torch.from_numpy(xb[cuts[1]:cuts[2]]).pin_memory())
        ix.add(torch.from_numpy(xb[cuts[2]:]).cuda())
        ix.finalize()
        D["tiered"][case] = ix
    return D["tiered"][case]


@pytest.mark.parametrize("case", list(_n_dev_cases(10)))
@pytest.mark.parametrize("d", [64, 768])
@pytest.mark.parametrize("n", [1000, 100_000])
def test_tiered_flat_matches_oracle_and_the_all_device_index(n, d, case):
    D = _data(n, d)
    ix = _tiered(n, d, case)
    n_dev = _n_dev_cases(n)[case]
    xb, xq, plain = D["xb"], D["xq"], D["plain"]
    assert ix.ntotal == n and ix.n_dev == min(n_dev, n)
    score_of = _score_of(xq, xb)
    for nq in (1, 7, NQ_ORACLE, NQ_BIG):
        q = torch.from_numpy(xq[:nq]).cuda()
        for k in (1, 10, 100, 1000, 4096):
            Ia, Da = ix.search_ids(q, k)
            Ip, Dp = plain.search_ids(q, k)
            if n_dev >= n:                   # all rows in device memory: the all-device search itself
                assert torch.equal(Ia, Ip) and torch.equal(Da, Dp), (nq, k)
                continue
            Ia, Da, Ip, Dp = (t.cpu().numpy() for t in (Ia, Da, Ip, Dp))
            if k > n:                        # padding
                assert (Ia[:, n:] == -1).all() and (Da[:, n:] == np.finfo(np.float32).min).all()
            if nq <= NQ_ORACLE:
                kk = min(k, n)
                atol = 2e-5 * float(np.abs(D["Dr"][:nq, 0]).max())
                O.assert_topk_equivalent(Da[:, :kk], Ia[:, :kk], D["Dr"][:nq, :kk], D["Ir"][:nq, :kk], score_of=score_of,
                                         rtol=1e-5, atol=atol)
            _check_same_index(Da, Ia, Dp, Ip, k, score_of)


def test_concentrated_rows_in_a_host_chunk_take_the_exhaustive_path():
    """test_flat_fp16_concentrated_rows_take_the_exhaustive_path with the 30 near-duplicate best rows (columns 1024..1151)
    inside the first host chunk [1000, 1700) of a tiered index: the bound check flags those query rows inside the chunk
    and the fp16 exact_rows kernel re-does them there."""
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
    a = rsb.IndexFlatIP(d, dtype="float16", device_rows=1000, staging_bytes=700 * d * 2)   # chunk [1000, 1700) holds them
    a.add(xb)
    b = rsb.IndexFlatIP(d, dtype="float16")
    b.add(xb)
    q = torch.from_numpy(xq).cuda()
    Ia, Da = (t.cpu().numpy() for t in a.search_ids(q, k))
    Ib, Db = (t.cpu().numpy() for t in b.search_ids(q, k))
    Dr, Ir = O.flat_search(xq, xb.astype(np.float32), k)
    O.assert_topk_equivalent(Da, Ia, Dr, Ir, score_of=_score_of(xq, xb), rtol=1e-5, atol=1e-5)
    assert set(Ia[0].tolist()) <= set(cols.tolist())
    _check_same_index(Da, Ia, Db, Ib, k, _score_of(xq, xb))


def test_custom_ids_fp32_adds_and_tier_bytes():
    rsb = _rsb()
    rng = np.random.default_rng(3)
    n, d, n_dev = 20000, 128, 7000
    x32 = (0.2 * rng.standard_normal((n, d))).astype(np.float32)
    # values that round (ties to even, subnormals, overflow to inf) differently under a wrong conversion
    x32[0, :8] = [1e-8, -3e-7, 6.1e-5, 65519.0, 65520.0, 1e6, 2049.0, 2051.0]
    x32[n - 1, :8] = [1e-8, -3e-7, 6.1e-5, 65519.0, 65520.0, 1e6, 2049.0, 2051.0]
    ids = (rng.permutation(n) * 3 + 7).astype(np.int64)
    a = rsb.IndexFlatIP(d, dtype="float16", device_rows=n_dev, staging_bytes=3000 * d * 2)
    b = rsb.IndexFlatIP(d, dtype="float16")
    for r0, r1 in ((0, 5000), (5000, 12000), (12000, n)):      # fp32 numpy: host-tier rows rounded on the host
        a.add(x32[r0:r1], ids[r0:r1])
        b.add(x32[r0:r1], ids[r0:r1])                          # rounded on the device
    a.finalize(); b.finalize()
    assert a.n_dev == n_dev and a.host_bytes == (n - n_dev) * d * 2
    assert a.index_bytes == n_dev * d * 2 + n * 8 and b.index_bytes == n * d * 2 + n * 8
    assert b.host_bytes == 0 and b.n_dev == n
    rows_a = a.export_rows(0, n)
    rows_b = b.export_rows(0, n)
    assert torch.equal(rows_a.view(torch.int16), rows_b.view(torch.int16))
    assert torch.equal(a.export_rows(6990, 20, out=torch.empty((20, d), dtype=torch.float16, device="cuda")).cpu(),
                       rows_b[6990:7010])
    assert torch.equal(a.export_ids().cpu(), torch.from_numpy(ids))
    xb = rows_b.float().numpy()
    xb[~np.isfinite(xb)] = 0
    a2 = rsb.IndexFlatIP(d, dtype="float16", device_rows=n_dev, staging_bytes=3000 * d * 2)
    b2 = rsb.IndexFlatIP(d, dtype="float16")
    for ix in (a2, b2):
        ix.add(xb.astype(np.float16), ids)
    xq = (0.2 * rng.standard_normal((300, d))).astype(np.float32)
    q = torch.from_numpy(xq).cuda()
    Ia, Da = (t.cpu().numpy() for t in a2.search_ids(q, 50))
    Ib, Db = (t.cpu().numpy() for t in b2.search_ids(q, 50))
    pos = {int(v): i for i, v in enumerate(ids)}
    score_of = lambda qi, i: float(xb[pos[i]].astype(np.float64) @ xq[qi].astype(np.float64))
    _check_same_index(Da, Ia, Db, Ib, 50, score_of)
    assert set(Ia.reshape(-1).tolist()) <= set(ids.tolist())


def test_search_on_a_side_stream():
    rsb = _rsb()
    rng = np.random.default_rng(4)
    n, d = 50000, 256
    xb = (0.2 * rng.standard_normal((n, d))).astype(np.float16)
    a = rsb.IndexFlatIP(d, dtype="float16", device_rows=10000, staging_bytes=9000 * d * 2)
    a.add(xb)
    a.finalize()
    q = torch.from_numpy((0.2 * rng.standard_normal((500, d))).astype(np.float32)).cuda()
    torch.cuda.synchronize()
    I0, D0 = a.search_ids(q, 100)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        I1, D1 = a.search_ids(q, 100)
    s.synchronize()                          # only the side stream: the copy stream was joined back to it
    assert torch.equal(I0, I1) and torch.equal(D0, D1)


def test_refusals():
    rsb = _rsb()
    from retrieval_scaling_b200 import _lib
    from retrieval_scaling_b200.dist import ShardedSearcher
    with pytest.raises(ValueError, match="float16"):
        rsb.IndexFlatIP(128, device_rows=10)
    f32 = rsb.IndexFlatIP(128)
    with pytest.raises(ValueError, match="RSB_DTYPE_F16"):                    # the C-ABI refuses fp32 Flat as well
        f32.set_option(_lib.OPT_DEVICE_ROWS, 10)
    ivf = rsb.IndexIVFFlat(128, 16, dtype="float16")
    with pytest.raises(ValueError, match="Flat index"):
        ivf.set_option(_lib.OPT_DEVICE_ROWS, 10)
    with pytest.raises(ValueError, match="Flat index"):
        ivf.set_option(_lib.OPT_STAGING_BYTES, 1 << 20)
    h = rsb.IndexFlatIP(128, dtype="float16")
    h.add(np.zeros((4, 128), np.float16))
    with pytest.raises(_lib.RsbError, match="device_rows"):                   # RSB_ERR_STATE after the first add
        h.set_option(_lib.OPT_DEVICE_ROWS, 2)
    with pytest.raises(NotImplementedError, match="64"):                      # d % 64
        rsb.IndexFlatIP(72, dtype="float16", device_rows=2)
    t = rsb.IndexFlatIP(128, dtype="float16", device_rows=2)
    with pytest.raises(ValueError, match="one row"):
        t.set_option(_lib.OPT_STAGING_BYTES, 255)
    with pytest.raises(ValueError, match="outside"):
        t.export_rows(0, 1)
    t.add(np.ones((5, 128), np.float16))
    for world in (1, 2):
        with pytest.raises(NotImplementedError, match="tiered Flat"):
            ShardedSearcher(t, world=world)


def test_persistence(tmp_path):
    rsb = _rsb()
    rng = np.random.default_rng(6)
    n, d = 30000, 128
    xb = (0.2 * rng.standard_normal((n, d))).astype(np.float16)
    a = rsb.IndexFlatIP(d, dtype="float16", device_rows=11111)
    for r0 in range(0, n, 7000):
        a.add(xb[r0:r0 + 7000])
    b = rsb.IndexFlatIP(d, dtype="float16")
    b.add(xb)
    pa, pb = str(tmp_path / "a.faiss"), str(tmp_path / "b.faiss")
    rsb.write_index(a, pa)
    rsb.write_index(b, pb)
    assert open(pa, "rb").read() == open(pb, "rb").read()
    back = rsb.read_index(pa, storage_dtype="float16", device_rows=20000)
    assert back.tiered and back.ntotal == n and back.n_dev == 20000 and back.host_bytes == (n - 20000) * d * 2
    assert torch.equal(back.export_rows(0, n), torch.from_numpy(xb))
    q = torch.from_numpy((0.2 * rng.standard_normal((64, d))).astype(np.float32)).cuda()
    xq = q.cpu().numpy()
    Ia, Da = (t.cpu().numpy() for t in back.search_ids(q, 100))
    Ib, Db = (t.cpu().numpy() for t in b.search_ids(q, 100))
    _check_same_index(Da, Ia, Db, Ib, 100, _score_of(xq, xb))
    # custom ids: the RSB1 container (faiss' IndexFlatIP has no id map)
    ids = (np.arange(n) * 5 + 1).astype(np.int64)
    c = rsb.IndexFlatIP(d, dtype="float16", device_rows=0)
    c.add(xb, ids)
    pc = str(tmp_path / "c.faiss")
    with pytest.warns(UserWarning, match="RSB1"):
        rsb.write_index(c, pc)
    with open(pc, "rb") as f:
        blob = pickle.load(f)
    assert np.array_equal(blob["ids"], ids) and np.array_equal(blob["payload"], xb)
    back_c = rsb.read_index(pc, storage_dtype="float16", device_rows=100)
    assert torch.equal(back_c.export_ids().cpu(), torch.from_numpy(ids))
    plain_c = rsb.read_index(pc)
    assert not plain_c.tiered and plain_c.dtype == "float16"
    Ia, Da = (t.cpu().numpy() for t in back_c.search_ids(q, 10))
    Ic, Dc = (t.cpu().numpy() for t in c.search_ids(q, 10))
    pos = {int(v): i for i, v in enumerate(ids)}
    _check_same_index(Da, Ia, Dc, Ic, 10, lambda qi, i: _score_of(xq, xb)(qi, pos[i]))


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
IDX_D = 64


def _datastore(root, n=3000):
    rng = np.random.default_rng(0)
    centres = rng.standard_normal((8, IDX_D)).astype(np.float32)
    emb_dir = os.path.join(root, "embeddings", "enc", "dom", "2-shards")
    psg_dir = os.path.join(root, "passages", "dom", "2-shards")
    os.makedirs(emb_dir); os.makedirs(psg_dir)
    for s in range(2):
        e = ((centres[rng.integers(0, 8, n)] + 0.3 * rng.standard_normal((n, IDX_D))) / 8.0).astype(np.float16)
        with open(os.path.join(emb_dir, f"passages_{s:02d}.pkl"), "wb") as f:
            pickle.dump((list(range(n)), e), f)
        with open(os.path.join(psg_dir, f"raw_passages-{s}-of-2.jsonl"), "w") as f:
            for c in range(n):
                f.write('{"text": "p%d_%d"}\n' % (s, c))
    return ((centres[rng.integers(0, 8, 12)] + 0.3 * rng.standard_normal((12, IDX_D))) / 8.0).astype(np.float32)


def _cfg(root, extra=()):
    from retrieval_scaling_b200 import config as C
    ov = [f"datastore.datastore_root_dir={root}", "datastore.domain=dom", "model.datastore_encoder=enc",
          "datastore.embedding.num_shards=2", "datastore.index.index_type=Flat",
          "datastore.index.index_shard_ids=[0,1]", f"datastore.index.projection_size={IDX_D}",
          "+datastore.index.storage_dtype=float16", "evaluation.search.n_docs=5"] + list(extra)
    return C.load_config("default", os.path.join(ROOT, "ric", "conf"), ov)


def test_indexer_device_rows(tmp_path):
    from retrieval_scaling_b200.indicies.base import Indexer
    r0, r1 = os.path.join(str(tmp_path), "a"), os.path.join(str(tmp_path), "b")
    q = _datastore(r0)
    _datastore(r1)
    plain = Indexer(_cfg(r0))
    key = ["+datastore.index.device_rows=2500"]                  # shard 0 partly, shard 1 wholly in host memory
    tiered = Indexer(_cfg(r1, key))
    ix = tiered.datastore.index
    assert ix.tiered and ix.n_dev == 2500 and ix.host_bytes == 3500 * IDX_D * 2
    s0, s1 = plain.search(q, 5), tiered.search(q, 5)
    assert s0[2] == s1[2] and s0[0] == s1[0]                      # the same db_ids and scores
    assert open(plain.datastore.index_path, "rb").read() == open(tiered.datastore.index_path, "rb").read()
    again = Indexer(_cfg(r1, key))                                # the .faiss artefact reloads tiered
    assert again.datastore.index.tiered and again.datastore.index.n_dev == 2500
    assert again.search(q, 5)[2] == s0[2]
