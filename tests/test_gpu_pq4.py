"""IVF-PQ with 4-bit sub-quantizers on the GPU (faiss nbits = 4): the pair tables of pq_lut4_kernel bit for bit, the
packed 4-bit codes against the oracle's, search parity with oracle/pq4_oracle.py for the generic and the three tuned
byte counts, the paired scan against the single-item scan, reproducible builds, file round trips, re-ranking over a
4-bit base and the `Indexer(cfg)` path with `n_bits: 4`."""
import ctypes
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import ann_oracle as O
from oracle import parity as P
from oracle import pq4_oracle as P4
from oracle import refine_oracle as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = 768
NLIST = 16


def _data(M, seed=0, n=4000, nq=1000):
    """Vectors around the first 12 of 16 unit centroids (lists 12..15 stay empty), a random [M, 16, d/M] codebook."""
    rng = np.random.default_rng(seed)
    c = rng.standard_normal((NLIST, D)).astype(np.float32)
    cent = c / np.linalg.norm(c, axis=1, keepdims=True)
    xb = (cent[rng.integers(0, 12, n)] + 0.05 * rng.standard_normal((n, D))).astype(np.float32)
    xq = (cent[rng.integers(0, 12, nq)] + 0.05 * rng.standard_normal((nq, D))).astype(np.float32)
    cb = (0.05 * rng.standard_normal((M, 16, D // M))).astype(np.float32)
    return cent, cb, xb, xq


def _index(M, cent, cb, xb):
    import retrieval_scaling_b200 as r
    ix = r.IndexIVFPQ(D, NLIST, M, nbits=4)
    ix.set_centroids(cent)
    ix.set_codebook(cb)
    ix.add(xb)
    ix.finalize()
    return ix


def _exported(ix):
    off, codes, ids = (t.cpu().numpy() for t in ix.export_lists())
    return off, codes, ids


def _fma_tables(xq, cb):
    """T[q][m][c] = <q_m, cb[m][c]> accumulated as the kernels do: s = fmaf(q[t], cb[t], s) for t = 0, 1, ..."""
    M, ksub, dsub = cb.shape
    q = xq.reshape(xq.shape[0], M, dsub).astype(np.float64)
    c = cb.astype(np.float64)
    s = np.zeros((xq.shape[0], M, ksub), np.float32)
    for t in range(dsub):
        s = (q[:, :, None, t] * c[None, :, :, t] + s.astype(np.float64)).astype(np.float32)
    return s


@pytest.mark.parametrize("M", [16, 32, 48, 64, 128])
def test_lut4_table_is_the_pair_table_bit_for_bit(M):
    from retrieval_scaling_b200 import _lib
    from retrieval_scaling_b200.index import _ptr, _stream
    cent, cb, xb, xq = _data(M, seed=M, n=64, nq=5)
    ix = _index(M, cent, cb, xb)
    L, Mb = ix.L, M // 2
    words = L.rsb_pq_lut_floats(ix._h)
    q = torch.from_numpy(xq).cuda()
    lut = torch.full((5, words), float("nan"), device="cuda")
    _lib.check(L.rsb_pq_tables(ix._h, _ptr(q), 5, _ptr(lut), _stream()))
    got = lut.cpu().numpy()
    T = _fma_tables(xq, cb)
    j = np.arange(256)
    Tp = (T[:, 0::2][:, :, j & 15] + T[:, 1::2][:, :, j >> 4]).astype(np.float32)      # [nq, Mb, 256]
    pos = np.array([[L.rsb_pq_lut_index(Mb, jj, b) for jj in range(256)] for b in range(Mb)])
    assert np.array_equal(got[:, pos].view(np.uint32), Tp.view(np.uint32))
    if Mb in (16, 32, 64):                        # replica words of the interleaved rows: word w holds b = w % Mb
        rows = got.reshape(5, 256, 64)
        assert np.array_equal(rows.view(np.uint32), rows[:, :, np.arange(64) % Mb].view(np.uint32))


@pytest.mark.parametrize("M", [32, 48, 64])
def test_gpu_codes_equal_oracle_codes(M):
    cent, cb, xb, _ = _data(M, seed=1 + M)
    ix = _index(M, cent, cb, xb)
    off, codes, ids = _exported(ix)
    assert codes.shape == (len(xb), M // 2)
    lists = np.repeat(np.arange(NLIST), np.diff(off))
    _, ref = P4.ivfpq4_encode(xb[ids], cent, cb, assign=lists)
    g, o = P4.unpack4(codes), P4.unpack4(ref)
    assert (g == o).mean() > 0.999
    # every disagreement is an L2 near-tie of the residual sub-vector
    r = (xb[ids] - cent[lists]).reshape(len(ids), M, D // M).astype(np.float64)
    for i, m in zip(*np.nonzero(g != o)):
        dg = ((r[i, m] - cb[m, g[i, m]]) ** 2).sum()
        do = ((r[i, m] - cb[m, o[i, m]]) ** 2).sum()
        assert abs(dg - do) <= 1e-5 * max(do, 1e-12)


@pytest.mark.parametrize("M", [16, 32, 48, 64, 128])
def test_search_parity_with_oracle(M):
    cent, cb, xb, xq = _data(M, seed=2 + M)
    ix = _index(M, cent, cb, xb)
    off, codes, ids = _exported(ix)
    assert (np.diff(off) == 0).any()                                     # empty lists are part of the case
    host = P4.host_ivfpq(cent, cb, off, codes, ids)
    for nq, k, nprobe in ((1, 10, 4), (7, 100, 4), (7, 4096, NLIST), (1000, 100, 4), (1000, 10, NLIST)):
        ix.nprobe = nprobe
        Dg, Ig = ix.search(xq[:nq], k)
        Dr, Ir = P4.ivfpq4_search(xq[:nq], cent, cb, off, codes, ids, nprobe, k)
        par = P.topk_parity(Dg, Ig, Dr, Ir, rtol=1e-5, atol=2e-4,
                            score_of=lambda qs, tids: host.rescore(xq[:nq], qs, tids))
        key = (M, nq, k, nprobe)
        assert par["non_tie_mismatches"] == 0 and par["scores_out_of_tol"] == 0, (key, par)
        assert par["padding_mismatches"] == 0, (key, par)
        assert host.verify_pairs(xq[:nq], Dg, Ig)["rescore_out_of_tol"] == 0, key


CHILD = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, sys.argv[1] + "/tests")
import test_gpu_pq4 as T
out = {}
for M in (32, 64, 128):
    cent, cb, xb, xq = T._data(M, seed=5 + M, nq=2000)
    xq[1::2] = xq[0::2]                                                 # pairs of identical queries
    ix = T._index(M, cent, cb, xb)
    for nq, k in ((1, 10), (1000, 100), (2000, 10), (7, 4096)):
        ix.nprobe = 8
        D, I = ix.search(xq[:nq], k)
        out[f"M{M}_nq{nq}_k{k}_D"] = D
        out[f"M{M}_nq{nq}_k{k}_I"] = I
np.savez(sys.argv[2], **out)
"""


def test_paired_scan_is_bit_identical_to_single_item_scan(tmp_path):
    res = {}
    for single in (False, True):
        env = dict(os.environ)
        env.pop("RSB_PQ_SINGLE_ITEMS", None)
        if single:
            env["RSB_PQ_SINGLE_ITEMS"] = "1"
        path = str(tmp_path / f"s{int(single)}.npz")
        r = subprocess.run([sys.executable, "-c", CHILD, ROOT, path], env=env, capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, r.stderr[-4000:]
        res[single] = np.load(path)
    a, b = res[False], res[True]
    assert sorted(a.files) == sorted(b.files)
    for name in a.files:
        assert a[name].tobytes() == b[name].tobytes(), name


def test_two_builds_are_bit_identical():
    """Training (coarse k-means + 4-bit PQ k-means, ksub = 16), encoding and search: the same bits on every run."""
    import retrieval_scaling_b200 as r
    cent, _, xb, xq = _data(64, seed=9, n=6000)
    outs = []
    for _ in range(2):
        ix = r.IndexIVFPQ(D, NLIST, 64, nbits=4)
        ix.train(xb)
        ix.add(xb)
        ix.nprobe = 4
        Dq, Iq = ix.search(xq[:200], 50)
        off, codes, ids = _exported(ix)
        outs.append((ix.get_codebook().cpu().numpy(), codes, ids, off, Dq, Iq))
        assert tuple(outs[-1][0].shape) == (64, 16, D // 64)
    for a, b in zip(*outs):
        assert a.tobytes() == b.tobytes()


@pytest.mark.parametrize("fmt", ["faiss", "rsb1"])
def test_file_round_trip(tmp_path, fmt):
    import retrieval_scaling_b200 as r
    cent, cb, xb, xq = _data(48, seed=11)
    ix = _index(48, cent, cb, xb)
    ix.nprobe = 6
    path = str(tmp_path / f"pq4.{fmt}")
    r.write_index(ix, path, fmt=fmt)
    back = r.read_index(path)
    assert back.nbits == 4 and back.M == 48 and back.nprobe == 6
    for a, b in zip(_exported(ix), _exported(back)):
        assert a.tobytes() == b.tobytes()
    Da, Ia = ix.search(xq[:300], 100)
    Db, Ib = back.search(xq[:300], 100)
    assert Da.tobytes() == Db.tobytes() and Ia.tobytes() == Ib.tobytes()
    if fmt == "faiss":                                              # the file's inverted lists hold faiss' packed bytes
        from retrieval_scaling_b200 import faiss_io
        parts = faiss_io.read_faiss(path)
        assert parts["nbits"] == 4 and parts["codes"].shape == (len(xb), 24)


def test_refine_over_4bit_base_matches_oracle():
    import retrieval_scaling_b200 as r
    cent, cb, xb, xq = _data(64, seed=13)
    ix = _index(64, cent, cb, xb)
    ix.nprobe = 8
    ref = r.IndexRefine(ix, "float32", 4)
    ref.add_store(xb)
    k = 20
    Dg, Ig = ref.search(xq[:256], k)
    _, Ib = ix.search(xq[:256], k * 4)
    Dr, Ir = R.refine_candidates(xq[:256], xb, Ib, k)
    par = P.topk_parity(Dg, Ig, Dr, Ir, rtol=1e-5, atol=1e-5,
                        score_of=lambda qs, ids: np.einsum("ij,ij->i", xq[qs].astype(np.float64), xb[ids].astype(np.float64)))
    assert par["non_tie_mismatches"] == 0 and par["scores_out_of_tol"] == 0 and par["padding_mismatches"] == 0, par


def _make_datastore(root, nshards=2, n=3000, d=64):
    rng = np.random.default_rng(0)
    centres = rng.standard_normal((8, d)).astype(np.float32)
    emb_dir = os.path.join(root, "embeddings", "enc", "dom", f"{nshards}-shards")
    psg_dir = os.path.join(root, "passages", "dom", f"{nshards}-shards")
    os.makedirs(emb_dir); os.makedirs(psg_dir)
    embs = []
    for s in range(nshards):
        e = ((centres[rng.integers(0, 8, n)] + 0.3 * rng.standard_normal((n, d))) / 8.0).astype(np.float16)
        embs.append(e)
        with open(os.path.join(emb_dir, f"passages_{s:02d}.pkl"), "wb") as f:
            pickle.dump((list(range(n)), e), f)
        with open(os.path.join(psg_dir, f"raw_passages-{s}-of-{nshards}.jsonl"), "w") as f:
            for c in range(n):
                f.write(json.dumps({"text": f"passage s{s} c{c}", "id": c, "shard_id": s}) + "\n")
    q = ((centres[rng.integers(0, 8, 12)] + 0.3 * rng.standard_normal((12, d))) / 8.0).astype(np.float32)
    return embs, q


def test_indexer_n_bits_4_equals_direct_index(tmp_path):
    import retrieval_scaling_b200 as r
    from retrieval_scaling_b200 import config as C
    from retrieval_scaling_b200.indicies.base import Indexer
    embs, q = _make_datastore(str(tmp_path))
    ov = [f"datastore.datastore_root_dir={tmp_path}", "datastore.domain=dom", "model.datastore_encoder=enc",
          "datastore.embedding.num_shards=2", "datastore.index.index_type=IVFPQ", "datastore.index.index_shard_ids=[0,1]",
          "datastore.index.projection_size=64", "datastore.index.ncentroids=16", "datastore.index.probe=4",
          "datastore.index.n_subquantizers=16", "datastore.index.n_bits=4", "datastore.index.sample_train_size=4000",
          "evaluation.search.n_docs=5"]
    cfg = C.load_config("default", os.path.join(ROOT, "ric", "conf"), ov)
    ix = Indexer(cfg).datastore.index
    assert ix.nbits == 4 and ix.M == 16
    direct = r.IndexIVFPQ(64, 16, 16, nbits=4)
    direct.set_centroids(ix.get_centroids())
    direct.set_codebook(ix.get_codebook())
    for e in embs:
        direct.add(e.astype(np.float32))
    direct.nprobe = 4
    for a, b in zip(_exported(ix), _exported(direct)):
        assert a.tobytes() == b.tobytes()
    Ia, Da = ix.search_ids(q, 5)
    Ib, Db = direct.search_ids(q, 5)
    assert torch.equal(Ia, Ib) and torch.equal(Da, Db)
    again = Indexer(cfg).datastore.index                               # reload of the written .faiss file
    assert again.nbits == 4 and torch.equal(again.search_ids(q, 5)[0], Ia)
    # composes with exact re-ranking
    cfg2 = C.load_config("default", os.path.join(ROOT, "ric", "conf"),
                         ov + ["+datastore.index.refine_k_factor=4", "+datastore.index.refine_dtype=float32"])
    refd = Indexer(cfg2).datastore.index
    ref = r.IndexRefine(direct, "float32", 4)
    ref.add_store(np.concatenate(embs).astype(np.float32))
    Ir, Dr = refd.search_ids(q, 5)
    Ir2, Dr2 = ref.search_ids(q, 5)
    assert torch.equal(Ir, Ir2) and torch.equal(Dr, Dr2)
