"""IVF-PQ with 4-bit sub-quantizers (faiss nbits = 4) without a GPU: the oracle's known answers, a numpy restatement of
the pair tables the 8-bit scan kernels read, the C-ABI's accept / refuse rules, PQ training with ksub = 16 on the host
logic, the IwPQ file round trip and the Indexer's handling of `n_bits: 4`."""
import ctypes
import io

import numpy as np
import pytest
import torch

from oracle import ann_oracle as O
from oracle import pq4_oracle as P4
from retrieval_scaling_b200 import _lib, faiss_io, train


# ---- oracle known answers ------------------------------------------------------------------------------------------
def _faiss_generic_pack(codes, nbits=4):
    """PQEncoderGeneric::encode, bit by bit: code m occupies bits [m * nbits, (m + 1) * nbits) of the code, LSB first."""
    M = len(codes)
    out = np.zeros((M * nbits + 7) // 8, np.uint8)
    for m, c in enumerate(codes):
        for bit in range(nbits):
            if (int(c) >> bit) & 1:
                pos = m * nbits + bit
                out[pos // 8] |= np.uint8(1 << (pos % 8))
    return out


def test_nibble_order_is_faiss_pq_encoder_generic():
    assert P4.pack4(np.array([[1, 2, 3, 4]], np.uint8)).tolist() == [[0x21, 0x43]]
    rng = np.random.default_rng(0)
    codes = rng.integers(0, 16, (50, 24)).astype(np.uint8)
    packed = P4.pack4(codes)
    assert packed.shape == (50, 12)
    for row, p in zip(codes, packed):
        assert p.tobytes() == _faiss_generic_pack(row).tobytes()
    assert np.array_equal(P4.unpack4(packed), codes)


def test_pq4_with_residuals_as_codebook_is_exact():
    """16 vectors, one list per pair of vectors; sub-quantizer m's entry j is the residual sub-vector of vector j, so
    every vector encodes to j in every sub-quantizer and the ADC score equals the exact inner product."""
    rng = np.random.default_rng(1)
    d, M, nlist = 32, 8, 4
    x = rng.standard_normal((16, d)).astype(np.float32)
    cent = rng.standard_normal((nlist, d)).astype(np.float32)
    assign = O.ivf_assign(x, cent)
    r = x - cent[assign]
    cb = np.ascontiguousarray(r.reshape(16, M, d // M).transpose(1, 0, 2))       # [M, 16, dsub]
    a2, packed = P4.ivfpq4_encode(x, cent, cb)
    assert np.array_equal(a2, assign)
    assert np.array_equal(P4.unpack4(packed), np.repeat(np.arange(16, dtype=np.uint8)[:, None], M, axis=1))
    off, perm, ids = O.build_csr(assign, nlist)
    xq = rng.standard_normal((5, d)).astype(np.float32)
    D, I = P4.ivfpq4_search(xq, cent, cb, off, packed[perm], ids, nlist, 16)
    Df, If = O.flat_search(xq, x, 16)
    O.assert_topk_equivalent(D, I, Df, If, rtol=1e-5, atol=1e-5)


def test_ivfpq4_full_probe_is_brute_force_over_decoded_vectors():
    rng = np.random.default_rng(2)
    d, M, nlist, n = 48, 16, 6, 400
    x = rng.standard_normal((n, d)).astype(np.float32)
    cent = rng.standard_normal((nlist, d)).astype(np.float32)
    cb = (0.5 * rng.standard_normal((M, 16, d // M))).astype(np.float32)
    assign, packed = P4.ivfpq4_encode(x, cent, cb)
    recon = cent[assign] + P4.pq4_decode(packed, cb)
    off, perm, ids = O.build_csr(assign, nlist)
    xq = rng.standard_normal((7, d)).astype(np.float32)
    D, I = P4.ivfpq4_search(xq, cent, cb, off, packed[perm], ids, nlist, 20)
    Df, If = O.flat_search(xq, recon, 20)
    O.assert_topk_equivalent(D, I, Df, If, rtol=1e-5, atol=1e-4)
    # the fp64 re-score from the exported (packed) codes is the definition of the score
    host = P4.host_ivfpq(cent, cb, off, packed[perm], ids)
    assert host.verify_pairs(xq, D, I, rtol=1e-5, atol=1e-4)["rescore_out_of_tol"] == 0


# ---- the pair tables -----------------------------------------------------------------------------------------------
def pair_table(T):
    """T [M, 16] fp32 -> T' [M/2, 256]: T'[b][j] = T[2b][j & 15] + T[2b+1][j >> 4] (one fp32 rounding)."""
    j = np.arange(256)
    return (T[0::2][:, j & 15] + T[1::2][:, j >> 4]).astype(np.float32)


def test_pair_table_entries_and_score_bound():
    rng = np.random.default_rng(3)
    M, n = 64, 5000
    T = rng.standard_normal((M, 16)).astype(np.float32)
    Tp = pair_table(T)
    for b in (0, 7, M // 2 - 1):
        for jj in (0, 15, 16, 0x5a, 255):
            assert Tp[b, jj] == np.float32(T[2 * b, jj & 15] + T[2 * b + 1, jj >> 4])
    codes = rng.integers(0, 16, (n, M)).astype(np.uint8)
    packed = P4.pack4(codes)
    dis0 = np.float32(0.75)
    seq = np.full(n, dis0, np.float32)                                  # faiss: dis0, then one term at a time
    for m in range(M):
        seq = (seq + T[m][codes[:, m]]).astype(np.float32)
    pair = np.full(n, dis0, np.float32)                                 # the kernel: byte sub-quantizer pair sums
    for b in range(M // 2):
        pair = (pair + Tp[b][packed[:, b]]).astype(np.float32)
    exact = float(dis0) + T.astype(np.float64)[np.arange(M)[None, :], codes].sum(1)
    mag = abs(float(dis0)) + np.abs(T.astype(np.float64))[np.arange(M)[None, :], codes].sum(1)
    u = 2.0 ** -24
    # |fl(sum of m terms) - sum| <= (m - 1) u sum|terms| / (1 - (m - 1) u), per order; the pair form rounds each entry once
    bound = 1.01 * M * u * mag
    assert (np.abs(seq - exact) <= bound).all() and (np.abs(pair - exact) <= bound).all()
    assert (np.abs(pair.astype(np.float64) - seq) <= 2 * bound).all()
    assert (pair != seq).any()                                          # rounding differs, as stated


@pytest.mark.parametrize("Mb", [16, 32, 64, 24])
def test_pair_table_layout_positions(Mb):
    """Where the scan reads entry (j, b) of the byte sub-quantizer table: the 8-bit layout, used unchanged."""
    L = _lib.lib()
    pos = np.array([[L.rsb_pq_lut_index(Mb, j, b) for b in range(Mb)] for j in range(256)])
    assert len(np.unique(pos)) == 256 * Mb and pos.min() == 0
    if Mb in (16, 32, 64):      # rows of 64 words, word w holding byte sub-quantizer w % Mb (replicas for Mb < 64)
        assert np.array_equal(pos, np.arange(256)[:, None] * 64 + np.arange(Mb)[None, :])
    else:                       # generic [b][256]
        assert np.array_equal(pos, np.arange(Mb)[None, :] * 256 + np.arange(256)[:, None])


# ---- C-ABI ---------------------------------------------------------------------------------------------------------
def _create(d, nlist, M, nbits):
    L = _lib.lib()
    h = ctypes.c_void_p(0)
    rc = L.rsb_ivfpq_create(d, nlist, M, nbits, ctypes.byref(h))
    if rc == _lib.RSB_OK:
        L.rsb_free(h)
    return rc, L.rsb_last_error()


ACCEPTED = (_lib.RSB_OK, _lib.RSB_ERR_OOM, _lib.RSB_ERR_CUDA)    # shape accepted; without a GPU the handle's allocation fails


@pytest.mark.parametrize("M", [16, 32, 48, 64, 96, 128, 256])
def test_ivfpq_create_accepts_4bit_shapes(M):
    rc, _ = _create(768, 16, M, 4)
    assert rc in ACCEPTED


@pytest.mark.parametrize("d,M,nbits,want,word", [
    (768, 64, 6, _lib.RSB_ERR_UNSUPPORTED, b"nbits"),
    (768, 64, 16, _lib.RSB_ERR_UNSUPPORTED, b"nbits"),
    (768, 12, 4, _lib.RSB_ERR_INVALID, b"M % 8"),        # M % 8 != 0
    (768, 384, 4, _lib.RSB_ERR_INVALID, b"M / 2"),       # 192 code bytes > 128
    (768, 40, 4, _lib.RSB_ERR_INVALID, b"divisible"),    # d % M != 0
    (768, 3, 8, _lib.RSB_ERR_UNSUPPORTED, b"n_subquantizers"),      # 8-bit M not a multiple of 4
    (768, 256, 8, _lib.RSB_ERR_UNSUPPORTED, b"n_subquantizers"),    # 8-bit M > 128
])
def test_ivfpq_create_refuses_bad_nbits_and_shapes(d, M, nbits, want, word):
    rc, msg = _create(d, 16, M, nbits)
    assert rc == want and word in msg


def test_pq_training_steps_refuse_other_ksub():
    L = _lib.lib()
    p = ctypes.c_void_p(16)          # never dereferenced: the arguments are refused first
    assert L.rsb_pq_assign(p, 10, 64, 16, 32, p, p, None) == _lib.RSB_ERR_UNSUPPORTED
    assert L.rsb_pq_accumulate(p, 10, 64, 16, 64, p, p, p, None) == _lib.RSB_ERR_UNSUPPORTED
    assert L.rsb_pq_assign(p, 10, 64, 15, 16, p, p, None) == _lib.RSB_ERR_INVALID      # d % M
    assert L.rsb_pq_lut_floats(None) == -1


# ---- PQ training with ksub = 16 (host logic; the three heavy steps are a numpy stand-in) ----------------------------
class NumpyOps:
    def pq_assign(self, r, cb):
        M, ksub, dsub = cb.shape
        rm = r.reshape(-1, M, dsub).permute(1, 0, 2)
        return torch.cdist(rm, cb).argmin(2).T.contiguous().to(torch.uint8)

    def pq_accumulate(self, r, codes, M, ksub):
        dsub = r.shape[1] // M
        rm = r.reshape(-1, M, dsub)
        sums, counts = torch.zeros(M, ksub, dsub), torch.zeros(M, ksub)
        for m in range(M):
            sums[m].index_add_(0, codes[:, m].long(), rm[:, m])
            counts[m] = torch.bincount(codes[:, m].long(), minlength=ksub).float()
        return sums, counts


def test_train_pq_ksub16():
    g = torch.Generator().manual_seed(4)
    r = torch.randn(3000, 32, generator=g) * torch.linspace(0.2, 2.0, 32)
    cb1 = train.train_pq(r, M=8, ksub=16, niter=1, seed=5, ops=NumpyOps())
    cb = train.train_pq(r, M=8, ksub=16, niter=10, seed=5, ops=NumpyOps())
    assert tuple(cb.shape) == (8, 16, 4) and torch.isfinite(cb).all()

    def err(codebook):
        dist = torch.cdist(r.reshape(-1, 8, 4).permute(1, 0, 2), codebook)
        return dist.min(dim=2).values.pow(2).sum().item()
    assert err(cb) < err(cb1)
    # one Lloyd step of the host logic is the oracle's (no empty entries at this size)
    step = train.train_pq(r, M=8, ksub=16, niter=1, seed=5, ops=NumpyOps())
    init = train.train_pq(r, M=8, ksub=16, niter=0, seed=5, ops=NumpyOps())
    assert np.allclose(step.numpy(), P4.pq_lloyd_step(r.numpy(), init.numpy()), atol=1e-5)
    assert tuple(train.train_pq(r[:10], M=8, ksub=16, niter=2, ops=NumpyOps()).shape) == (8, 16, 4)
    with pytest.raises(NotImplementedError, match="ksub"):
        train.train_pq(r, M=8, ksub=64, ops=NumpyOps())


# ---- IwPQ file with nbits = 4 --------------------------------------------------------------------------------------
def test_iwpq_nbits4_round_trip_byte_for_byte():
    rng = np.random.default_rng(5)
    d, M, nlist, n = 64, 16, 8, 300
    assign = np.sort(rng.integers(0, nlist - 2, n))                    # the last two lists stay empty
    offsets = np.zeros(nlist + 1, np.int64)
    np.cumsum(np.bincount(assign, minlength=nlist), out=offsets[1:])
    parts = {"kind": "IVFPQ", "centroids": rng.standard_normal((nlist, d)).astype(np.float32), "offsets": offsets,
             "ids": rng.permutation(10 * n)[:n].astype(np.int64), "nprobe": 3,
             "codebook": rng.standard_normal((M, 16, d // M)).astype(np.float32),
             "codes": rng.integers(0, 256, (n, M // 2)).astype(np.uint8)}
    buf = io.BytesIO()
    faiss_io.write_faiss(buf, parts)
    back = faiss_io.read_faiss(io.BytesIO(buf.getvalue()))
    assert back["nbits"] == 4 and back["M"] == M and back["codes"].shape == (n, M // 2)
    for key in ("codes", "codebook", "offsets", "ids", "centroids"):
        assert np.array_equal(back[key], parts[key]), key
    buf2 = io.BytesIO()
    faiss_io.write_faiss(buf2, back)
    assert buf2.getvalue() == buf.getvalue()
    # code_size in the IwPQ header and in the inverted lists is M * 4 / 8
    assert np.frombuffer(buf.getvalue(), np.uint64, count=1, offset=buf.getvalue().index(b"ilar") + 12)[0] == M // 2


# ---- Indexer config and multi-GPU refusal ---------------------------------------------------------------------------
def test_indexer_passes_n_bits_4(tmp_path, monkeypatch):
    import os
    from retrieval_scaling_b200 import config as C
    from retrieval_scaling_b200.indicies import base, ivf_pq
    conf = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ric", "conf")
    cfg = C.load_config("default", conf, [f"datastore.datastore_root_dir={tmp_path}", "datastore.domain=dom",
                                          "model.datastore_encoder=enc", "datastore.embedding.num_shards=2",
                                          "datastore.index.index_shard_ids=[0,1]", "datastore.index.index_type=IVFPQ",
                                          "datastore.index.n_bits=4", "datastore.index.n_subquantizers=64",
                                          "+datastore.index.refine_k_factor=8", "+datastore.index.refine_dtype=sq8"])
    seen = {}

    class Recorder:
        def __init__(self, **kw):
            seen.update(kw)
    monkeypatch.setattr(base, "IVFPQIndexer", Recorder)
    base.Indexer(cfg)
    assert seen["code_size"] == 4 and seen["n_subquantizers"] == 64
    assert seen["refine_k_factor"] == 8 and seen["refine_dtype"] == "sq8"
    made = {}
    monkeypatch.setattr(ivf_pq.rsb_index, "IndexIVFPQ", lambda *a: made.setdefault("args", a))
    obj = ivf_pq.IVFPQIndexer.__new__(ivf_pq.IVFPQIndexer)
    obj.dimension, obj.ncentroids, obj.n_subquantizers, obj.code_size = 768, 4096, 64, 4
    obj._new_index()
    assert made["args"] == (768, 4096, 64, 4)


def test_sharded_searcher_refuses_4bit_over_gpus():
    from retrieval_scaling_b200 import dist

    class Fake4:
        nbits = 4

        def search_ids(self, q, k):
            raise AssertionError("not reached")
    with pytest.raises(NotImplementedError, match="nbits = 4"):
        dist.ShardedSearcher(Fake4(), world=2, rank=0)
    dist.ShardedSearcher(Fake4(), world=1, rank=0)                # one GPU: the index searches itself
