"""Exact re-ranking (IndexRefine) without a GPU: the oracle's known answers, the IxRF file layout and its fp16
round-trip refusal, the config keys, the C-ABI's argument checks, and a faiss cross-check where faiss is importable."""
import io
import struct

import numpy as np
import pytest

from oracle import ann_oracle as O
from oracle import refine_oracle as R
from retrieval_scaling_b200 import _lib
from retrieval_scaling_b200 import faiss_io as F

NEG = np.finfo(np.float32).min


def test_oracle_rerank_changes_the_pq_order():
    """Hand-built: the base (PQ) order is 0, 1, 2, 3 but the exact scores order them 3, 1, 0, 2, so re-ranking has to
    change both the order and, for k = 2, the set."""
    store = np.array([[1, 0], [2, 0], [0, 1], [3, 1]], dtype=np.float32)
    q = np.array([[1.0, 0.5]], dtype=np.float32)             # exact: 1.0, 2.0, 0.5, 3.5
    D, I = R.refine_candidates(q, store, np.array([[0, 1, 2, 3]]), 2)
    assert I.tolist() == [[3, 1]] and D.tolist() == [[3.5, 2.0]]
    D, I = R.refine_candidates(q, store, np.array([[0, 1, 2, 3]]), 4)
    assert I.tolist() == [[3, 1, 0, 2]]


def test_oracle_padding_ties_and_fp16_store():
    store = np.array([[1, 1], [1, 1], [2, 0], [0, 0]], dtype=np.float16)
    q = np.array([[1, 1], [1, 1]], dtype=np.float32)
    cand = np.array([[1, 0, 2, -1], [3, -1, -1, -1]])          # ties 1 / 0 / 2 all score 2: ascending id
    D, I = R.refine_candidates(q, store, cand, 4)
    assert I.tolist() == [[0, 1, 2, -1], [3, -1, -1, -1]]
    assert D[0, :3].tolist() == [2.0, 2.0, 2.0] and D[0, 3] == NEG and D[1, 1:].tolist() == [NEG] * 3
    # labels after the first -1 are not looked at (faiss: `if (idx < 0) break`)
    D, I = R.refine_candidates(q, store, np.array([[-1, 2, 0, 1]] * 2), 2)
    assert (I == -1).all() and (D == NEG).all()


def test_oracle_refine_search_with_k_factor():
    rng = np.random.default_rng(3)
    xb = rng.standard_normal((300, 16)).astype(np.float32)
    xq = rng.standard_normal((5, 16)).astype(np.float32)
    noisy = xb + 0.5 * rng.standard_normal(xb.shape).astype(np.float32)   # a lossy "base" index
    base = lambda q, kb: O.flat_search(q, noisy, kb)                     # noqa: E731
    Dx, Ix = O.flat_search(xq, xb, 10)
    D, I = R.refine_search(xq, xb, base, 10, 300 // 10)              # k_base = ntotal: re-ranking is exact search
    assert np.array_equal(I, Ix) and np.allclose(D, Dx, rtol=1e-6)
    D1, I1 = R.refine_search(xq, xb, base, 10, 1)                    # k_factor 1: the base's set, exactly ordered
    _, Ib = base(xq, 10)
    assert all(set(a) == set(b) for a, b in zip(I1.tolist(), Ib.tolist()))
    assert (np.diff(D1, axis=1) <= 0).all()
    D64, _ = R.refine_search(xq, xb, base, 10, 4, dtype=np.float64)
    D32, _ = R.refine_search(xq, xb, base, 10, 4)
    assert np.allclose(D64, D32, rtol=1e-5)


def _ivfpq_parts(rng, d=16, nlist=3, sizes=(2, 0, 3)):
    offsets = np.zeros(nlist + 1, np.int64)
    np.cumsum(sizes, out=offsets[1:])
    n = int(offsets[-1])
    return {"kind": "IVFPQ", "centroids": rng.standard_normal((nlist, d)).astype(np.float32), "offsets": offsets,
            "ids": np.arange(n, dtype=np.int64), "nprobe": 2,
            "codebook": rng.standard_normal((4, 256, d // 4)).astype(np.float32),
            "codes": rng.integers(0, 256, (n, 4), dtype=np.uint8)}


def test_ixrf_layout_and_round_trip():
    rng = np.random.default_rng(0)
    base = _ivfpq_parts(rng)
    xb = rng.standard_normal((5, 16)).astype(np.float32)
    buf = io.BytesIO()
    F.write_faiss(buf, {"kind": "Refine", "base": base, "xb": xb, "k_factor": 4.0})
    raw = buf.getvalue()
    # IxRF | index header (d, ntotal, 2 dummies, is_trained, metric) | base (IwPQ ...) | IxFI refine | k_factor f32
    assert raw[:4] == b"IxRF" and struct.unpack_from("<iq", raw, 4) == (16, 5) and raw[37:41] == b"IwPQ"
    flat = b"IxFI" + struct.pack("<iqqqBi", 16, 5, 1 << 20, 1 << 20, 1, 0) + struct.pack("<Q", xb.size) + xb.tobytes()
    assert raw.endswith(flat + struct.pack("<f", 4.0))
    back = F.read_faiss(io.BytesIO(raw))
    assert back["kind"] == "Refine" and back["k_factor"] == 4.0 and back["ntotal"] == 5
    assert np.array_equal(back["xb"], xb) and back["base"]["kind"] == "IVFPQ"
    assert np.array_equal(back["base"]["codes"], base["codes"]) and back["base"]["nprobe"] == 2


def test_ixrf_fp16_read_refuses_values_that_do_not_round_trip():
    from retrieval_scaling_b200 import index as rsb_index
    rng = np.random.default_rng(1)
    xb = rng.standard_normal((5, 16)).astype(np.float32)           # not fp16-representable
    parts = {"kind": "Refine", "d": 16, "ntotal": 5, "metric": 0, "base": _ivfpq_parts(rng), "xb": xb, "k_factor": 2.0}
    with pytest.raises(ValueError, match="float16"):
        rsb_index._from_faiss_parts(parts, refine_dtype="float16")   # refused before any device allocation
    with pytest.raises(NotImplementedError):
        rsb_index._from_faiss_parts({**parts, "k_factor": 1.5})


def test_config_keys():
    import os
    from retrieval_scaling_b200 import config as C
    from retrieval_scaling_b200.indicies.base import Indexer
    conf = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ric", "conf")
    base = ["datastore.domain=x", "datastore.index.index_type=IVFPQ"]
    assert Indexer.refine_options(C.load_config("default", conf, base).datastore.index) == (0, None)   # key absent
    cfg = C.load_config("default", conf, base + ["+datastore.index.refine_k_factor=8", "+datastore.index.refine_dtype=float16"])
    assert Indexer.refine_options(cfg.datastore.index) == (8, "float16")
    cfg = C.load_config("default", conf, base + ["+datastore.index.refine_k_factor=0"])
    assert Indexer.refine_options(cfg.datastore.index) == (0, None)
    for kind in ("Flat", "IVFFlat"):
        cfg = C.load_config("default", conf, ["datastore.domain=x", f"datastore.index.index_type={kind}",
                                              "+datastore.index.refine_k_factor=4"])
        with pytest.raises(ValueError, match="already exact"):
            Indexer(cfg)                                            # refused before anything is built
    cfg = C.load_config("default", conf, base + ["+datastore.index.refine_k_factor=4", "+datastore.index.refine_dtype=bf16"])
    with pytest.raises(ValueError):
        Indexer.refine_options(cfg.datastore.index)


def test_all_device_refine_argument_checks():
    L = _lib.lib()
    z = None
    # k * k_factor beyond the scan's 4096 limit: unsupported, reported, not a fault
    # an all-device store (n_dev = ntotal): store_host, sq_dev and staging_bytes are ignored
    def refine(dtype, d, k_base, k):
        return L.rsb_refine(z, 1, z, 0, z, dtype, z, d, 0, z, k_base, k, z, z, z, 0, 0, z, z)
    assert refine(_lib.RSB_DTYPE_F16, 768, 4097, 10) == _lib.RSB_ERR_UNSUPPORTED
    assert b"4096" in L.rsb_last_error()
    assert refine(7, 768, 100, 10) == _lib.RSB_ERR_INVALID                                        # dtype
    assert refine(_lib.RSB_DTYPE_F32, 768, 5, 10) == _lib.RSB_ERR_INVALID                         # k > k_base
    assert refine(_lib.RSB_DTYPE_F32, 36, 50, 10) == _lib.RSB_ERR_INVALID                         # d % 8
    assert L.rsb_search_refine(z, z, 1, 10, 4, 8, z, 0, z, 0, z, 0, z, z, z, 0, 0, z, z) == _lib.RSB_ERR_INVALID  # null handle


def test_faiss_cross_check():
    faiss = pytest.importorskip("faiss")
    rng = np.random.default_rng(0)
    d, n = 32, 2000
    xb = rng.standard_normal((n, d)).astype(np.float32)
    xq = rng.standard_normal((8, d)).astype(np.float32)
    base = faiss.IndexIVFPQ(faiss.IndexFlatIP(d), d, 8, 8, 8, faiss.METRIC_INNER_PRODUCT)
    base.train(xb)
    ref = faiss.IndexRefineFlat(base)
    ref.add(xb)
    ref.k_factor = 4
    base.nprobe = 8
    parts = F.read_faiss(io.BytesIO(faiss.serialize_index(ref).tobytes()))
    assert parts["kind"] == "Refine" and parts["k_factor"] == 4.0 and np.array_equal(parts["xb"], xb)
    Df, If = ref.search(xq, 10)
    _, Ib = base.search(xq, 40)
    Do, Io = R.refine_candidates(xq, xb, Ib, 10)
    O.assert_topk_equivalent(Df, If, Do, Io, rtol=1e-5, atol=1e-5)
