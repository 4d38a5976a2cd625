"""SQ8 re-rank store (IndexRefine(store_dtype="sq8"), faiss Refine(SQ8)) without a GPU: the oracle's train / encode /
decode on hand-computed cases, the IxRF + IxSQ file layout and its round trip, the config key, the C-ABI's argument
checks (all return before any CUDA call), and a faiss cross-check where faiss is importable."""
import io
import struct

import numpy as np
import pytest

from oracle import ann_oracle as O
from oracle import refine_oracle as R
from oracle import sq8_oracle as S
from retrieval_scaling_b200 import _lib
from retrieval_scaling_b200 import faiss_io as F

f32 = np.float32


def test_train_is_per_dimension_min_and_range():
    x = np.array([[1.0, 5.0, -2.0], [3.0, 5.0, 0.5], [2.0, 5.0, -4.0]], f32)
    sq = S.sq8_train(x)
    assert sq.dtype == np.float32 and sq.shape == (2, 3)
    assert sq[0].tolist() == [1.0, 5.0, -4.0]            # vmin first
    assert sq[1].tolist() == [2.0, 0.0, 4.5]             # vdiff = max - min; the constant column has vdiff 0
    assert np.array_equal(S.sq8_train(x.astype(np.float16)), sq)    # fp16 input: its exact fp32 values


def test_encode_hand_computed_codes():
    sq = np.array([[0.0, 5.0], [1.0, 0.0]], f32)         # column 0: [0, 1]; column 1: constant 5
    x = np.array([[0.0, 5.0],          # x = vmin -> 0; constant column -> 0 whatever the value
                  [1.0, 7.0],          # x = vmax -> 255
                  [-3.0, -1.0],        # below the range clamps to 0
                  [9.0, 5.0],          # above the range clamps to 255
                  [0.5, 5.0],          # 127.5 truncates to 127
                  [f32(2.0) / f32(255.0), 5.0],                                     # exactly on code 2
                  [np.nextafter(f32(2.0) / f32(255.0), f32(0.0)), 5.0]], f32)       # one ulp below it
    codes = S.sq8_encode(x, sq)
    assert codes.dtype == np.uint8
    assert codes[:, 1].tolist() == [0] * 7
    assert codes[:, 0].tolist() == [0, 255, 0, 255, 127, 2, 1]      # truncation: one ulp below 2/255 is code 1
    assert f32(255.0) * x[6, 0] < f32(2.0)


def test_encode_fp16_input_matches_fp32_values():
    rng = np.random.default_rng(0)
    xh = rng.standard_normal((50, 32)).astype(np.float16)
    sq = S.sq8_train(xh)
    assert np.array_equal(S.sq8_encode(xh, sq), S.sq8_encode(xh.astype(f32), sq))


def test_decode_rule_and_the_quotient():
    sq = np.array([[-1.0], [2.0]], f32)
    codes = np.arange(256, dtype=np.uint8).reshape(-1, 1)
    dec = S.sq8_decode(codes, sq)[:, 0]
    t = (np.arange(256, dtype=f32) + f32(0.5)) / f32(255.0)
    assert np.array_equal(dec, f32(-1.0) + t * f32(2.0))
    assert dec[0] == f32(-1.0) + (f32(0.5) / f32(255.0)) * f32(2.0)
    assert dec[0] > -1.0 and dec[-1] > 1.0               # bin centres: code 255 decodes just past vmax, as in faiss
    # the quotient is the correctly rounded division: a reciprocal multiply differs for most codes
    recip = (np.arange(256, dtype=f32) + f32(0.5)) * (f32(1.0) / f32(255.0))
    assert int((recip != t).sum()) == 191
    # decoding the codes of the decoded values gives the same codes back (each decoded value lies inside its bin)
    assert np.array_equal(S.sq8_encode(dec.reshape(-1, 1), sq)[:, 0], np.arange(256))


def test_scores_of_the_decoded_store():
    rng = np.random.default_rng(1)
    xb = rng.standard_normal((40, 16)).astype(f32)
    sq = S.sq8_train(xb)
    dec = S.sq8_decode(S.sq8_encode(xb, sq), sq)
    assert np.abs(dec - xb).max() <= (sq[1].max() / 255) * 0.5 + 1e-6
    q = rng.standard_normal((3, 16)).astype(f32)
    D, I = R.refine_candidates(q, dec, np.tile(np.arange(40), (3, 1)), 5)
    assert np.allclose(D, np.sort(q @ dec.T, axis=1)[:, ::-1][:, :5], rtol=1e-6)


def _ivfpq_parts(rng, d=16, nlist=3, sizes=(2, 0, 3)):
    offsets = np.zeros(nlist + 1, np.int64)
    np.cumsum(sizes, out=offsets[1:])
    n = int(offsets[-1])
    return {"kind": "IVFPQ", "centroids": rng.standard_normal((nlist, d)).astype(f32), "offsets": offsets,
            "ids": np.arange(n, dtype=np.int64), "nprobe": 2,
            "codebook": rng.standard_normal((4, 256, d // 4)).astype(f32),
            "codes": rng.integers(0, 256, (n, 4), dtype=np.uint8)}


def _sq8_refine_parts(rng, d=16, n=5):
    xb = rng.standard_normal((n, d)).astype(f32)
    sq = S.sq8_train(xb)
    return {"kind": "Refine", "base": _ivfpq_parts(rng, d), "sq": sq, "codes": S.sq8_encode(xb, sq), "k_factor": 4.0}


def test_ixrf_ixsq_layout_and_round_trip():
    rng = np.random.default_rng(0)
    parts = _sq8_refine_parts(rng)
    buf = io.BytesIO()
    F.write_faiss(buf, parts)
    raw = buf.getvalue()
    assert raw[:4] == b"IxRF" and struct.unpack_from("<iq", raw, 4) == (16, 5) and raw[37:41] == b"IwPQ"
    sq_bytes = (b"IxSQ" + struct.pack("<iqqqBi", 16, 5, 1 << 20, 1 << 20, 1, 0)
                + struct.pack("<iifQQ", 0, 0, 0.0, 16, 16)                     # QT_8bit, RS_minmax, arg, d, code_size
                + struct.pack("<Q", 32) + parts["sq"].tobytes()                # trained: vmin [16], vdiff [16]
                + struct.pack("<Q", 80) + parts["codes"].tobytes())            # codes [5, 16]
    assert raw.endswith(sq_bytes + struct.pack("<f", 4.0))
    back = F.read_faiss(io.BytesIO(raw))
    assert back["kind"] == "Refine" and back["k_factor"] == 4.0 and back["ntotal"] == 5 and "xb" not in back
    assert np.array_equal(back["sq"], parts["sq"]) and np.array_equal(back["codes"], parts["codes"])
    assert np.array_equal(back["base"]["codes"], parts["base"]["codes"])
    buf2 = io.BytesIO()
    F.write_faiss(buf2, back)
    assert buf2.getvalue() == raw


def test_ixsq_other_qtypes_and_read_dtypes_are_refused():
    from retrieval_scaling_b200 import index as rsb_index
    rng = np.random.default_rng(2)
    parts = _sq8_refine_parts(rng)
    buf = io.BytesIO()
    F.write_faiss(buf, parts)
    raw = bytearray(buf.getvalue())
    at = raw.index(b"IxSQ") + 4 + 33                     # qtype follows the IxSQ index header
    for qtype in (1, 2, 4, 6):                           # QT_4bit, QT_8bit_uniform, QT_fp16, QT_6bit
        raw[at:at + 4] = struct.pack("<i", qtype)
        with pytest.raises(NotImplementedError, match="QT_8bit"):
            F.read_faiss(io.BytesIO(bytes(raw)))
    back = F.read_faiss(io.BytesIO(buf.getvalue()))
    back.update(d=16, metric=0)
    for dtype in ("float16", "float32"):                 # refused before any device allocation
        with pytest.raises(ValueError, match="sq8"):
            rsb_index._from_faiss_parts(back, refine_dtype=dtype)


def test_config_key():
    import os
    from retrieval_scaling_b200 import config as C
    from retrieval_scaling_b200.indicies.base import Indexer
    conf = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ric", "conf")
    base = ["datastore.domain=x", "datastore.index.index_type=IVFPQ", "+datastore.index.refine_k_factor=8"]
    cfg = C.load_config("default", conf, base + ["+datastore.index.refine_dtype=sq8"])
    assert Indexer.refine_options(cfg.datastore.index) == (8, "sq8")
    for bad in ("SQ8", "int8", "sq4", "bf16"):
        cfg = C.load_config("default", conf, base + [f"+datastore.index.refine_dtype={bad}"])
        with pytest.raises(ValueError, match="sq8"):
            Indexer.refine_options(cfg.datastore.index)


def test_sq8_store_argument_checks():
    L = _lib.lib()
    z = None
    SQ8 = _lib.RSB_DTYPE_SQ8
    assert SQ8 == 2
    # an SQ8 store without its range is refused, naming sq_dev
    # (rsb_search_refine checks its handle first: tests/test_gpu_refine_sq8.py)
    for rc in (L.rsb_refine(z, 1, z, 0, z, SQ8, z, 768, 0, z, 100, 10, z, z, z, 0, 0, z, z),
               L.rsb_refine(z, 1, z, 0, FAKE_HOST, SQ8, z, 768, 1000, z, 100, 10, z, z, z, 0, 1 << 30, z, z)):
        assert rc == _lib.RSB_ERR_INVALID
        assert b"sq_dev" in L.rsb_last_error()
    # d % 16, k' > 4096, null range, staging below one query's worst case, null handle
    sq = ctypes_ptr(16)
    assert L.rsb_refine(z, 1, z, 0, z, SQ8, sq, 40, 0, z, 100, 10, z, z, z, 0, 1 << 30, z, z) == _lib.RSB_ERR_INVALID
    assert b"16" in L.rsb_last_error()
    assert L.rsb_refine(z, 1, z, 0, z, SQ8, sq, 768, 0, z, 4097, 10, z, z, z, 0, 1 << 30, z, z) == _lib.RSB_ERR_UNSUPPORTED
    assert L.rsb_refine(z, 1, z, 0, z, SQ8, z, 768, 0, z, 100, 10, z, z, z, 0, 1 << 30, z, z) == _lib.RSB_ERR_INVALID
    assert b"sq_dev" in L.rsb_last_error()
    assert L.rsb_refine(z, 1, z, 0, z, SQ8, ctypes_ptr(8), 768, 0, z, 100, 10, z, z, z, 0, 1 << 30, z, z) == _lib.RSB_ERR_INVALID
    # staging is checked for a tiered store only (n_dev < ntotal)
    assert L.rsb_refine(z, 1, z, 0, FAKE_HOST, SQ8, sq, 768, 1000, z, 100, 10, z, z, z, 0, 100 * 768 - 1, z, z) == _lib.RSB_ERR_INVALID
    assert b"staging_bytes" in L.rsb_last_error()
    assert L.rsb_search_refine(z, z, 1, 10, 4, 8, z, 0, z, SQ8, sq, 0, z, z, z, 0, 1 << 30, z, z) == _lib.RSB_ERR_INVALID
    assert L.rsb_refine_workspace_bytes(1, 100, 10, 40, SQ8, 0, 0, 1 << 30) == 0          # d % 16
    # train / encode: dtype, n, d, null pointers
    assert L.rsb_sq8_train(z, 7, 10, 16, sq, z) == _lib.RSB_ERR_INVALID
    assert L.rsb_sq8_train(z, _lib.RSB_DTYPE_F32, 0, 16, sq, z) == _lib.RSB_ERR_INVALID
    assert L.rsb_sq8_train(z, _lib.RSB_DTYPE_F32, 10, 16, sq, z) == _lib.RSB_ERR_INVALID
    assert L.rsb_sq8_encode(sq, _lib.RSB_DTYPE_F16, 10, 0, sq, sq, z) == _lib.RSB_ERR_INVALID
    assert L.rsb_sq8_encode(sq, _lib.RSB_DTYPE_F32, 10, 16, z, sq, z) == _lib.RSB_ERR_INVALID
    assert L.rsb_sq8_encode(sq, _lib.RSB_DTYPE_F32, 10, 16, sq, z, z) == _lib.RSB_ERR_INVALID


FAKE_HOST = 1 << 20            # a non-null, 16-byte aligned host tier address: never dereferenced by the checks above


def ctypes_ptr(align):
    """A non-null pointer value with the given alignment (never dereferenced: every call above fails its checks first)."""
    import ctypes
    return ctypes.c_void_p(1 << 20 | align)


def test_faiss_cross_check():
    faiss = pytest.importorskip("faiss")
    rng = np.random.default_rng(0)
    d, n = 32, 2000
    xb = rng.standard_normal((n, d)).astype(f32)
    xq = rng.standard_normal((8, d)).astype(f32)
    base = faiss.IndexIVFPQ(faiss.IndexFlatIP(d), d, 8, 8, 8, faiss.METRIC_INNER_PRODUCT)
    ref = faiss.IndexRefine(base, faiss.IndexScalarQuantizer(d, faiss.ScalarQuantizer.QT_8bit, faiss.METRIC_INNER_PRODUCT))
    ref.train(xb)
    ref.add(xb)
    ref.k_factor = 4
    base.nprobe = 8
    parts = F.read_faiss(io.BytesIO(faiss.serialize_index(ref).tobytes()))
    assert parts["kind"] == "Refine" and parts["k_factor"] == 4.0
    assert np.array_equal(parts["sq"], S.sq8_train(xb))
    assert np.abs(parts["codes"].astype(int) - S.sq8_encode(xb, parts["sq"]).astype(int)).max() <= 1
    Df, If = ref.search(xq, 10)
    _, Ib = base.search(xq, 40)
    Do, Io = R.refine_candidates(xq, S.sq8_decode(parts["codes"], parts["sq"]), Ib, 10)
    O.assert_topk_equivalent(Df, If, Do, Io, rtol=1e-5, atol=1e-5)
