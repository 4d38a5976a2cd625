"""IVF-SQ8 (faiss IndexIVFScalarQuantizer, QT_8bit), host side: the oracle's known answers with and without residuals,
the IwSq / IwSQ file layout, the C-ABI's refusals (reported, never fatal), and the `storage_dtype=sq8` config key."""
import ctypes
import io
import os
import struct
from fractions import Fraction

import numpy as np
import pytest

from ivfsq8_oracle import ivfsq8_encode, ivfsq8_search, ivfsq8_train
from oracle.sq8_oracle import sq8_decode
from retrieval_scaling_b200 import _lib, faiss_io

F32 = np.float32
CONF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ric", "conf")


def _dec(c):
    """(c + 0.5) / 255 rounded to fp32: the decoded value of code c for vmin = 0, vdiff = 1."""
    return F32(float(Fraction(2 * c + 1, 510)))


def _known_case():
    d = 16
    cent = np.zeros((2, d), F32)
    cent[0, 0], cent[1, 1] = 1.0, 2.0
    sq = np.stack([np.zeros(d, F32), np.ones(d, F32)])                 # vmin = 0, vdiff = 1
    codes = np.zeros((4, d), np.uint8)
    codes[:, 0] = [127, 255, 0, 254]                                   # rows 0, 1 in list 0; rows 2, 3 in list 1
    offsets = np.array([0, 2, 4], np.int64)
    ids = np.array([10, 11, 12, 13], np.int64)
    q = np.zeros((1, d), F32)
    q[0, 0] = 1.0                                                      # <q, c0> = 1, <q, c1> = 0
    return cent, sq, codes, offsets, ids, q


def test_oracle_known_answer_without_residuals():
    cent, sq, codes, offsets, ids, q = _known_case()
    D, I = ivfsq8_search(q, cent, sq, offsets, codes, ids, nprobe=2, k=4, by_residual=False)
    # scores = the decoded element 0: 255 -> 511/510, 254 -> 509/510, 127 -> 1/2, 0 -> 1/510
    assert I.tolist() == [[11, 13, 10, 12]]
    assert D.tolist() == [[_dec(255), _dec(254), F32(0.5), _dec(0)]]


def test_oracle_known_answer_with_residuals():
    cent, sq, codes, offsets, ids, q = _known_case()
    D, I = ivfsq8_search(q, cent, sq, offsets, codes, ids, nprobe=2, k=4, by_residual=True)
    # list 0 adds <q, c0> = 1 after the sum, list 1 adds 0: the order changes
    assert I.tolist() == [[11, 10, 13, 12]]
    assert D.tolist() == [[F32(1) + _dec(255), F32(1.5), _dec(254), _dec(0)]]
    # nprobe = 1 probes list 0 only; search_preassigned with the caller's coarse score
    D1, I1 = ivfsq8_search(q, cent, sq, offsets, codes, ids, nprobe=1, k=3, by_residual=True)
    assert I1.tolist() == [[11, 10, -1]]
    Dp, Ip = ivfsq8_search(q, cent, sq, offsets, codes, ids, 1, 2, True, lists=np.array([[1]]),
                           coarse_dis=np.array([[F32(0.25)]]))
    assert Ip.tolist() == [[13, 12]] and Dp.tolist() == [[F32(0.25) + _dec(254), F32(0.25) + _dec(0)]]


def test_oracle_encode_and_train_use_residuals():
    rng = np.random.default_rng(0)
    cent = rng.standard_normal((3, 16)).astype(F32)
    x = rng.standard_normal((50, 16)).astype(F32)
    a = rng.integers(0, 3, 50)
    sq_r = ivfsq8_train(x, cent, a, True)
    assert np.array_equal(sq_r[0], (x - cent[a]).min(0))
    codes = ivfsq8_encode(x, cent, sq_r, a, True)
    err = np.abs(sq8_decode(codes, sq_r) - (x - cent[a]))
    assert (err <= sq_r[1] / 255 + 1e-6).all()
    assert np.array_equal(ivfsq8_train(x, cent, a, False), ivfsq8_train(x, cent * 0, a, True))


def _parts(by_residual=True, n=9, nlist=4, d=16, seed=1):
    rng = np.random.default_rng(seed)
    sizes = np.array([4, 0, 5, 0])[:nlist]
    offsets = np.zeros(nlist + 1, np.int64)
    np.cumsum(sizes, out=offsets[1:])
    return {"kind": "IVFSQ", "d": d, "nlist": nlist, "nprobe": 3, "by_residual": by_residual,
            "centroids": rng.standard_normal((nlist, d)).astype(F32),
            "sq": np.stack([rng.standard_normal(d), rng.random(d) + 0.5]).astype(F32),
            "offsets": offsets, "codes": rng.integers(0, 256, (n, d)).astype(np.uint8),
            "ids": rng.permutation(100)[:n].astype(np.int64)}


@pytest.mark.parametrize("by_residual", [True, False])
def test_iwsq_round_trip_and_layout(by_residual):
    p = _parts(by_residual)
    f = io.BytesIO()
    faiss_io.write_faiss(f, p)
    raw = f.getvalue()
    assert raw[:4] == b"IwSq"
    # after the ivf header (incl. the IxFI quantizer and an empty direct map): the ScalarQuantizer, code_size, by_residual
    d, nlist = p["d"], p["nlist"]
    o = 4 + 4 + 8 + 8 + 8 + 1 + 4 + 8 + 8                   # header, nlist, nprobe
    o += 4 + 4 + 8 + 8 + 8 + 1 + 4 + 8 + nlist * d * 4       # IxFI quantizer
    o += 1 + 8                                               # direct map
    qtype, rangestat, arg, sd, cs, ntr = struct.unpack_from("<iifQQQ", raw, o)
    assert (qtype, rangestat, arg, sd, cs, ntr) == (0, 0, 0.0, d, d, 2 * d)
    o += struct.calcsize("<iifQQQ")
    assert np.array_equal(np.frombuffer(raw, F32, 2 * d, o).reshape(2, d), p["sq"])
    o += 8 * d
    assert struct.unpack_from("<QB", raw, o) == (d, int(by_residual))
    assert raw[o + 9:o + 13] == b"ilar"
    q = faiss_io.read_faiss(io.BytesIO(raw))
    assert q["kind"] == "IVFSQ" and q["by_residual"] == by_residual
    for key in ("centroids", "sq", "offsets", "codes", "ids"):
        assert np.array_equal(q[key], p[key]), key
    path_like = io.BytesIO()
    faiss_io.write_faiss(path_like, q)
    assert path_like.getvalue() == raw


def test_legacy_iwsq_reads_as_by_residual():
    p = _parts(by_residual=False)
    f = io.BytesIO()
    faiss_io.write_faiss(f, p)
    raw = bytearray(f.getvalue())
    # the older tag carries no by_residual byte: drop it and rename the tag
    pos = raw.index(b"ilar") - 1
    assert raw[pos] == 0
    legacy = b"IwSQ" + bytes(raw[4:pos]) + bytes(raw[pos + 1:])
    q = faiss_io.read_faiss(io.BytesIO(legacy))
    assert q["kind"] == "IVFSQ" and q["by_residual"] is True
    assert np.array_equal(q["codes"], p["codes"]) and np.array_equal(q["sq"], p["sq"])


def test_is_faiss_file_knows_both_tags(tmp_path):
    for tag in (b"IwSq", b"IwSQ"):
        path = os.path.join(str(tmp_path), tag.decode())
        with open(path, "wb") as f:
            f.write(tag + b"\0" * 8)
        assert faiss_io.is_faiss_file(path)


@pytest.mark.parametrize("by_residual", [True, False])
def test_faiss_cross_check(tmp_path, by_residual):
    """Both directions against a real faiss build, where one is importable: a file faiss writes reads here with the
    same codes and range, and a file written here searches in faiss like the oracle."""
    faiss = pytest.importorskip("faiss")
    rng = np.random.default_rng(3)
    d, nlist, n = 32, 4, 300
    x = rng.standard_normal((n, d)).astype(F32)
    quant = faiss.IndexFlatIP(d)
    ix = faiss.IndexIVFScalarQuantizer(quant, d, nlist, faiss.ScalarQuantizer.QT_8bit, faiss.METRIC_INNER_PRODUCT,
                                       by_residual)
    ix.train(x)
    ix.add(x)
    path = os.path.join(str(tmp_path), "ivfsq8.faiss")
    faiss.write_index(ix, path)
    p = faiss_io.read_faiss(path)
    assert p["kind"] == "IVFSQ" and p["by_residual"] == by_residual
    assert np.array_equal(p["sq"].reshape(-1), faiss.vector_to_array(ix.sq.trained))
    ix.nprobe = 2
    D, I = ix.search(x[:5], 10)
    Do, Io = ivfsq8_search(x[:5], p["centroids"], p["sq"], p["offsets"], p["codes"], p["ids"], 2, 10, by_residual)
    from oracle import ann_oracle as A
    A.assert_topk_equivalent(D, I, Do, Io, rtol=1e-5, atol=1e-5)
    out = os.path.join(str(tmp_path), "ours.faiss")
    faiss_io.write_faiss(out, p)
    back = faiss.read_index(out)
    back.nprobe = 2
    D2, I2 = back.search(x[:5], 10)
    A.assert_topk_equivalent(D2, I2, Do, Io, rtol=1e-5, atol=1e-5)


def test_abi_create_and_option_refusals():
    """Refusals that come before any device allocation (the handle-level ones are in tests/test_gpu_ivfsq8.py)."""
    L = _lib.lib()
    h = ctypes.c_void_p(0)
    SQ8 = _lib.RSB_DTYPE_SQ8
    assert L.rsb_ivfflat_create(72, 16, SQ8, ctypes.byref(h)) == _lib.RSB_ERR_INVALID      # d % 16: 16-byte rows
    assert b"16" in L.rsb_last_error()
    assert L.rsb_flat_create(768, SQ8, ctypes.byref(h)) == _lib.RSB_ERR_INVALID            # Flat SQ8: not implemented
    assert not h.value
    p = ctypes.c_void_p(16)            # never dereferenced: the arguments are refused first
    assert L.rsb_set_option(None, _lib.OPT_BY_RESIDUAL, 1) == _lib.RSB_ERR_INVALID
    assert L.rsb_set_sq_range(None, p, None) == _lib.RSB_ERR_INVALID
    assert L.rsb_get_sq_range(None, p, None) == _lib.RSB_ERR_INVALID
    assert L.rsb_add_codes(None, p, 1, None, p, None) == _lib.RSB_ERR_INVALID


def test_abi_table_has_the_new_entry_points():
    names = {n for n, _, _ in _lib.SIGNATURES}
    assert {"rsb_set_sq_range", "rsb_get_sq_range"} <= names
    header = open(os.path.join(os.path.dirname(CONF), "..", "include", "rsb.h")).read()
    assert "RSB_INFO_BY_RESIDUAL = 10" in header and "RSB_OPT_BY_RESIDUAL = 1" in header


def _index_cfg(kind, extra=()):
    from retrieval_scaling_b200 import config as C
    return C.load_config("default", CONF, ["datastore.domain=x", f"datastore.index.index_type={kind}", *extra]).datastore.index


def test_storage_dtype_sq8_key():
    from retrieval_scaling_b200.indicies.base import Indexer
    assert Indexer.storage_dtype(_index_cfg("IVFFlat", ["+datastore.index.storage_dtype=sq8"])) == "sq8"
    with pytest.raises(ValueError, match="IVFFlat"):
        Indexer.storage_dtype(_index_cfg("Flat", ["+datastore.index.storage_dtype=sq8"]))
    with pytest.raises(ValueError, match="PQ codes"):
        Indexer.storage_dtype(_index_cfg("IVFPQ", ["+datastore.index.storage_dtype=sq8"]))
    with pytest.raises(ValueError, match="float16 or float32") as e:
        Indexer.storage_dtype(_index_cfg("IVFFlat", ["+datastore.index.storage_dtype=sq4"]))
    assert "sq8" in str(e.value)


def test_read_refuses_dtype_conversions_before_any_device_work():
    from retrieval_scaling_b200 import index as rsb_index
    p = _parts()
    for bad in ("float16", "float32"):
        with pytest.raises(ValueError, match="sq8"):
            rsb_index._from_faiss_parts(dict(p, metric=0), storage_dtype=bad)
    flat = {"kind": "IVFFlat", "metric": 0, "d": 16, "nlist": 1}
    with pytest.raises(ValueError, match="IVF-SQ8"):
        rsb_index._from_faiss_parts(flat, storage_dtype="sq8")
