"""Tiered Flat index (rows past `device_rows` in pinned host memory, streamed to the GPU by each search) without a GPU:
the config key, the C-ABI symbols and enum values, and the refusals that happen before any device allocation."""
import ctypes
import os
import re

import numpy as np
import pytest

from retrieval_scaling_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(*extra, index_type="Flat"):
    from retrieval_scaling_b200 import config as C
    conf = os.path.join(ROOT, "ric", "conf")
    return C.load_config("default", conf, ["datastore.domain=x", f"datastore.index.index_type={index_type}",
                                           *extra]).datastore.index


def _header():
    return open(os.path.join(ROOT, "include", "rsb.h")).read()


def test_device_rows_key():
    from retrieval_scaling_b200.indicies.base import Indexer
    assert Indexer.device_rows(_cfg()) is None                                            # absent: all on device
    assert Indexer.device_rows(_cfg("+datastore.index.storage_dtype=float16", "+datastore.index.device_rows=0")) == 0
    cfg = _cfg("+datastore.index.storage_dtype=float16", "+datastore.index.device_rows=36000000")
    assert Indexer.device_rows(cfg) == 36_000_000 and Indexer.storage_dtype(cfg) == "float16"
    for bad in ("-1", "1.5", "abc", "true"):
        cfg = _cfg("+datastore.index.storage_dtype=float16", f"+datastore.index.device_rows={bad}")
        with pytest.raises(ValueError, match="device_rows must be an integer"):
            Indexer.device_rows(cfg)
    # every other combination names the requirement
    for extra, it in ((["+datastore.index.device_rows=10"], "Flat"),                                     # fp32 Flat
                      (["+datastore.index.storage_dtype=float32", "+datastore.index.device_rows=10"], "Flat"),
                      (["+datastore.index.storage_dtype=float16", "+datastore.index.device_rows=10"], "IVFFlat"),
                      (["+datastore.index.device_rows=10"], "IVFPQ")):
        with pytest.raises(ValueError, match="index_type Flat and storage_dtype float16"):
            Indexer.device_rows(_cfg(*extra, index_type=it))


def test_storage_dtype_rules_are_unchanged_by_device_rows():
    from retrieval_scaling_b200.indicies.base import Indexer
    cfg = _cfg("+datastore.index.storage_dtype=sq8", "+datastore.index.device_rows=10")
    with pytest.raises(ValueError, match="storage_dtype sq8 applies to IVFFlat indexes only"):
        Indexer.storage_dtype(cfg)
    cfg = _cfg("+datastore.index.storage_dtype=float16", "+datastore.index.device_rows=10", index_type="IVFPQ")
    with pytest.raises(ValueError, match="applies to Flat and IVFFlat indexes"):
        Indexer.storage_dtype(cfg)


def test_tiered_flat_symbols_and_enum_values():
    L = _lib.lib()
    assert "rsb_export_rows" in {name for name, _, _ in _lib.SIGNATURES} and hasattr(L, "rsb_export_rows")
    h = re.sub(r"/\*.*?\*/", "", _header(), flags=re.S)
    # existing values keep their numbers; the new ones follow them
    for name, value in (("RSB_OPT_COARSE_TENSOR", 0), ("RSB_OPT_BY_RESIDUAL", 1), ("RSB_OPT_DEVICE_ROWS", 2),
                        ("RSB_OPT_STAGING_BYTES", 3), ("RSB_INFO_INDEX_BYTES", 8), ("RSB_INFO_BY_RESIDUAL", 10),
                        ("RSB_INFO_HOST_BYTES", 11), ("RSB_INFO_DEVICE_ROWS", 12)):
        assert re.search(rf"\b{name}\s*=\s*{value}\b", h), name
    assert (_lib.OPT_DEVICE_ROWS, _lib.OPT_STAGING_BYTES) == (2, 3)
    assert (_lib.INFO_HOST_BYTES, _lib.INFO_DEVICE_ROWS) == (11, 12)


def test_null_handle_refusals():
    L = _lib.lib()
    assert L.rsb_set_option(None, _lib.OPT_DEVICE_ROWS, 10) == _lib.RSB_ERR_INVALID
    assert L.rsb_set_option(None, _lib.OPT_STAGING_BYTES, 1 << 20) == _lib.RSB_ERR_INVALID
    assert L.rsb_export_rows(None, 0, 1, ctypes.c_void_p(16), None) == _lib.RSB_ERR_INVALID
    assert b"null handle" in L.rsb_last_error()


def test_index_flat_device_rows_argument_before_any_allocation():
    from retrieval_scaling_b200.index import IndexFlatIP
    with pytest.raises(ValueError, match="float16"):
        IndexFlatIP(768, device_rows=10)                       # fp32 Flat stays in device memory
    with pytest.raises(ValueError, match="float16"):
        IndexFlatIP(768, dtype="float32", device_rows=0)
    for bad in (-1, 1.5, "3", True):
        with pytest.raises(ValueError, match="device_rows"):
            IndexFlatIP(768, dtype="float16", device_rows=bad)


def test_read_index_device_rows_refusals(tmp_path):
    from retrieval_scaling_b200 import faiss_io
    from retrieval_scaling_b200.index import read_index
    flat = str(tmp_path / "flat.faiss")
    faiss_io.write_faiss(flat, {"kind": "Flat", "xb": np.ones((3, 64), np.float32)})
    for dt in (None, "float32"):
        with pytest.raises(ValueError, match="storage_dtype='float16'"):
            read_index(flat, storage_dtype=dt, device_rows=1)
    with pytest.raises(ValueError, match="device_rows"):
        read_index(flat, storage_dtype="float16", device_rows=-2)
    ivf = str(tmp_path / "ivf.faiss")
    faiss_io.write_faiss(ivf, {"kind": "IVFFlat", "centroids": np.ones((2, 64), np.float32),
                               "offsets": np.array([0, 1, 1]), "vectors": np.ones((1, 64), np.float32),
                               "ids": np.zeros(1, np.int64)})
    with pytest.raises(ValueError, match="IxFI"):
        read_index(ivf, storage_dtype="float16", device_rows=1)


def test_streamed_flat_writer_matches_the_whole_array_writer(tmp_path):
    """write_flat_rows (the tiered index's writer) writes the bytes of _write_flat, and flat_rows_memmap reads them."""
    from retrieval_scaling_b200 import faiss_io
    rng = np.random.default_rng(0)
    xb = rng.standard_normal((1000, 64)).astype(np.float16).astype(np.float32)
    a, b = str(tmp_path / "a.faiss"), str(tmp_path / "b.faiss")
    faiss_io.write_faiss(a, {"kind": "Flat", "xb": xb})
    with open(b, "wb") as f:
        faiss_io.write_flat_rows(f, 64, 1000, (xb[i:i + 333] for i in range(0, 1000, 333)))
    assert open(a, "rb").read() == open(b, "rb").read()
    d, n, rows = faiss_io.flat_rows_memmap(b)
    assert (d, n) == (64, 1000) and np.array_equal(np.asarray(rows), xb)
    with open(b, "wb") as f, pytest.raises(ValueError, match="rows"):
        faiss_io.write_flat_rows(f, 64, 1000, [xb[:10]])
