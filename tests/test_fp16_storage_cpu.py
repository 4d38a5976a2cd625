"""fp16 vector storage for Flat / IVF-Flat, host side: the `datastore.index.storage_dtype` key, the C-ABI's new error
paths (reported, never fatal), and the host-side fp16 representability checks that run before any device work."""
import ctypes
import os

import numpy as np
import pytest

from retrieval_scaling_b200 import _lib

CONF = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ric", "conf")


def _index_cfg(kind, extra=()):
    from retrieval_scaling_b200 import config as C
    return C.load_config("default", CONF, ["datastore.domain=x", f"datastore.index.index_type={kind}", *extra]).datastore.index


def test_storage_dtype_key():
    from retrieval_scaling_b200.indicies.base import Indexer
    for kind in ("Flat", "IVFFlat"):
        assert Indexer.storage_dtype(_index_cfg(kind)) is None                                   # key absent
        for v in ("float16", "float32"):
            assert Indexer.storage_dtype(_index_cfg(kind, [f"+datastore.index.storage_dtype={v}"])) == v
        for bad in ("bf16", "fp16", "int8"):
            with pytest.raises(ValueError, match="float16 or float32"):
                Indexer.storage_dtype(_index_cfg(kind, [f"+datastore.index.storage_dtype={bad}"]))
    assert Indexer.storage_dtype(_index_cfg("IVFPQ")) is None
    for v in ("float16", "float32"):
        with pytest.raises(ValueError, match="PQ codes"):
            Indexer.storage_dtype(_index_cfg("IVFPQ", [f"+datastore.index.storage_dtype={v}"]))


def test_storage_dtype_is_refused_for_ivfpq_before_anything_is_built():
    from retrieval_scaling_b200 import config as C
    from retrieval_scaling_b200.indicies.base import Indexer
    cfg = C.load_config("default", CONF, ["datastore.domain=x", "datastore.index.index_type=IVFPQ",
                                          "+datastore.index.storage_dtype=float16"])
    with pytest.raises(ValueError, match="storage_dtype"):
        Indexer(cfg)


def test_dtype_arguments_of_create_and_add_are_checked():
    L = _lib.lib()
    h = ctypes.c_void_p(0)
    F16 = _lib.RSB_DTYPE_F16
    # fp16 Flat scores on wgmma with 64 fp16 per K step: d = 72 is a valid fp16 row size but has no scorer
    assert L.rsb_flat_create(72, F16, ctypes.byref(h)) == _lib.RSB_ERR_UNSUPPORTED
    assert b"64" in L.rsb_last_error()
    with pytest.raises(NotImplementedError):
        _lib.check(L.rsb_flat_create(72, F16, ctypes.byref(h)))
    assert L.rsb_flat_create(68, F16, ctypes.byref(h)) == _lib.RSB_ERR_INVALID            # d % 8: 16-byte rows
    assert L.rsb_ivfflat_create(68, 16, F16, ctypes.byref(h)) == _lib.RSB_ERR_INVALID
    assert L.rsb_ivfflat_create(768, 16, 7, ctypes.byref(h)) == _lib.RSB_ERR_INVALID      # unknown dtype
    assert L.rsb_flat_create(768, 7, ctypes.byref(h)) == _lib.RSB_ERR_INVALID
    assert L.rsb_add(None, None, F16, 1, None, None, 0, None) == _lib.RSB_ERR_INVALID      # null handle
    assert L.rsb_add_preassigned(None, None, F16, 1, None, None, None) == _lib.RSB_ERR_INVALID
    assert not h.value


def test_fp16_storage_refuses_values_that_do_not_round_trip():
    from retrieval_scaling_b200 import index as rsb_index
    rng = np.random.default_rng(0)
    x = rng.standard_normal((6, 64)).astype(np.float32)
    with pytest.raises(ValueError, match="float16"):
        rsb_index._as_storage(x, "float16", "shard")
    xh = x.astype(np.float16)
    assert rsb_index._as_storage(xh.astype(np.float32), "float16", "shard").dtype == np.float16   # exact: accepted
    assert rsb_index._as_storage(x, "float32", "shard") is x
    # faiss parts: refused before any device allocation
    with pytest.raises(ValueError, match="float16"):
        rsb_index._from_faiss_parts({"kind": "Flat", "d": 64, "ntotal": 6, "xb": x, "metric": 0}, storage_dtype="float16")
    with pytest.raises(ValueError, match="float16 or float32"):
        rsb_index._from_faiss_parts({"kind": "Flat", "d": 64, "ntotal": 6, "xb": x, "metric": 0}, storage_dtype="bf16")
    with pytest.raises(ValueError, match="Flat and IVFFlat"):
        rsb_index._from_faiss_parts({"kind": "IVFPQ", "metric": 0}, storage_dtype="float16")


def test_fp32_shard_that_does_not_round_trip_is_refused_with_its_name(tmp_path):
    import pickle
    from retrieval_scaling_b200.indicies._common import BaseIndexer
    path = os.path.join(str(tmp_path), "passages_03.pkl")
    with open(path, "wb") as f:
        pickle.dump((list(range(4)), np.random.default_rng(1).standard_normal((4, 64)).astype(np.float32)), f)
    ix = BaseIndexer.__new__(BaseIndexer)
    ix.storage_dtype = "float16"
    with pytest.raises(ValueError, match="passages_03"):
        ix._load_shard_for_add(path)
    ix.storage_dtype = None
    assert ix._load_shard_for_add(path).dtype == np.float32
