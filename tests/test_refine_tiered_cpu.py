"""Tiered re-rank store (rows past `refine_device_rows` in pinned host memory) without a GPU: the config key, the
C-ABI symbols, and the argument checks that return before any CUDA call."""
import ctypes
import os

import pytest

from retrieval_scaling_b200 import _lib

REFINE_SYMBOLS = ("rsb_host_alloc", "rsb_host_free", "rsb_refine_workspace_bytes", "rsb_refine",
               "rsb_search_refine_workspace_bytes", "rsb_search_refine", "rsb_refine_tiered_profile")
F16, F32 = _lib.RSB_DTYPE_F16, _lib.RSB_DTYPE_F32
INVALID = _lib.RSB_ERR_INVALID
FAKE_HOST = 1 << 20            # a non-null, 16-byte aligned address: never dereferenced by the checks tested here


def _cfg(*extra):
    from retrieval_scaling_b200 import config as C
    conf = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "ric", "conf")
    return C.load_config("default", conf, ["datastore.domain=x", "datastore.index.index_type=IVFPQ", *extra]).datastore.index


def test_refine_device_rows_key():
    from retrieval_scaling_b200.indicies.base import Indexer
    assert Indexer.refine_device_rows(_cfg("+datastore.index.refine_k_factor=8")) is None          # absent: all on device
    cfg = _cfg("+datastore.index.refine_k_factor=8", "+datastore.index.refine_device_rows=0")
    assert Indexer.refine_device_rows(cfg) == 0 and Indexer.refine_options(cfg) == (8, None)
    cfg = _cfg("+datastore.index.refine_k_factor=8", "+datastore.index.refine_device_rows=40000000")
    assert Indexer.refine_device_rows(cfg) == 40_000_000
    for bad in ("-1", "1.5", "abc", "true"):
        cfg = _cfg("+datastore.index.refine_k_factor=8", f"+datastore.index.refine_device_rows={bad}")
        with pytest.raises(ValueError, match="refine_device_rows"):
            Indexer.refine_options(cfg)                            # refused where the other refine keys are parsed
    for kf in ([], ["+datastore.index.refine_k_factor=0"]):
        cfg = _cfg(*kf, "+datastore.index.refine_device_rows=10")
        with pytest.raises(ValueError, match="refine_k_factor"):
            Indexer.refine_options(cfg)


def test_index_refine_device_rows_argument():
    from retrieval_scaling_b200.index import _check_device_rows
    assert _check_device_rows(None) is None and _check_device_rows(0) == 0 and _check_device_rows(7) == 7
    for bad in (-1, 1.5, "3", True):
        with pytest.raises(ValueError, match="device_rows"):
            _check_device_rows(bad)


def test_refine_symbols_are_exported_and_bound():
    L = _lib.lib()
    bound = {name for name, _, _ in _lib.SIGNATURES}
    for name in REFINE_SYMBOLS:
        assert name in bound and hasattr(L, name)


def _tiered(q=None, nq=1, store_dev=None, n_dev=0, store_host=FAKE_HOST, dtype=F16, d=768, ntotal=1000, cand=None,
            k_base=800, k=100, D=None, I=None, staging=800 * 768 * 2):
    L = _lib.lib()
    return L.rsb_refine(q, nq, store_dev, n_dev, store_host, dtype, None, d, ntotal, cand, k_base, k, D, I, None, 0,
                        staging, None, None)


def test_tiered_store_argument_checks_before_any_cuda_call():
    L = _lib.lib()
    assert _tiered(dtype=7) == INVALID and b"store_dtype" in L.rsb_last_error()
    for n_dev in (-1, 1001):
        assert _tiered(n_dev=n_dev) == INVALID and b"n_dev" in L.rsb_last_error()
    assert _tiered(staging=800 * 768 * 2 - 1) == INVALID and b"staging_bytes" in L.rsb_last_error()
    assert _tiered(dtype=F32, staging=800 * 768 * 2) == INVALID                    # fp32 rows: twice the bytes
    assert _tiered(store_host=None) == INVALID and b"host tier" in L.rsb_last_error()
    assert _tiered(store_host=FAKE_HOST + 8) == INVALID                            # not 16-byte aligned
    assert _tiered(n_dev=500, store_dev=None) == INVALID and b"device pointer" in L.rsb_last_error()
    assert _tiered(q=None) == INVALID and b"null" in L.rsb_last_error()            # queries / candidates / outputs
    assert _tiered(k_base=4097) == _lib.RSB_ERR_UNSUPPORTED
    assert _tiered(nq=0) == _lib.RSB_OK
    assert L.rsb_search_refine(None, None, 1, 10, 4, 8, None, 0, FAKE_HOST, F16, None, 0, None, None, None, 0,
                               1 << 20, None, None) == INVALID                   # null handle
    assert L.rsb_refine_workspace_bytes(1, 800, 100, 768, 7, 0, 1000, 1 << 30) == 0
    assert L.rsb_refine_workspace_bytes(1, 10, 100, 768, F16, 0, 1000, 1 << 30) == 0     # k > k_base
    assert L.rsb_search_refine_workspace_bytes(None, 1, 10, 4, 8, F16, 0, 1000, 1 << 30) == 0


def test_host_alloc_arguments():
    L = _lib.lib()
    assert L.rsb_host_alloc(16, None) == INVALID
    p = ctypes.c_void_p(123)
    assert L.rsb_host_alloc(0, ctypes.byref(p)) == _lib.RSB_OK and not p.value      # nothing to allocate
    assert L.rsb_host_free(None) == _lib.RSB_OK
