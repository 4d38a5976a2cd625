"""CPU checks of the decode diagnostics of include/rsb.h (rsb_llm_decode_attention, rsb_llm_greedy): both are bound
and exported, and the refusals that need no device memory come back as errors, not as a launch or an abort.  The
pointers passed are never dereferenced: each call carries one bad argument, which is refused first."""
import ctypes

import pytest

from retrieval_scaling_b200 import _lib

P = ctypes.c_void_p(16)                          # 16-byte aligned, never read


def test_decode_symbols_are_bound_and_exported():
    L = _lib.lib()
    bound = {name for name, _, _ in _lib.SIGNATURES}
    for name in ("rsb_llm_decode_attention", "rsb_llm_greedy"):
        assert name in bound and hasattr(L, name)


@pytest.mark.parametrize("k", [0, 1, 2, 3, 5, 6, 9])
def test_decode_attention_refuses_null_pointers(k):
    L = _lib.lib()
    args = [P, P, P, P, 1, P, P, 1, 64, P, None]
    args[k] = None
    assert L.rsb_llm_decode_attention(*args) == _lib.RSB_ERR_INVALID
    assert b"null" in L.rsb_llm_last_error()


@pytest.mark.parametrize("k, v, msg", [
    (0, _lib.RSB_DTYPE_F32, b"dtype"), (0, _lib.RSB_DTYPE_SQ8, b"dtype"), (0, 7, b"dtype"),
    (1, None, b"null"), (5, None, b"null"), (6, None, b"null"),
    (2, 0, b"vocab"), (2, -5, b"vocab"), (3, 1000, b"ld"), (3, 1004, b"ld"), (4, -1, b"n_rows"),
    (1, ctypes.c_void_p(24), b"aligned")])
def test_greedy_refusals_are_reported_not_fatal(k, v, msg):
    L = _lib.lib()
    args = [_lib.RSB_DTYPE_F16, P, 1001, 1024, 4, P, P, None]
    args[k] = v
    assert L.rsb_llm_greedy(*args) == _lib.RSB_ERR_INVALID
    assert msg in L.rsb_llm_last_error()


def test_greedy_with_no_rows_launches_nothing():
    L = _lib.lib()
    assert L.rsb_llm_greedy(_lib.RSB_DTYPE_BF16, P, 1001, 1024, 0, P, P, None) == _lib.RSB_OK
