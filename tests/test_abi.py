"""CPU-side checks of the drop-in boundary: librsb.so builds/loads, exports every symbol include/rsb.h
declares, reports errors instead of aborting, and the interleaved PQ layout arithmetic (rsb_layout.h) is a
bank-conflict-free bijection.  No compute call needs a GPU here."""
import ctypes
import os
import re

import numpy as np
import pytest

from retrieval_scaling_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_ctypes_table_exports_and_version_301_agree():
    L = _lib.lib()
    header = open(os.path.join(ROOT, "include", "rsb.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    declared = set(re.findall(r"\b(rsb_[a-z0-9_]+)\s*\(", header))
    assert len(declared) >= 25
    bound = {name for name, _, _ in _lib.SIGNATURES}
    assert declared == bound, f"header vs ctypes table mismatch: {declared ^ bound}"
    for name in declared:
        assert hasattr(L, name), f"librsb.so does not export {name}"
    assert L.rsb_version() == 301


def test_create_refusals_are_reported_not_fatal():
    L = _lib.lib()
    h = ctypes.c_void_p(0)
    assert L.rsb_ivfpq_create(768, 16, 64, 6, ctypes.byref(h)) == _lib.RSB_ERR_UNSUPPORTED  # nbits not 8 / 4
    assert b"nbits" in L.rsb_last_error()
    assert L.rsb_ivfpq_create(770, 16, 64, 8, ctypes.byref(h)) == _lib.RSB_ERR_INVALID      # d % 4, d % M
    assert L.rsb_flat_create(-1, _lib.RSB_DTYPE_F32, ctypes.byref(h)) == _lib.RSB_ERR_INVALID
    with pytest.raises(NotImplementedError):
        _lib.check(_lib.RSB_ERR_UNSUPPORTED)
    with pytest.raises(ValueError):
        _lib.check(_lib.RSB_ERR_INVALID)


def test_search_preassigned_refuses_peers_without_local_thresholds():
    """Shared thresholds start at this GPU's array: peers without tau_local_dev are refused before any launch."""
    L = _lib.lib()
    p = ctypes.c_void_p(16)          # never dereferenced: the arguments are refused first
    assert L.rsb_search_preassigned(None, p, 1, 1, 1, p, p, p, p, p, 256, None, None, 2, None) == _lib.RSB_ERR_INVALID
    assert b"threshold arrays" in L.rsb_last_error()
    assert L.rsb_search_preassigned(None, p, 1, 1, 1, p, p, p, p, p, 256, None, p, 0, None) == _lib.RSB_ERR_INVALID
    assert b"threshold arrays" in L.rsb_last_error()


@pytest.mark.parametrize("M", [16, 32, 64])
def test_pq_block_layout_is_a_bijection(M):
    L = _lib.lib()
    offs = np.array([[L.rsb_pq_layout_offset(M, v, m) for m in range(M)] for v in range(32)])
    assert offs.min() == 0 and offs.max() == 32 * M - 1
    assert len(np.unique(offs)) == 32 * M              # every byte of the block is used exactly once
    assert L.rsb_pq_layout_offset(M, 32, 0) == -1 and L.rsb_pq_layout_offset(50, 0, 0) == -1


@pytest.mark.parametrize("M", [24, 48, 96, 128])
def test_generic_m_layout_is_natural_order(M):
    """Sub-quantizer counts outside {16, 32, 64} (faiss and the reference's `n_subquantizers` accept any divisor of d):
    natural [vector][M] code order and a [m][256] look-up table."""
    L = _lib.lib()
    assert all(L.rsb_pq_layout_offset(M, v, m) == v * M + m for v in (0, 7, 31) for m in (0, 1, M - 1))
    assert all(L.rsb_pq_lut_index(M, j, m) == m * 256 + j for j in (0, 255) for m in (0, M - 1))
    assert L.rsb_pq_layout_offset(130, 0, 0) == -1 and L.rsb_pq_layout_offset(132, 0, 0) == -1


@pytest.mark.parametrize("M", [16, 32, 64])
def test_pq_lookups_are_bank_conflict_free(M):
    """Re-derive, from the exported layout, which sub-quantizer every lane reads at every step and check
    that the 32 lanes of a warp always address 32 distinct shared-memory banks (word index mod 32)."""
    L = _lib.lib()
    K = M // 16
    for t in range(K):              # pass
        for s in range(16):         # step inside the pass
            banks = []
            for lane in range(32):
                g, r = lane // K, lane % K
                v = g * K + t
                byte = t * 512 + lane * 16 + s          # the byte lane `lane` consumes at (pass t, step s)
                m = [mm for mm in range(M) if L.rsb_pq_layout_offset(M, v, mm) == byte]
                assert len(m) == 1
                pos = m[0] + M * (g >> 4)               # replica row for M == 16
                assert pos < 64
                banks.append(pos % 32)
            assert len(set(banks)) == 32, (M, t, s, banks)
