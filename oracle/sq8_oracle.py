"""CPU ORACLE (test infrastructure, NOT product code) for the SQ8 re-rank store: faiss 1.8.0 `ScalarQuantizer` with
qtype QT_8bit and rangestat RS_minmax, non-uniform (one range per dimension), restated from the published source
(`faiss/impl/ScalarQuantizer.cpp`: `train_Uniform` / `train_NonUniform`, `QuantizerTemplate<Codec8bit, false, 1>`).
[FAISS-ext]: faiss is not importable here, so these rules are pinned by hand-computed tests only.

  train   vmin[j] = min over the training rows of x[:, j]; vdiff[j] = max - vmin[j]      -> sq [2, d] = (vmin, vdiff)
  encode  xi = vdiff != 0 ? (x - vmin) / vdiff : 0, clamped to [0, 1]; code = (int)(255.f * xi)
  decode  x = vmin + ((code + 0.5f) / 255.f) * vdiff

Every operation is a separately rounded fp32 operation (numpy float32 arithmetic rounds each one; nothing is fused).
fp16 input is encoded from its exact fp32 value.  Scores of a decoded store follow `refine_oracle.refine_candidates`.

Only tests/, __graft_entry__.smoke() and bench.py may import this module.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32


def sq8_train(x: np.ndarray) -> np.ndarray:
    """x [n, d] (n >= 1) -> sq [2, d] float32: vmin, then vdiff = vmax - vmin."""
    x = np.asarray(x).astype(F32)
    vmin = x.min(axis=0)
    vdiff = x.max(axis=0) - vmin
    return np.stack([vmin, vdiff]).astype(F32)


def sq8_encode(x: np.ndarray, sq: np.ndarray) -> np.ndarray:
    """x [n, d] -> codes [n, d] uint8 for the trained sq [2, d]."""
    x = np.asarray(x).astype(F32)
    vmin, vdiff = np.asarray(sq, F32)
    safe = np.where(vdiff != 0, vdiff, F32(1))
    xi = np.where(vdiff != 0, (x - vmin) / safe, F32(0)).astype(F32)
    xi = np.clip(xi, F32(0), F32(1))
    return (F32(255) * xi).astype(np.int32).astype(np.uint8)


def sq8_decode(codes: np.ndarray, sq: np.ndarray) -> np.ndarray:
    """codes [n, d] uint8 -> the decoded rows [n, d] float32."""
    vmin, vdiff = np.asarray(sq, F32)
    t = (np.asarray(codes).astype(F32) + F32(0.5)) / F32(255)
    return (vmin + t * vdiff).astype(F32)
