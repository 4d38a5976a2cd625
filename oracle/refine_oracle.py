"""CPU ORACLE (test infrastructure, NOT product code) for exact re-ranking: faiss 1.8.0 `IndexRefine::search`
(`faiss/IndexRefine.cpp`), restated from the published source:

  1. base search at k_base = k * k_factor                     base_index->search(n, x, k_base, ...)
  2. exact fp32 score of every valid label, in rank order      dc(idx) = fvec_inner_product(q, x_idx); `if (idx < 0) break`
  3. keep the best k                                           reorder_2_heaps<CMin<float, idx_t>> for METRIC_INNER_PRODUCT

Labels past the first -1 are padding, so their (-FLT_MAX, -1) entries stay unless a valid one displaces them.  The
heap leaves the order of exactly equal scores unspecified; this oracle breaks ties by ascending id, the rule of
`ann_oracle._topk_desc`.  `dtype=np.float64` gives the fp64 shadow for the tie tolerance of `parity.py`.

Only tests/, __graft_entry__.smoke() and bench.py may import this module.
"""
from __future__ import annotations

import numpy as np

from .ann_oracle import NEG, _topk_desc


def refine_candidates(xq: np.ndarray, store: np.ndarray, I_base: np.ndarray, k: int, dtype=np.float32):
    """Steps 2-3: re-score the candidates I_base [nq, k_base] against store [ntotal, d] (row = id; fp16 or fp32, decoded
    to `dtype`), keep the best k by (score desc, id asc), pad with (-FLT_MAX, -1)."""
    xq = np.ascontiguousarray(xq, dtype=dtype)
    I_base = np.asarray(I_base, dtype=np.int64)
    nq = xq.shape[0]
    D = np.full((nq, k), NEG, dtype=np.float32)
    I = np.full((nq, k), -1, dtype=np.int64)
    for i in range(nq):
        ids = I_base[i]
        stop = np.nonzero(ids < 0)[0]
        ids = ids[: stop[0]] if stop.size else ids
        if ids.size:
            s = np.asarray(store[ids], dtype=dtype) @ xq[i]
            D[i], I[i] = _topk_desc(s.astype(np.float32), ids, k)
    return D, I


def refine_search(xq: np.ndarray, store: np.ndarray, base_search, k: int, k_factor: int, dtype=np.float32):
    """IndexRefine::search.  base_search(xq, k_base) -> (D, I) is the base index's search (e.g. ann_oracle.ivfpq_search
    bound to an index)."""
    k_base = int(k * k_factor)
    _, I_base = base_search(xq, k_base)
    return refine_candidates(xq, store, I_base, k, dtype)
