"""CPU oracle (test infrastructure, not product code) for IVF-SQ8: faiss 1.8.0 IndexIVFScalarQuantizer with QT_8bit,
RS_minmax and METRIC_INNER_PRODUCT, restated from the published source (`faiss/IndexScalarQuantizer.cpp`:
`IndexIVFScalarQuantizer::encode_vectors`, `IVFSQScannerIP::distance_to_code` = accu0 + query_to_code).
[FAISS-ext]: faiss is not importable here, so these rules are pinned by hand-computed tests and, wherever faiss is
importable, by tests/test_ivfsq8_cpu.py's cross-check.

  add     list = argmax_c <x, c> (IndexFlatIP quantizer); code = encode(x - c_list) by residual, else encode(x)
  train   the range is sq8_train of the rows (residuals against their assigned list when by_residual)
  search  the nprobe best lists by <q, c> (fp32); score = fl32(<q, c_list> + s) by residual, else s,
          s = <q, decode(code)> in fp32

The scalar quantizer's train / encode / decode rules are oracle/sq8_oracle.py's.  Only tests/ and scripts may import
this module.
"""
from __future__ import annotations

import numpy as np

from oracle import ann_oracle as A
from oracle.sq8_oracle import sq8_decode, sq8_encode, sq8_train

F32 = np.float32


def ivfsq8_rows(x: np.ndarray, centroids: np.ndarray, assign: np.ndarray, by_residual: bool) -> np.ndarray:
    """The rows the scalar quantizer sees: x (fp32; fp16 widens exactly), minus its list's centroid by residual."""
    x = np.asarray(x).astype(F32)
    return (x - np.asarray(centroids, F32)[assign]).astype(F32) if by_residual else x


def ivfsq8_train(x, centroids, assign, by_residual: bool) -> np.ndarray:
    return sq8_train(ivfsq8_rows(x, centroids, assign, by_residual))


def ivfsq8_encode(x, centroids, sq, assign, by_residual: bool) -> np.ndarray:
    return sq8_encode(ivfsq8_rows(x, centroids, assign, by_residual), sq)


def ivfsq8_search(xq, centroids, sq, offsets, codes, ids, nprobe: int, k: int, by_residual: bool,
                  lists=None, coarse_dis=None):
    """Top-k (scores desc, ids asc on ties) over the probed lists.  lists / coarse_dis [nq, nprobe] (optional) replace
    the coarse quantizer, as faiss' search_preassigned does.  Each probed list is decoded once and scored for every
    query that probes it, so an index far larger than its decoded form in host memory can be checked."""
    xq = np.ascontiguousarray(xq, dtype=F32)
    nq = xq.shape[0]
    if lists is None:
        coarse_dis, lists = A.coarse_probe(xq, centroids, min(nprobe, np.asarray(centroids).shape[0]))
    lists = np.asarray(lists)
    ss = [[] for _ in range(nq)]
    ii = [[] for _ in range(nq)]
    for l in np.unique(lists[lists >= 0]):
        a, b = offsets[l], offsets[l + 1]
        if b <= a:
            continue
        V = sq8_decode(codes[a:b], sq)
        qi, pj = np.nonzero(lists == l)
        S = (V @ xq[qi].T).astype(F32)                           # [list length, probing queries]
        for c, (i, j) in enumerate(zip(qi, pj)):
            ss[i].append((F32(coarse_dis[i][j]) + S[:, c]).astype(F32) if by_residual else S[:, c])
            ii[i].append(ids[a:b])
    D = np.full((nq, k), A.NEG, dtype=F32)
    I = np.full((nq, k), -1, dtype=np.int64)
    for i in range(nq):
        if ss[i]:
            D[i], I[i] = A._topk_desc(np.concatenate(ss[i]).astype(F32), np.concatenate(ii[i]), k)
    return D, I
