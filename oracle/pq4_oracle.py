"""CPU ORACLE (test infrastructure, NOT product code) for IVF-PQ with 4-bit sub-quantizers:
`faiss.IndexIVFPQ(IndexFlatIP, d, nlist, M, 4, METRIC_INNER_PRODUCT)` (the reference's `n_bits` setting,
`src/indicies/ivf_pq.py:146-152`), restated on top of `ann_oracle`'s 8-bit rules.

[FAISS-ext] faiss is not importable here, so these rules are restated from the published faiss 1.8.0 source and pinned by
hand-computed tests only (tests/test_pq4_cpu.py):
  * code packing (`PQEncoderGeneric`, nbits = 4): codes are written LSB first, two per byte,
        byte b = c[2b] | c[2b+1] << 4;   code_size = M * 4 / 8 = M / 2 bytes per vector
  * encoding: ksub = 16 entries per sub-quantizer, nearest by L2 (the rule of `ann_oracle.pq_encode`)
  * search (`IVFPQScanner` with `PQDecoderGeneric`): the score of a code is accumulated term by term in fp32,
        dis = dis0;  for m in 0..M-1: dis += T[m][c_m]
  * training (`ProductQuantizer::train`): M independent L2 k-means of ksub = 16 on the residuals; one Lloyd step is
    assignment by `pq_encode`, then each entry becomes the mean of its members (entries without members are kept here;
    the product re-seeds them, retrieval_scaling_b200/train.py)

`host_ivfpq` gives `parity.HostIVFPQ` (fp64 re-score from the exported codes) for either code width.

Only tests/, __graft_entry__.smoke() and scripts may import this module.
"""
from __future__ import annotations

import numpy as np

from . import ann_oracle as ao
from .parity import HostIVFPQ


def pack4(codes: np.ndarray) -> np.ndarray:
    """[n, M] codes < 16 -> [n, M/2] bytes, byte b = c[2b] | c[2b+1] << 4 (faiss PQEncoderGeneric, LSB first)."""
    c = np.asarray(codes, dtype=np.uint8)
    assert c.ndim == 2 and c.shape[1] % 2 == 0 and (c < 16).all()
    return (c[:, 0::2] | (c[:, 1::2] << 4)).astype(np.uint8)


def unpack4(packed: np.ndarray) -> np.ndarray:
    """[n, M/2] bytes -> [n, M] codes (inverse of pack4)."""
    p = np.asarray(packed, dtype=np.uint8)
    out = np.empty((p.shape[0], 2 * p.shape[1]), dtype=np.uint8)
    out[:, 0::2] = p & 15
    out[:, 1::2] = p >> 4
    return out


def pq4_encode(r: np.ndarray, codebook: np.ndarray) -> np.ndarray:
    """Packed codes [n, M/2] of residuals r [n, d]; codebook [M, 16, dsub]."""
    assert codebook.shape[1] == 16
    return pack4(ao.pq_encode(r, codebook))


def ivfpq4_encode(x, centroids, codebook, assign=None):
    """IndexIVFPQ.add with nbits = 4: l = argmax_c <x, c>; r = x - c_l; packed code = PQ4(r)."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    if assign is None:
        assign = ao.ivf_assign(x, centroids)
    return assign, pq4_encode(x - centroids[assign], codebook)


def pq4_decode(packed: np.ndarray, codebook: np.ndarray) -> np.ndarray:
    return ao.pq_decode(unpack4(packed), codebook)


def ivfpq4_search(xq, centroids, codebook, offsets, packed_sorted, ids_sorted, nprobe: int, k: int):
    """IndexIVFPQ.search with nbits = 4: score = dis0 + T[0][c_0] + T[1][c_1] + ..., added one term at a time in fp32."""
    xq = np.ascontiguousarray(xq, dtype=np.float32)
    nq, nlist, M = xq.shape[0], centroids.shape[0], codebook.shape[0]
    D = np.full((nq, k), ao.NEG, dtype=np.float32)
    I = np.full((nq, k), -1, dtype=np.int64)
    _, probes = ao.flat_search(xq, centroids, min(nprobe, nlist))
    T = ao.pq_lut(xq, codebook)                                   # [nq, M, 16] fp32
    codes = unpack4(packed_sorted) if len(packed_sorted) else np.zeros((0, M), np.uint8)
    for i in range(nq):
        ss, ii = [], []
        for l in probes[i]:
            if l < 0:
                continue
            a, b = offsets[l], offsets[l + 1]
            if b > a:
                s = np.full(b - a, np.float32(xq[i] @ np.asarray(centroids[l], dtype=np.float32)), dtype=np.float32)
                c = codes[a:b]
                for m in range(M):
                    s = (s + T[i, m][c[:, m]]).astype(np.float32)
                ss.append(s)
                ii.append(ids_sorted[a:b])
        if ss:
            D[i], I[i] = ao._topk_desc(np.concatenate(ss), np.concatenate(ii), k)
    return D, I


def pq_lloyd_step(r: np.ndarray, codebook: np.ndarray) -> np.ndarray:
    """One L2 k-means step of every sub-quantizer (any ksub): assign, then mean of the members (empty entries kept)."""
    M, ksub, dsub = codebook.shape
    n = r.shape[0]
    codes = ao.pq_encode(r, codebook)
    rm = np.asarray(r, dtype=np.float64).reshape(n, M, dsub)
    out = np.array(codebook, dtype=np.float32, copy=True)
    for m in range(M):
        sums = np.zeros((ksub, dsub))
        np.add.at(sums, codes[:, m], rm[:, m])
        cnt = np.bincount(codes[:, m], minlength=ksub)
        nz = cnt > 0
        out[m, nz] = (sums[nz] / cnt[nz, None]).astype(np.float32)
    return out


def host_ivfpq(centroids, codebook, offsets, codes, ids) -> HostIVFPQ:
    """parity.HostIVFPQ over exported codes of either width: [n, M] (nbits 8) or packed [n, M/2] (codebook [M, 16, .])."""
    codebook = np.asarray(codebook, dtype=np.float32)
    codes = np.asarray(codes)
    if codebook.shape[1] == 16:
        codes = unpack4(codes) if len(codes) else np.zeros((0, codebook.shape[0]), np.uint8)
    return HostIVFPQ(centroids, codebook, offsets, codes, ids)
