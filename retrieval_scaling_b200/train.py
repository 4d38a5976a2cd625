"""Index training (build side; SURVEY.md §8f-1): k-means for the coarse quantizer and the PQ codebooks.

Restates what `index.train(x)` does in the reference's call sites (`src/indicies/ivf_flat.py:166`,
`src/indicies/ivf_pq.py:170`) with faiss 1.8.0 defaults: Level-1 clustering niter=10, at most 256 training
points per centroid, seed 1234, *spherical* because the metric is inner product (the IndexIVF constructor sets
`cp.spherical = true` for METRIC_INNER_PRODUCT: centroids L2-normalised every iteration, assignment by max inner
product through the IndexFlatIP quantizer); PQ sub-quantizers: L2 k-means, ksub=256 (or 16 for 4-bit codes), niter=25,
on residuals of at most 256*ksub points.  Parity is defined *given* the trained centroids / codebooks (SURVEY §8a row a10).

The Lloyd iterations are driven from here; the arithmetic of every step runs in librsb (`LibrsbOps`):
  assignment (coarse)  : the coarse quantizer itself -- fused fp16 hi/lo wgmma scorer + exact fp32 re-score (rsb_coarse on a
                         scratch handle holding the current centroids) -> fp32-exact argmax
  assignment (PQ)      : rsb_pq_assign (the residual-encoding kernel without the residual step)
  update               : rsb_kmeans_accumulate / rsb_pq_accumulate (member sums and counts)
torch only divides sums by counts, normalises and re-seeds empty clusters (O(k d) element-wise work) and draws the
random subsets.  There is no CPU path: `LibrsbOps` raises without CUDA; the CPU unit tests of the host logic pass
their own numpy stand-in for the three operations (tests/test_train_cpu.py).
"""
from __future__ import annotations

import ctypes

import torch


def _subsample(x: torch.Tensor, max_n: int, gen: torch.Generator) -> torch.Tensor:
    if x.shape[0] <= max_n:
        return x
    perm = torch.randperm(x.shape[0], generator=gen, device=x.device)[:max_n]
    return x[perm]


class LibrsbOps:
    """The three heavy steps of Lloyd's algorithm on librsb's CUDA kernels."""

    def __init__(self):
        if not torch.cuda.is_available():
            raise RuntimeError("index training runs on librsb's CUDA kernels: a CUDA device (H100, sm_90a) is required")
        self._scratch = {}

    @staticmethod
    def _st():
        return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def assign_ip(self, x: torch.Tensor, c: torch.Tensor) -> torch.Tensor:
        """argmax_c <x, c> per row, int64 [n] (lowest id wins exact ties, like the IndexFlatIP quantizer)."""
        from . import index as _index
        key = (int(c.shape[0]), int(c.shape[1]), x.device)
        ix = self._scratch.get(key)
        if ix is None:
            ix = _index.IndexIVFFlat(c.shape[1], c.shape[0], device=x.device)
            self._scratch = {key: ix}
        ix.set_centroids(c)
        return ix.assign(x).long()

    def accumulate(self, x: torch.Tensor, a: torch.Tensor, k: int):
        """(sums [k, d] float32, counts [k] float32) of the members of every cluster."""
        from . import _lib
        n, d = x.shape
        sums = torch.zeros(k, d, dtype=torch.float32, device=x.device)
        counts = torch.zeros(k, dtype=torch.float32, device=x.device)
        a32 = a.to(torch.int32).contiguous()
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().rsb_kmeans_accumulate(ctypes.c_void_p(x.data_ptr()), n, d, ctypes.c_void_p(a32.data_ptr()), k,
                                                        ctypes.c_void_p(sums.data_ptr()), ctypes.c_void_p(counts.data_ptr()), self._st()))
        return sums, counts

    def pq_assign(self, r: torch.Tensor, cb: torch.Tensor) -> torch.Tensor:
        """codes uint8 [n, M] (one code per byte): nearest (L2) codebook entry of every sub-vector; cb [M, ksub, dsub],
        ksub 256 or 16."""
        from . import _lib
        n, d = r.shape
        M, ksub = cb.shape[0], cb.shape[1]
        codes = torch.empty(n, M, dtype=torch.uint8, device=r.device)
        with torch.cuda.device(r.device):
            _lib.check(_lib.lib().rsb_pq_assign(ctypes.c_void_p(r.data_ptr()), n, d, M, ksub,
                                                ctypes.c_void_p(cb.contiguous().data_ptr()),
                                                ctypes.c_void_p(codes.data_ptr()), self._st()))
        return codes

    def pq_accumulate(self, r: torch.Tensor, codes: torch.Tensor, M: int, ksub: int):
        from . import _lib
        n, d = r.shape
        sums = torch.zeros(M, ksub, d // M, dtype=torch.float32, device=r.device)
        counts = torch.zeros(M, ksub, dtype=torch.float32, device=r.device)
        with torch.cuda.device(r.device):
            _lib.check(_lib.lib().rsb_pq_accumulate(ctypes.c_void_p(r.data_ptr()), n, d, M, ksub,
                                                    ctypes.c_void_p(codes.data_ptr()), ctypes.c_void_p(sums.data_ptr()),
                                                    ctypes.c_void_p(counts.data_ptr()), self._st()))
        return sums, counts


_default_ops = None


def default_ops() -> LibrsbOps:
    global _default_ops
    if _default_ops is None:
        _default_ops = LibrsbOps()
    return _default_ops


def assign_ip(x: torch.Tensor, c: torch.Tensor, ops=None) -> torch.Tensor:
    """argmax_c <x, c> per row (the IndexFlatIP quantizer's assignment), int64 [n]."""
    return (ops or default_ops()).assign_ip(x.float().contiguous(), c.float().contiguous())


def kmeans(x: torch.Tensor, k: int, niter: int = 10, metric: str = "ip", spherical: bool = False,
           seed: int = 1234, max_points_per_centroid: int = 256, verbose: bool = False, ops=None) -> torch.Tensor:
    """x [n, d] float32 -> centroids [k, d] float32.  metric "ip": assignment by max inner product (what an IVF index
    with an IndexFlatIP quantizer does, spherical or not)."""
    if metric != "ip":
        raise NotImplementedError("coarse k-means assigns by inner product (the reference builds IP indexes only); "
                                  "L2 k-means exists for the PQ sub-quantizers: train_pq")
    assert x.dim() == 2 and x.shape[0] >= 1
    ops = ops or default_ops()
    x = x.float().contiguous()
    gen = torch.Generator(device=x.device)
    gen.manual_seed(seed)
    x = _subsample(x, k * max_points_per_centroid, gen).contiguous()
    n, d = x.shape
    if n <= k:  # degenerate: faiss would complain; keep going deterministically
        c = torch.zeros(k, d, dtype=torch.float32, device=x.device)
        c[:n] = x
        if n < k:
            c[n:] = x[torch.arange(k - n, device=x.device) % n]
        return torch.nn.functional.normalize(c, dim=1) if spherical else c
    c = x[torch.randperm(n, generator=gen, device=x.device)[:k]].clone()
    if spherical:
        c = torch.nn.functional.normalize(c, dim=1)
    for it in range(niter):
        a = ops.assign_ip(x, c.contiguous())
        sums, counts = ops.accumulate(x, a, k)
        nz = counts > 0
        c = torch.where(nz[:, None], sums / counts.clamp(min=1)[:, None], c)
        # empty clusters: split the largest ones with a symmetric perturbation (faiss split_clusters idea)
        empty = torch.nonzero(~nz).flatten()
        if empty.numel():
            donors = torch.argsort(counts, descending=True)[: empty.numel()]
            eps = 1.0 / 1024.0
            c[empty] = c[donors] * (1.0 + eps)
            c[donors] = c[donors] * (1.0 - eps)
        if spherical:
            c = torch.nn.functional.normalize(c, dim=1)
        if verbose:
            print(f"  kmeans it {it}: empty {int(empty.numel())}, largest cluster {int(counts.max().item())}")
    return c.contiguous()


def train_pq(residuals: torch.Tensor, M: int, ksub: int = 256, niter: int = 25, seed: int = 1234, ops=None) -> torch.Tensor:
    """residuals [n, d] -> codebook [M, ksub, d/M]; M independent L2 k-means.  ksub 256 (nbits 8) or 16 (nbits 4)."""
    if ksub not in (256, 16):
        raise NotImplementedError(f"ksub = {ksub}: only 8-bit (256) and 4-bit (16) sub-quantizers are implemented")
    ops = ops or default_ops()
    r = residuals.float()
    n, d = r.shape
    assert d % M == 0
    dsub = d // M
    gen = torch.Generator(device=r.device)
    gen.manual_seed(seed)
    r = _subsample(r, 256 * ksub, gen).contiguous()
    n = r.shape[0]
    xm = r.reshape(n, M, dsub).permute(1, 0, 2)                       # [M, n, dsub] view
    if n < ksub:
        reps = (ksub + n - 1) // n
        return xm.repeat(1, reps, 1)[:, :ksub].contiguous()
    perm = torch.randperm(n, generator=gen, device=r.device)[:ksub]
    cb = xm[:, perm].contiguous()                                     # [M, ksub, dsub]
    for _ in range(niter):
        codes = ops.pq_assign(r, cb)
        sums, counts = ops.pq_accumulate(r, codes, M, ksub)
        nz = counts > 0
        cb = torch.where(nz[..., None], sums / counts.clamp(min=1)[..., None], cb)
        # re-seed empty entries from random training points of the same sub-space
        if (~nz).any():
            idx = torch.randint(0, n, (M, ksub), generator=gen, device=r.device)
            repl = torch.gather(xm, 1, idx[..., None].expand(M, ksub, dsub))
            cb = torch.where(nz[..., None], cb, repl)
    return cb.contiguous()
