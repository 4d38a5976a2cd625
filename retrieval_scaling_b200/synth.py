"""Deterministic, chunk-addressable synthetic corpora (SURVEY.md §8d).

  iid : corpus and queries ~ N(0,1) i.i.d.  (BASELINE config 1 parity; worst case for IVF recall)
  gmm : `n_centres` latent centres ~ N(0,1); point = centre + sigma * N(0,1); queries from the same mixture
        with fresh noise (meaningful recall@k at nprobe 32-64; unbalanced inverted lists like real data).

Chunk c (rows [c*rows, (c+1)*rows)) is generated from torch.Generator seed `seed_corpus + c` on the device it
is asked for, so a 100M x 768 corpus (307 GB in fp32) never materialises: it streams through the index
builder one chunk at a time and any rank can regenerate any chunk.  CPU and CUDA generators produce different
streams: small oracle-sized sets must be generated on one device and copied, never regenerated on the other.
"""
from __future__ import annotations

import torch


class Corpus:
    def __init__(self, d: int = 768, mode: str = "gmm", n_centres: int = 4096, sigma: float = 0.35,
                 seed_centres: int = 7, seed_corpus: int = 1234, seed_queries: int = 4321, device="cuda"):
        assert mode in ("gmm", "iid")
        self.d, self.mode, self.sigma = d, mode, sigma
        self.seed_corpus, self.seed_queries = seed_corpus, seed_queries
        self.device = torch.device(device)
        self.centres = None
        self.scale = 1.0 / float(d) ** 0.5
        if mode == "gmm":
            g = torch.Generator(device=self.device).manual_seed(seed_centres)
            self.centres = torch.randn(n_centres, d, generator=g, device=self.device)

    def _draw(self, n: int, seed: int) -> torch.Tensor:
        g = torch.Generator(device=self.device).manual_seed(seed)
        if self.mode == "iid":
            return torch.randn(n, self.d, generator=g, device=self.device)
        a = torch.randint(0, self.centres.shape[0], (n,), generator=g, device=self.device)
        x = torch.randn(n, self.d, generator=g, device=self.device)
        x.mul_(self.sigma).add_(self.centres[a])
        # Unit-scale norms (|centre| ~ 1, like real encoder outputs).  Inner-product ranking is scale invariant, but
        # faiss trains IP indexes with *spherical* (unit-norm) centroids (SURVEY App. A.2): with |x| ~ sqrt(d) the
        # residual x - c barely shrinks and residual PQ drowns the signal (recall@100 near zero).
        x.mul_(self.scale)
        return x

    def chunk(self, c: int, rows: int = 1_000_000) -> torch.Tensor:
        return self._draw(rows, self.seed_corpus + c)

    def queries(self, nq: int) -> torch.Tensor:
        return self._draw(nq, self.seed_queries)

    def calibration_queries(self, nq: int) -> torch.Tensor:
        """Queries from the query distribution but an independent stream (never the ones that are searched):
        used to estimate how often each inverted list is probed when lists are assigned to GPUs."""
        return self._draw(nq, self.seed_queries + 1_000_003)

    def train_sample(self, n: int, seed: int = 99) -> torch.Tensor:
        """Training points drawn from the corpus distribution (independent stream)."""
        return self._draw(n, seed * 1_000_003)
