"""fp64 ORACLE (test infrastructure, NOT product code) of the reader's greedy choice (`rsb_llm_greedy`, the last step of
every `rsb_llm_generate` step): per row of logits, the id of the largest value over the real vocabulary [0, vocab) --
the lowest id on ties, as numpy's and torch's argmax -- and its log-softmax x[id] - logsumexp(x[:vocab]), with a bound
on the error of a kernel that computes it in fp32 as greedy_rows_kernel does."""
from __future__ import annotations

import numpy as np


def greedy(x, vocab: int, threads: int = 256):
    """(ids int64 [n], logprob float64 [n], bound float64 [n]) for logits x [n, >= vocab] (any float dtype; columns at
    or past vocab are ignored, whatever they hold).

    bound is the largest |kernel - logprob| of a kernel that, like greedy_rows_kernel, keeps per thread a running
    (max m, sum s) over vectors of 8 logits (`threads` threads, so it = ceil(vocab / (8 threads)) vectors each), rescales
    s by expf(m_old - m_new) when the maximum grows, merges the threads' pairs in 5 shuffle levels and 7 more merges
    across warps, and returns x[id] - (M + logf(S)).  In units of u = 2^-24 (fp32 unit roundoff):
      relative error of S  rho = 5u (it + 13)             one expf (2 ulp = 4u) and one product per rescale a term goes
                                                          through, plus its own expf
                                 + u (8 it + 13)          the sums: 8 adds per vector, 13 merges
                                 + 2u sum_j p_j |x_j - M| the fp32 rounding of every exponent argument x - m; along the
                                                          chain of rescales of a term these arguments add up to at most
                                                          |x_j - M| twice
      |error| <= rho (1 + 2 rho) + 2u |log S| + u (|M + log S| + |logprob|)   logf to 1 ulp, the two final roundings."""
    x = np.asarray(x)[:, :vocab].astype(np.float64)
    ids = np.argmax(x, axis=1)
    M = x[np.arange(len(x)), ids]
    with np.errstate(invalid="ignore"):
        d = x - M[:, None]                       # -inf entries give -inf (weight 0)
    e = np.exp(d)
    S = e.sum(1)
    lp = -np.log(S)                              # x[id] - (M + log S)
    u = 2.0 ** -24
    it = -(-vocab // (8 * threads))
    spread = np.where(e > 0, e * np.abs(np.where(np.isfinite(d), d, 0.0)), 0.0).sum(1) / S
    rho = 5 * u * (it + 13) + u * (8 * it + 13) + 2 * u * spread
    bound = rho * (1 + 2 * rho) + 2 * u * np.abs(np.log(S)) + u * (np.abs(M + np.log(S)) + np.abs(lp))
    return ids, lp, bound
