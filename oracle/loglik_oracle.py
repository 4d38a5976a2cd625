"""fp64 ORACLE (test infrastructure, NOT product code) of the reader's multiple-choice scoring (`rsb_llm_loglikelihood`,
choice_rows_kernel): the log-softmax x[row, token] - logsumexp(x[row, :vocab]) of chosen (row, token) targets and
whether token is the row's argmax (lowest id on ties), with a bound on the error of a kernel that computes it in fp32
by greedy_rows_kernel's single pass."""
from __future__ import annotations

import numpy as np

from .greedy_oracle import greedy


def choices(x, vocab: int, rows, tokens, threads: int = 256):
    """(logprob float64 [n], greedy bool [n], bound float64 [n]) of the targets (rows[i], tokens[i]) of logits
    x [m, >= vocab] (columns at or past vocab ignored).  The bound is greedy_oracle.greedy's, whose last term u |lp|
    (the final subtraction's rounding) is taken at the target's log-probability instead of the argmax's."""
    ids, lp_top, bound = greedy(x, vocab, threads)
    x = np.asarray(x)[:, :vocab].astype(np.float64)
    rows, tokens = np.asarray(rows, dtype=np.int64), np.asarray(tokens, dtype=np.int64)
    lse = x[np.arange(len(x)), ids] - lp_top     # M + log S
    lp = x[rows, tokens] - lse[rows]
    u = 2.0 ** -24
    b = bound[rows] - u * np.abs(lp_top[rows]) + u * np.abs(lp)
    return lp, ids[rows] == tokens, b
