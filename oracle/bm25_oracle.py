"""numpy restatement of BM25 search (Lucene 9 BM25Similarity, k1 = 0.9, b = 0.4) over a term-major posting index, the
oracle of `rsb_bm25_search`.  It takes the index's raw arrays and the queries' (term id, count) clauses and derives
everything else itself: docCount, avgdl, the norm cache, idf and the clause weights.

`scores_f32`: per-term contributions in numpy float32, accumulated in ascending term id.  numpy never fuses a multiply
and an add, so every operation is one IEEE float rounding, as in Java's float arithmetic.
`scores_f64`: the same scores from a float64 scipy.sparse [documents, terms] matrix, as a second check.
`topk`: documents with score > 0, best first, ties to the lower document number."""
from __future__ import annotations

import numpy as np
from scipy import sparse

K1, B = np.float32(0.9), np.float32(0.4)


def _byte4_to_int(b: int) -> int:        # SmallFloat.byte4ToInt (NUM_FREE_VALUES = 24)
    if b < 24:
        return b
    i = b - 24
    bits, shift = i & 7, (i >> 3) - 1
    return 24 + (bits if shift < 0 else (bits | 8) << shift)


def _cache(norms, sum_len):
    n = np.count_nonzero(norms)                                        # docCount
    avgdl = np.float32(sum_len / float(n)) if n else np.float32(1)
    table = np.array([_byte4_to_int(i) for i in range(256)], dtype=np.float32)
    return (np.float32(1) / (K1 * ((np.float32(1) - B) + B * table / avgdl))).astype(np.float32), n


def _weight(count, df, n):
    return np.float32(count) * np.float32(np.log(1.0 + (n - df + 0.5) / (df + 0.5)))


def scores_f32(offsets, docs, tfs, norms, sum_len, clauses):
    """clauses: [(term id, count)] of one query.  Returns fp32 [n_docs]."""
    cache, n = _cache(norms, sum_len)
    acc = np.zeros(len(norms), dtype=np.float32)
    for t, c in sorted(clauses):
        a, e = int(offsets[t]), int(offsets[t + 1])
        w = _weight(c, e - a, n)
        d = docs[a:e].astype(np.int64)
        x = np.float32(1) + tfs[a:e].astype(np.float32) * cache[norms[d]]
        acc[d] = acc[d] + (w - w / x)
    return acc


def scores_f64(offsets, docs, tfs, norms, sum_len, queries):
    """queries: [[(term id, count)]].  Returns float64 [nq, n_docs] = Q @ M^T with M[d, t] = 1 - 1 / x."""
    cache, n = _cache(norms, sum_len)
    n_terms = len(offsets) - 1
    terms = np.repeat(np.arange(n_terms), np.diff(offsets))
    x = 1.0 + tfs.astype(np.float64) * cache[norms[docs]].astype(np.float64)
    M = sparse.csr_matrix((1.0 - 1.0 / x, (docs, terms)), shape=(len(norms), n_terms))
    rows, cols, vals = [], [], []
    for qi, clauses in enumerate(queries):
        for t, c in clauses:
            df = int(offsets[t + 1] - offsets[t])
            rows.append(qi)
            cols.append(t)
            vals.append(float(c) * float(np.log(1.0 + (n - df + 0.5) / (df + 0.5))))
    Q = sparse.csr_matrix((vals, (rows, cols)), shape=(len(queries), n_terms))
    return np.asarray((Q @ M.T).todense())


def topk(scores, k):
    """(D fp32 [k], I int64 [k]) of the documents with score > 0: lexsort((doc, -score)), padded with -FLT_MAX / -1."""
    hit = np.nonzero(scores > 0)[0]
    order = hit[np.lexsort((hit, -scores[hit].astype(np.float64)))][:k]
    D = np.full(k, np.finfo(np.float32).min, dtype=np.float32)
    I = np.full(k, -1, dtype=np.int64)
    D[:len(order)] = scores[order]
    I[:len(order)] = order
    return D, I
