"""BM25 search on the GPU (rsb_bm25.cu through retrieval_scaling_b200.bm25) against the numpy oracle on seeded corpora.

The scorer sums the same fp32 contributions in the same order (ascending term id) as `oracle/bm25_oracle.scores_f32`,
so ids and scores are compared bit for bit, single- and multi-term alike; the float64 matrix of `scores_f64` bounds
the fp32 summation error.  Then `ric/main_ric.py` end to end on a tiny passage directory."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import bm25_oracle as O

from bm25_fixture import overrides, write_eval_data, write_passages, zipf_corpus, zipf_queries

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILE = 16384


def _index(tok, doc_off, n_terms):
    from retrieval_scaling_b200 import bm25
    return bm25.BM25Index.from_tokens(tok, doc_off, n_terms, sort_device="cuda").to_device("cuda")


def _search(ix, queries, k):
    D, I = ix.search_terms([ix.term_query(c) for c in queries], k)
    return D.cpu().numpy(), I.cpu().numpy()


def _check(ix, queries, k, D, I, f64_rows=8):
    arrays = (ix.offsets, ix.docs, ix.tfs, ix.norms, ix.sum_len)
    queries = [{t: c for t, c in qc.items() if 0 <= t < ix.n_terms} for qc in queries]    # unknown terms are dropped
    for q, clauses in enumerate(queries):
        Do, Io = O.topk(O.scores_f32(*arrays, list(clauses.items())), k)
        assert np.array_equal(I[q], Io), (q, np.nonzero(I[q] != Io)[0][:5])
        assert np.array_equal(D[q].view(np.uint32), Do.view(np.uint32)), q
    # float64: every returned score within the fp32 summation error, and nothing left out that beats the last hit by
    # more than that error
    sub = list(range(min(f64_rows, len(queries))))
    S = O.scores_f64(*arrays, [list(queries[q].items()) for q in sub])
    for r, q in enumerate(sub):
        hit = I[q] >= 0
        ref = S[r, I[q][hit]]
        tol = (len(queries[q]) + 2) * 2.0 ** -22 * np.maximum(ref, 1e-30)
        assert np.all(np.abs(D[q][hit].astype(np.float64) - ref) <= tol), q
        assert hit.sum() == min(k, int((S[r] > 0).sum())), q
        if hit.sum() == k:
            rest = np.ones(S.shape[1], bool)
            rest[I[q]] = False
            assert not rest.any() or S[r, rest].max() <= ref.min() + 2 * tol.max(), q


@pytest.mark.parametrize("n_docs", [1000, 2 * TILE + 77, 120_000])
def test_tile_edges_match_the_oracle_bit_for_bit(n_docs):
    n_terms = 3000
    tok, off = zipf_corpus(n_docs, n_terms, seed=n_docs)
    ix = _index(tok, off, n_terms)
    queries = zipf_queries(n_terms, 24, seed=1) + [{t: 1} for t in (0, 7, 1500)]          # single-term queries
    D, I = _search(ix, queries, 100)
    _check(ix, queries, 100, D, I)


def test_df_n_df_1_boosts_and_duplicates():
    n_docs, n_terms = 3 * TILE + 5, 500
    tok, off = zipf_corpus(n_docs, n_terms, seed=3)
    lens = np.diff(off)
    docs = [tok[off[d]:off[d + 1]] for d in range(n_docs)]
    every, once = n_terms, n_terms + 1                        # a term in every document, a term in one document
    docs = [np.concatenate([d, [every]]) for d in docs]
    docs[TILE + 3] = np.concatenate([docs[TILE + 3], [once]])
    for src, dst in ((10, 20), (10, TILE + 40), (5000, 2 * TILE + 1)):   # identical documents: equal scores
        docs[dst] = docs[src].copy()
    tok2 = np.concatenate(docs).astype(np.int32)
    off2 = np.concatenate([[0], np.cumsum([len(d) for d in docs])])
    ix = _index(tok2, off2, n_terms + 2)
    assert ix.df[every] == n_docs and ix.df[once] == 1 and lens.min() == 0
    queries = [{every: 1}, {once: 1}, {every: 3, once: 2}, {once: 1, 3: 4, 9: 2},
               {int(t): 1 for t in docs[10]}, {int(t): 2 for t in docs[5000]}]
    for k in (1, 100, 1000, 4096):
        D, I = _search(ix, queries, k)
        _check(ix, queries, k, D, I)
    D, I = _search(ix, [{int(t): 1 for t in docs[10]}], 100)
    at = list(I[0]).index(10)                                 # ties: the lower document first
    assert list(I[0][at:at + 3]) == [10, 20, TILE + 40] and D[0][at] == D[0][at + 1] == D[0][at + 2]


def test_k_beyond_hits_empty_and_unknown_queries():
    n_terms = 2000
    tok, off = zipf_corpus(5000, n_terms, seed=4)
    ix = _index(tok, off, n_terms)
    rare = int(np.argmin(np.where(ix.df > 0, ix.df, 10 ** 9)))
    queries = [{rare: 1}, {}, {n_terms + 5: 1}, {-1: 2}]
    D, I = _search(ix, queries, 50)
    _check(ix, queries, 50, D, I)
    assert (I[0] >= 0).sum() == ix.df[rare] < 50
    assert (I[1:] == -1).all() and (D[1:] == np.finfo(np.float32).min).all()


def test_long_queries_and_batches():
    n_docs, n_terms = 40_000, 5000
    tok, off = zipf_corpus(n_docs, n_terms, seed=5, mean_len=60)
    ix = _index(tok, off, n_terms)
    long_q = zipf_queries(n_terms, 3, seed=6, n_tokens=6000, s=0.6)
    assert min(len(q) for q in long_q) > 1000
    D, I = _search(ix, long_q, 1000)
    _check(ix, long_q, 1000, D, I, f64_rows=3)
    one = zipf_queries(n_terms, 1, seed=7)
    D, I = _search(ix, one, 10)
    _check(ix, one, 10, D, I)
    many = zipf_queries(n_terms, 2048, seed=8, n_tokens=20)
    D, I = _search(ix, many, 100)
    _check(ix, many, 100, D, I, f64_rows=16)
    # the same batch again, and split into workspace-sized batches: bitwise equal
    D2, I2 = _search(ix, many, 100)
    assert np.array_equal(D.view(np.uint32), D2.view(np.uint32)) and np.array_equal(I, I2)
    D3, I3 = (t.cpu().numpy() for t in ix.search_terms([ix.term_query(c) for c in many], 100, ws_budget=1 << 20))
    assert np.array_equal(D.view(np.uint32), D3.view(np.uint32)) and np.array_equal(I, I3)


def test_refusals_before_allocation():
    from retrieval_scaling_b200 import _lib, bm25
    tok, off = zipf_corpus(100, 50, seed=9)
    ix = _index(tok, off, 50)
    with pytest.raises(NotImplementedError):
        ix.search(["river"], 4097)
    L = _lib.lib()
    p = 16
    assert L.rsb_bm25_search(p, p, 100, p, p, p, 1, 4097, p, p, p, 1 << 20, None) == _lib.RSB_ERR_UNSUPPORTED
    assert b"4096" in L.rsb_bm25_last_error()
    assert L.rsb_bm25_search(p, p, 100, p, p, p, 1, 10, p, p, p, 8, None) == _lib.RSB_ERR_OOM
    assert b"workspace" in L.rsb_bm25_last_error()
    huge = bm25.BM25Index(np.array([0, 0]), np.zeros(0), np.zeros(0), np.zeros(1, np.uint8), 0)
    huge.device_bytes = lambda: 1 << 50
    with pytest.raises(MemoryError, match=str(1 << 50)):
        huge.to_device("cuda")


def test_main_ric_index_and_search_end_to_end(tmp_path):
    from retrieval_scaling_b200 import bm25, perplexity
    from retrieval_scaling_b200 import config as rcfg
    from retrieval_scaling_b200.search import get_search_output_path, load_jsonl
    root = str(tmp_path)
    pdir, texts = write_passages(root)
    eval_path = write_eval_data(root)
    ov = overrides(root, pdir, eval_path, n_docs=5)
    env = dict(os.environ, PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "ric", "main_ric.py"), "tasks.datastore.index=true",
                        "tasks.eval.search=true", *ov], cwd=root, env=env, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    cfg = rcfg.load_config("default", os.path.join(ROOT, "ric", "conf"), ov)
    out = load_jsonl(get_search_output_path(cfg, [0, 1]))
    ix = bm25.BM25Index.build(texts, sort_device=None)        # the same analysis, independently of the saved index
    rows = [json.loads(line) for line in open(eval_path)]
    assert len(out) == len(rows)
    for ex, row in zip(out, rows):
        assert ex["query"] == row["query"]
        if not row["query"]:
            assert ex["ctxs"] == [None]
            continue
        ids, w = ix.query_terms(row["query"])
        counts = {int(t): c for t, c in zip(*np.unique([ix.term_id[t] for t in bm25.analyze(row["query"])
                                                        if t in ix.term_id], return_counts=True))}
        assert sorted(counts) == list(ids)
        D, I = O.topk(O.scores_f32(ix.offsets, ix.docs, ix.tfs, ix.norms, ix.sum_len, list(counts.items())), 5)
        want = [{"retrieval text": texts[i], "retrieval score": float(d)} for d, i in zip(D, I) if i >= 0]
        assert ex["ctxs"] == want
    assert out[4]["ctxs"] == [] and out[5]["ctxs"] == []      # stopwords only; unknown words only
    contexts, _, _ = perplexity.build_doc_prompts(out, {"concate_k": 3})
    for ctx, ex in zip(contexts, out[1:]):
        docs = [c["retrieval text"] + " \n" for c in (ex["ctxs"] if ex["ctxs"] and ex["ctxs"][0] else [])][:3]
        assert ctx == "".join(reversed(docs)) + ex["raw_query"]


def _empty_rows(D, I):
    return (I == -1).all() and (D == np.finfo(np.float32).min).all()


def test_batches_without_a_known_term_return_empty_rows(tmp_path):
    """A batch in which no query has a clause hands the scorer zero-length term / weight arrays: every row is empty."""
    from retrieval_scaling_b200 import bm25
    _, texts = write_passages(str(tmp_path))
    ix = bm25.BM25Index.build(texts, sort_device="cuda").to_device("cuda")
    for batch in (["the"], ["zzyzx"], [""], ["the", "zzyzx quux", "and of it", ""]):
        D, I = ix.search(batch, 10)
        assert D.shape == I.shape == (len(batch), 10) and _empty_rows(D, I), batch
    D, I = _search(ix, [{}], 7)                                 # nq = 1, no clause, through the term-id path
    assert _empty_rows(D, I)
    q = "river banks and the national library"                  # nq = 1 with terms: the oracle's hits
    D, I = ix.search([q], 10)
    counts = {ix.term_id[t]: c for t, c in zip(*np.unique(bm25.analyze(q), return_counts=True)) if t in ix.term_id}
    Do, Io = O.topk(O.scores_f32(ix.offsets, ix.docs, ix.tfs, ix.norms, ix.sum_len, list(counts.items())), 10)
    assert np.array_equal(I[0], Io) and np.array_equal(D[0].view(np.uint32), Do.view(np.uint32)) and (Io >= 0).any()


def test_index_without_postings():
    from retrieval_scaling_b200 import bm25
    ix = bm25.BM25Index.build(["the of and", "... !", "it is"], sort_device="cuda")
    assert len(ix.docs) == 0 and ix.n_docs == 3 and ix.n_terms == 0
    ix.to_device("cuda")
    D, I = ix.search(["river", "the", ""], 5)
    assert _empty_rows(D, I)


def test_search_task_with_only_stopword_and_unknown_queries(tmp_path):
    from retrieval_scaling_b200 import bm25, search
    from retrieval_scaling_b200 import config as rcfg
    root = str(tmp_path)
    pdir, _ = write_passages(root)
    eval_path = os.path.join(root, "only_empty.jsonl")
    with open(eval_path, "w") as f:
        for q in ("", "the and of it", "zzyzx"):
            f.write(json.dumps({"query": q, "raw_inputs": q}) + "\n")
    cfg = rcfg.load_config("default", os.path.join(ROOT, "ric", "conf"), overrides(root, pdir, eval_path))
    bm25.build_index(cfg)
    search.search_topk(cfg)
    out = search.load_jsonl(search.get_search_output_path(cfg, [0, 1]))
    assert [ex["ctxs"] for ex in out] == [[None], [], []]
