"""Seeded corpora for the BM25 tests: Zipf token-id corpora for the scorer, and a tiny passage directory of English
text (two shards, duplicate passages, possessives, stopwords) with eval data for the `main_ric` pipeline."""
import json
import os

import numpy as np

WORDS = ("running runner runs ran river rivers bank banks banking money monies loan loans city cities garden gardens "
         "gardening house houses housing market markets marketing energy energetic nation national nationalization "
         "study studies studied student students teacher teaching school schools library libraries book books").split()
FILLERS = ("the a of and to in is was it that this with for on not".split())


def zipf_corpus(n_docs, n_terms, seed, mean_len=30, s=1.1):
    """(tok, doc_off): document lengths uniform in [0, 2 * mean_len), empty documents included; term t drawn with
    probability proportional to (t + 1) ** -s."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 2 * mean_len, n_docs)
    p = (np.arange(1, n_terms + 1, dtype=np.float64)) ** -s
    tok = rng.choice(n_terms, size=int(lens.sum()), p=p / p.sum()).astype(np.int32)
    doc_off = np.zeros(n_docs + 1, dtype=np.int64)
    np.cumsum(lens, out=doc_off[1:])
    return tok, doc_off


def zipf_queries(n_terms, nq, seed, n_tokens=12, s=1.1):
    """[{term id: count}] drawn from the corpus distribution (so terms repeat: boosts)."""
    rng = np.random.default_rng(seed)
    p = (np.arange(1, n_terms + 1, dtype=np.float64)) ** -s
    p /= p.sum()
    out = []
    for _ in range(nq):
        ids, cnt = np.unique(rng.choice(n_terms, size=n_tokens, p=p), return_counts=True)
        out.append({int(i): int(c) for i, c in zip(ids, cnt)})
    return out


def _sentence(rng, n):
    words = []
    for _ in range(n):
        w = WORDS[rng.integers(len(WORDS))] if rng.random() < 0.7 else FILLERS[rng.integers(len(FILLERS))]
        if rng.random() < 0.05:
            w = w.capitalize() + "'s"
        words.append(w)
    return " ".join(words) + "."


def write_passages(root, seed=0, per_shard=(40, 30)):
    """{root}/passages/raw_passages-{i}-of-2.jsonl; shard 1 repeats three passages of shard 0 (duplicates), and each
    shard holds one passage with no indexed term.  Returns (passages_dir, texts in document order)."""
    rng = np.random.default_rng(seed)
    pdir = os.path.join(root, "passages")
    os.makedirs(pdir, exist_ok=True)
    texts = []
    shards = []
    for s, n in enumerate(per_shard):
        rows = [_sentence(rng, int(rng.integers(3, 40))) for _ in range(n)]
        rows[5] = "the of and ... !"                              # nothing left after analysis
        if s == 1:
            rows[2], rows[9], rows[20] = shards[0][1], shards[0][3], shards[0][1]
        shards.append(rows)
        with open(os.path.join(pdir, f"raw_passages-{s}-of-{len(per_shard)}.jsonl"), "w") as f:
            for i, t in enumerate(rows):
                f.write(json.dumps({"id": f"{s}-{i}", "text": t, "title": "not indexed"}) + "\n")
        texts.extend(rows)
    return pdir, texts


def write_eval_data(root, seed=1, n=12):
    """lm-eval style rows: `query` (the raw query), `raw_inputs`; one empty query, one of stopwords only and one of
    unknown words."""
    rng = np.random.default_rng(seed)
    rows = []
    for i in range(n):
        q = _sentence(rng, int(rng.integers(2, 30)))
        rows.append({"query": q, "raw_inputs": q + " continuation " + str(i)})
    rows[3]["query"] = ""
    rows[4]["query"] = "the and of it"
    rows[5]["query"] = "zzyzx quux"
    path = os.path.join(root, "eval.jsonl")
    with open(path, "w") as f:
        for r in rows:
            f.write(json.dumps(r) + "\n")
    return path


def overrides(root, pdir, eval_path, n_docs=5):
    return [f"datastore.datastore_root_dir={root}", "datastore.domain=toy", f"datastore.embedding.passages_dir={pdir}",
            "datastore.embedding.num_shards=2", "datastore.index.index_shard_ids=[[0],[1]]", "evaluation.domain=toy",
            f"evaluation.data.eval_data={eval_path}", f"evaluation.eval_output_dir={root}/out",
            f"evaluation.search.n_docs={n_docs}", "model.sparse_retriever=bm25"]
