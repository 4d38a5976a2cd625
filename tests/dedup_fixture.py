"""Seeded synthetic retrieval results for the multi-source merge / de-duplication tests: queries whose passages
include planted near-duplicate families, copies of the query, passages shorter than 13 words and non-ASCII text."""
import json
import os
import random

VOCAB = ["alpha", "beta", "gamma", "delta", "epsilon", "zeta", "eta", "theta", "iota", "kappa", "lambda", "mu",
         "nu", "xi", "omicron", "pi", "rho", "sigma", "tau", "upsilon", "phi", "chi", "psi", "omega", "café", "naïve",
         "Zürich", "東京", "данные", "𝔘nicode", "co-op", "l'été"] + [f"w{i}" for i in range(400)]
SEPARATORS = [" "] * 20 + ["\n", "\t", "  ", " ", "　", " "]


def _text(rng, n_words):
    words = [rng.choice(VOCAB) for _ in range(n_words)]
    return "".join(w + rng.choice(SEPARATORS) for w in words).strip(" ")


def _mutate(rng, text, n_edits):
    words = text.split(" ")
    for _ in range(n_edits):
        words[rng.randrange(len(words))] = rng.choice(VOCAB)
    return " ".join(words)


def passages_for_query(rng, query, n):
    out = []
    while len(out) < n:
        kind = rng.random()
        if kind < 0.55 or not out:
            out.append(_text(rng, rng.randint(20, 90)))
        elif kind < 0.8:                                 # a near-duplicate of an earlier passage
            out.append(_mutate(rng, rng.choice(out), rng.randint(0, 3)))
        elif kind < 0.87:                                # contaminated by the query
            out.append(query + " " + _text(rng, rng.randint(0, 3)))
        else:                                            # short
            out.append(_text(rng, rng.randint(1, 14)))
    return out


def make_examples(seed, n_queries, n_docs):
    rng = random.Random(seed)
    data = []
    for q in range(n_queries):
        if q % 7 == 3:
            query = "The passage refers to the following information: " + _text(rng, 30)
        else:
            query = _text(rng, rng.choice([5, 12, 13, 30, 60]))
        data.append({"raw_query": query, "ctxs": [{"retrieval text": t} for t in passages_for_query(rng, query, n_docs)]})
    return data


def write_sources(root, seed, n_queries, n_docs, domains=("pes2o", "wiki", "c4")):
    """One result file per domain under <root>/<domain>_datastore-256_chunk_size/..., as search_dense_topk writes them
    (scores as strings, "source" null); returns the path of the text file listing them."""
    rng = random.Random(seed)
    base = make_examples(seed, n_queries, len(domains) * n_docs)
    paths = []
    for d, dom in enumerate(domains):
        rows = []
        for q, ex in enumerate(base):
            ctxs = [None] if q == 0 else [
                {"id": [d, k], "source": None, "retrieval text": c["retrieval text"],
                 "retrieval score": str(round(rng.uniform(0.5, 2.5), 3 if k % 3 else 2))}
                for k, c in enumerate(ex["ctxs"][d * n_docs:(d + 1) * n_docs])]
            rows.append({"query": ex["raw_query"], "raw_query": ex["raw_query"], "ctxs": ctxs})
        path = os.path.join(root, f"{dom}_datastore-256_chunk_size", "top_100", "eval_retrieved_results.jsonl")
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")
        paths.append(path)
    listing = os.path.join(root, "paths_to_merge.txt")
    with open(listing, "w") as f:
        f.write("\n".join(paths) + "\n")
    return listing


def oracle_deduplicate(examples):
    from oracle import minhash_oracle as M
    for ex in examples:
        ex["ctxs"] = M.remove_duplicates_with_minhash(ex["ctxs"], string_for_decontamination=ex["raw_query"])
    return examples
