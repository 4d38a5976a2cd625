"""Passage-side embedding (`tasks.datastore.embedding`, reference `src/embed.py:24-167`): SURVEY.md §8(f) row 4.

Re-uses the query encoder kernels (`B200Contriever`) at the reference's passage batch size to turn already-chunked
passage shards into the `(ids, embeddings)` pickles the indexers read:

    {passages_dir}/raw_passages-{shard}-of-{num_shards}.jsonl   ->   {embedding_dir}/{prefix}_{shard:02d}.pkl

What is NOT here: chunking raw corpora into passages (`src/data.py::fast_load_jsonl_shard`, CPU text processing,
SURVEY.md §2 out of scope) -- a missing passage shard raises with that explanation -- and the decoder-LLM encoder
families (Qwen3, drama, GritLM), which raise `AttributeError` like the reference does for unknown names
(`src/embed.py:131-133`).  Sentence-transformers models (GTR-T5, e5-base) run through
`encoder.SentenceTransformerEncoder` (reference `src/embed.py:25-40,130`).
"""
from __future__ import annotations

import json
import logging
import os
import pickle
from typing import Iterable, List, Sequence, Tuple

import numpy as np
import torch

from .search import _tokenize

_UNSUPPORTED = ("sentence-transformers", "e5", "Qwen3", "drama", "ReasonIR", "GRIT")


def passage_text(args, p: dict) -> str:
    """title + " " + text unless `no_title` (reference :48-51), then optional lower-casing / normalisation."""
    text = p["text"] if (args.get("no_title", False) or "title" not in p) else p["title"] + " " + p["text"]
    if args.get("lowercase", False):
        text = text.lower()
    if args.get("normalize_text", False):
        from .text import normalize
        text = normalize(text)
    return text


def embed_passages(args, passages: Iterable[dict], model, tokenizer) -> Tuple[list, np.ndarray]:
    """list of {"id", "text"[, "title"]} -> (ids, embeddings [n, d]); batches of `per_gpu_batch_size`, truncation to
    `passage_maxlength` tokens; Contriever checkpoints mean-pool inside the model, other HF BERT checkpoints take the
    CLS row (reference :66-79)."""
    name = str(args.model_name_or_path)
    from .encoder import SentenceTransformerEncoder, is_sentence_transformers_name
    st = isinstance(model, SentenceTransformerEncoder) and is_sentence_transformers_name(name)
    if not st and any(t in name for t in _UNSUPPORTED):
        raise AttributeError(f"{name}: this encoder family is out of scope of the GPU hot path "
                             f"(BERT-architecture Contriever / dragon checkpoints only)")
    from . import search as _search                      # device is resolved there (tests patch it)
    bs = int(args.per_gpu_batch_size)
    max_len = int(args.passage_maxlength)
    ids: list = []
    chunks: List[torch.Tensor] = []          # HOST tensors: a shard's embeddings never pile up on the GPU
    pending: List[tuple] = []                # (host tensor, copy-done event) of asynchronous device->host copies
    batch_ids, batch_text = [], []

    def flush():
        if st:                               # the model's own tokenisation and max_seq_length (reference :25-40)
            out = model.encode_batch(batch_text)
        else:
            enc = _tokenize(tokenizer, batch_text, max_len)
            enc = {k: v.to(_search.device) for k, v in enc.items()}
            out = model(**enc)
        if "contriever" not in name and hasattr(out, "last_hidden_state"):
            out = out.last_hidden_state[:, 0, :]
        out = out if out.dtype == torch.float16 else out.float()
        if out.is_cuda:
            # like the reference's per-batch `.cpu()` (src/embed.py:79) but asynchronous: the copy into pinned memory
            # overlaps the next batch's forward; at most two batches of embeddings live on the GPU
            host = torch.empty(out.shape, dtype=out.dtype, pin_memory=True)
            host.copy_(out, non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            pending.append((host, ev, out))
            while len(pending) > 2:
                h, e, _keep = pending.pop(0)
                e.synchronize()
                chunks.append(h)
        else:
            chunks.append(out)
        ids.extend(batch_ids)
        batch_ids.clear()
        batch_text.clear()

    with torch.no_grad():
        for p in passages:
            batch_ids.append(p["id"])
            batch_text.append(passage_text(args, p))
            if len(batch_text) == bs:
                flush()
                if len(ids) % (20 * bs) == 0:
                    logging.info(f"Encoded passages {len(ids)}")
        if batch_text:
            flush()
    for h, e, _keep in pending:
        e.synchronize()
        chunks.append(h)
    if not chunks:
        return [], np.zeros((0, 768), dtype=np.float32)
    return ids, torch.cat(chunks, dim=0).numpy()


def get_sharded_passages(args, all_passages: Sequence[dict]) -> Sequence[dict]:
    """Contiguous slice `shard_id` of `num_shards`, the last shard takes the remainder (reference :97-107)."""
    n = len(all_passages)
    size = n // int(args.num_shards)
    lo = int(args.shard_id) * size
    hi = n if int(args.shard_id) == int(args.num_shards) - 1 else lo + size
    return all_passages[lo:hi]


def load_passage_shard(args, shard_id: int) -> List[dict]:
    path = os.path.join(args.passages_dir, f"raw_passages-{shard_id}-of-{int(args.num_shards)}.jsonl")
    if not os.path.exists(path):
        raise NotImplementedError(
            f"{path} not found: chunking raw text into passages (src/data.py::fast_load_jsonl_shard) is CPU text "
            f"processing outside the GPU hot path; produce the passage shards with the reference, then embed here")
    with open(path, "r", encoding="utf-8") as f:
        return [json.loads(line) for line in f if line.strip()]


def load_passage_encoder(args):
    name = str(args.model_name_or_path)
    from . import encoder as enc
    if enc.is_sentence_transformers_name(name) and not ("contriever" in name or "dragon" in name):
        return enc.load_sentence_transformer(name), None  # reference :130: SentenceTransformer(name), no tokenizer
    if any(t in name for t in _UNSUPPORTED) or not ("contriever" in name or "dragon" in name):
        print(f"{name} is not supported!")
        raise AttributeError(name)
    model, tokenizer, _ = enc.load_retriever(name, tokenizer_name=args.get("tokenizer", None) or name,
                                             pooling="average" if "contriever" in name else "cls",
                                             fp16=not args.get("no_fp16", False))
    return model, tokenizer


def generate_passage_embeddings(cfg) -> List[str]:
    """One `(ids, embeddings)` pickle per shard id in `datastore.embedding.shard_ids`; existing files are kept unless
    `use_saved_if_exists` is false.  Returns the paths written or found."""
    if cfg.model.get("sparse_retriever", None):
        print("No need to run the embedding step for sparse retrieval, skipping...")
        return []
    args = cfg.datastore.embedding
    out_paths, encoder = [], None
    for shard_id in [int(i) for i in args.shard_ids]:
        save_path = os.path.join(args.embedding_dir, f"{args.prefix}_{shard_id:02d}.pkl")
        out_paths.append(save_path)
        if os.path.exists(save_path) and args.get("use_saved_if_exists", True):
            print(f"Embeddings exist in {save_path}")
            continue
        passages = load_passage_shard(args, shard_id)
        if encoder is None:
            logging.info(f"Loading retriever model from {args.model_name_or_path}...")
            encoder = load_passage_encoder(args)
        ids, emb = embed_passages(args, passages, *encoder)
        os.makedirs(args.embedding_dir, exist_ok=True)
        print(f"Saving {len(ids)} passage embeddings to {save_path}.")
        with open(save_path, "wb") as f:
            pickle.dump((ids, emb), f)
    return out_paths
