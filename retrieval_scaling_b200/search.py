"""Search orchestration -- the reference's `tasks.eval.search` flow (`src/search.py`):

    search_topk(cfg) -> search_dense_topk(cfg)                  (:827-831, :213-309)
      load encoder -> load eval data -> embed_queries           (:48-108, GPU)
      Indexer(cfg).search(query_embs, n_docs)                   (:293-296, GPU here; faiss-CPU in the reference)
      add_passages_to_eval_data -> safe_write_jsonl             (:126-146, :810-824)
      post_hoc_merge_topk(cfg)                                  (:312-373)

Same function names, argument meaning, output file scheme and resume/overwrite behaviour, so the lm-eval
harness fork consumes the JSONL unchanged (`ctxs[i]["retrieval text"]`, `"retrieval score"` as str).
Multi-source merge with MinHash de-duplication and coin-flip subsampling (:386-546) is
`post_hoc_merge_topk_multi_domain`, its de-duplication on the GPU (`dedup.py`).

    search_topk(cfg) -> search_sparse_topk(cfg)   with model.sparse_retriever=bm25   (:763-807, :827-829)
      load eval data -> BM25Index.load(rsb_index/) -> analyze + score on the GPU (`bm25.py`, `rsb_bm25.cu`)
      passages by (shard, line) -> safe_write_jsonl, "retrieval score" as a JSON number as the reference writes it

Out of scope (SURVEY §2 #8): the answer-based re-ranking of the multi-source merge (`rerank_method`).
"""
from __future__ import annotations

import copy
import json
import logging
import os
import pickle as pkl
import random
import re
from typing import List

import numpy as np
import torch

from .config import ListConfig
from .indicies.base import Indexer

device = "cuda" if torch.cuda.is_available() else "cpu"


# ----------------------------------------------------------------------------------------------------------
# query embedding (reference src/search.py:48-108, Contriever / generic-HF-BERT branches)
# ----------------------------------------------------------------------------------------------------------
def _tokenize(tokenizer, texts: List[str], max_length: int):
    # transformers >= 5 dropped batch_encode_plus (SURVEY App. B); __call__ is equivalent
    fn = getattr(tokenizer, "batch_encode_plus", None) or tokenizer
    return fn(texts, return_tensors="pt", max_length=max_length, padding=True, truncation=True)


def embed_queries(args, queries, model, tokenizer, model_name_or_path):
    """list[str] -> np.ndarray [nq, d].  Batches of `per_gpu_batch_size`, pad-to-longest, truncate to
    `question_maxlength`; Contriever models mean-pool inside the model, other HF BERT checkpoints (dragon*)
    take the CLS row (`output.last_hidden_state[:, 0, :]`, reference :93-94).  A sentence-transformers model
    (`encoder.SentenceTransformerEncoder`, reference :49-61) tokenises with its own `max_seq_length` and returns its
    pooled (and Dense / Normalize) rows."""
    from .encoder import SentenceTransformerEncoder, is_sentence_transformers_name
    st = isinstance(model, SentenceTransformerEncoder) and is_sentence_transformers_name(model_name_or_path)
    if not st and any(t in model_name_or_path for t in ("sentence-transformers", "e5", "Qwen3", "drama", "ReasonIR", "GRIT")):
        raise AttributeError(f"{model_name_or_path}: this encoder family is out of scope of the GPU hot path "
                             f"(BERT-architecture Contriever / dragon checkpoints and sentence-transformers T5 / "
                             f"BERT-base models loaded with encoder.load_sentence_transformer only)")
    if hasattr(model, "eval"):
        model.eval()
    embeddings, batch = [], []
    bs = int(args.per_gpu_batch_size)
    # The encoder works on the un-padded token stream, so a sequence's embedding does not depend on what else
    # is in its batch: several reference-sized batches (default 64) are encoded in one forward (`encode_group`,
    # 2048 sequences, see bench.py's encoder block) and nothing is copied to the host until the end.
    group = max(bs, int(getattr(model, "encode_group", bs)) // bs * bs)
    lowercase = bool(args.get("lowercase", False)) if hasattr(args, "get") else False
    normalize = bool(args.get("normalize_text", False)) if hasattr(args, "get") else False
    if normalize:
        from .text import normalize as _normalize_text
    with torch.no_grad():
        for k, q in enumerate(queries):
            if lowercase:
                q = q.lower()
            if normalize:
                q = _normalize_text(q)
            batch.append(q)
            if len(batch) == group or k == len(queries) - 1:
                if st:
                    out = model.encode_batch(batch)
                else:
                    enc = _tokenize(tokenizer, batch, int(args.question_maxlength))
                    enc = {kk: vv.to(device) for kk, vv in enc.items()}
                    out = model(**enc)
                if "contriever" not in model_name_or_path and hasattr(out, "last_hidden_state"):
                    out = out.last_hidden_state[:, 0, :]
                embeddings.append(out)
                batch = []
    if not embeddings:   # reference quirk 7: torch.cat([]) raises on an empty query list; return an empty array
        return np.zeros((0, 768), dtype=np.float32)
    embeddings = torch.cat(embeddings, dim=0)
    embeddings = (embeddings if embeddings.dtype == torch.float16 else embeddings.float()).cpu().numpy()
    print(f"Questions embeddings shape: {embeddings.shape}")
    if hasattr(args, "get") and args.get("cache_query_embedding", False):
        with open(args.query_embedding_save_path, "wb") as fout:
            pkl.dump(embeddings, fout)
    return embeddings


# ----------------------------------------------------------------------------------------------------------
# result plumbing
# ----------------------------------------------------------------------------------------------------------
def add_passages_to_eval_data(data, passages, scores, db_ids, valid_query_idx, domain=None):
    assert len(valid_query_idx) == len(passages)
    valid = set(valid_query_idx)
    idx = 0
    for i, d in enumerate(data):
        if i in valid:
            d["ctxs"] = [
                {"id": db_ids[idx][c], "source": domain, "retrieval text": passages[idx][c],
                 "retrieval score": str(scores[idx][c])}
                for c in range(len(passages[idx]))
            ]
            idx += 1
        else:
            d["ctxs"] = [None]


def _shard_groups(index_args):
    ids = index_args.index_shard_ids
    if ids and isinstance(ids[0], (ListConfig, list, tuple)):
        return [list(g) for g in ids]
    return [list(ids)]


def get_search_output_path(cfg, index_shard_ids):
    eval_args = cfg.evaluation
    postfix = "_".join(str(s) for s in index_shard_ids)
    name = os.path.basename(eval_args.data.eval_data).replace(".jsonl", "_retrieved_results.jsonl")
    return os.path.join(eval_args.eval_output_dir, postfix, name)


def get_merged_search_output_path(cfg):
    eval_args = cfg.evaluation
    groups = sorted(_shard_groups(cfg.datastore.index), key=lambda g: int(g[0]))
    postfix = "-".join("_".join(str(s) for s in g) for g in groups)
    name = os.path.basename(eval_args.data.eval_data).replace(".jsonl", "_retrieved_results.jsonl")
    return os.path.join(eval_args.eval_output_dir, postfix, name)


def safe_write_jsonl(data, output_file):
    """Write all-or-nothing: a partial file is removed on error (reference :810-824)."""
    success = False
    try:
        with open(output_file, "w") as fout:
            for ex in data:
                fout.write(json.dumps(ex) + "\n")
        success = True
        logging.info(f"Saved results to {output_file}")
    except Exception as e:  # noqa: BLE001 -- the reference swallows and reports
        print(f"An error occurred: {e}")
    finally:
        if not success and os.path.exists(output_file):
            os.remove(output_file)
            print(f"File '{output_file}' has been deleted due to an error.")


def load_jsonl(path):
    with open(path) as f:
        return [json.loads(line) for line in f if line.strip()]


def load_eval_data(cfg):
    """Eval-data adapter (reference `src/data.py:271-318`).  `lm-eval`: query = ex['query'].  `perplexity`: windows
    of ex['text'] in the tokens of `model.lm_model` (`perplexity.prepare_ppl_eval_data`); its tokenizer is read from a
    local directory or the HF cache only when this task asks for it."""
    path = cfg.evaluation.data.eval_data
    task = cfg.tasks.eval.task_name
    if not path.endswith(".jsonl"):
        raise ValueError(f"only .jsonl eval data is supported here, got {path}")
    data = load_jsonl(path)
    if task == "lm-eval":
        for ex in data:
            ex["raw_query"] = ex["query"]
        return data
    if task == "perplexity":                     # windows of the eval text in the reader's tokens (src/data.py:283-295)
        from .perplexity import load_lm_tokenizer, prepare_ppl_eval_data
        d = cfg.evaluation.data
        return prepare_ppl_eval_data(data, load_lm_tokenizer(cfg.model.lm_model), d.get("max_eval_data_seq_length", 1024),
                                     d.get("eval_stride", 512), d.get("merge", True), d.get("num_eval_samples", None),
                                     d.get("seed", 310))
    raise AttributeError(task)


# ----------------------------------------------------------------------------------------------------------
# the task
# ----------------------------------------------------------------------------------------------------------
def load_query_encoder(cfg):
    name = cfg.model.query_encoder
    from . import encoder as enc
    if "contriever" in name or "dragon" in name:
        model, tokenizer, _ = enc.load_retriever(name, tokenizer_name=cfg.model.get("query_tokenizer", name),
                                                 pooling="average" if "contriever" in name else "cls",
                                                 fp16=not cfg.datastore.index.get("no_fp16", False))
        return model, tokenizer
    if enc.is_sentence_transformers_name(name):         # reference :244-246: SentenceTransformer(name), no tokenizer
        return enc.load_sentence_transformer(name), None
    print(f"{name} is not supported!")
    raise AttributeError(name)


# ----------------------------------------------------------------------------------------------------------
# multi-GPU form of the task: one process per GPU (torchrun), the index shard groups of
# `datastore.index.index_shard_ids=[[0],[1],...]` partitioned over the ranks, per-group top-k combined on the GPUs.
# The reference runs one process per shard group and merges their JSONL files afterwards (`src/search.py:282-296`,
# `:312-373`); here the same merge rule ("concat in group order, stable sort by score descending, keep n_docs") runs
# as the peer-memory gather + merge kernel of `dist.ShardedSearcher`, and rank 0 writes the merged JSONL directly.
# ----------------------------------------------------------------------------------------------------------
GROUP_ID_SHIFT = 40          # merged ids carry the group: (group position << 40) | id inside that group's index


def assign_groups_to_ranks(ngroups: int, world: int):
    """Contiguous blocks of groups per rank, so that rank order == group order and the cross-rank merge breaks score
    ties exactly like the reference's stable sort over the groups in configuration order."""
    base, extra = divmod(ngroups, world)
    out, g = [], 0
    for r in range(world):
        n = base + (1 if r < extra else 0)
        out.append(list(range(g, g + n)))
        g += n
    return out


class GroupSearcher:
    """Index-like adapter over the shard groups one rank owns: `search_ids(q, k[, out])` searches every group and
    merges them (group order) into (ids with the group position encoded, scores)."""

    def __init__(self, indexers, group_positions, device=None):
        self.indexers, self.group_positions = list(indexers), list(group_positions)
        self.device = device

    def search_ids(self, q, k, out=None):
        from .index import merge_topk
        q = q if isinstance(q, torch.Tensor) else torch.as_tensor(np.asarray(q, dtype=np.float32))
        q = q.to(device=self.device or "cuda", dtype=torch.float32)
        Ds, Is = [], []
        for ix, gpos in zip(self.indexers, self.group_positions):
            I, D = ix.search_ids(q, k)
            Is.append(torch.where(I >= 0, I + (int(gpos) << GROUP_ID_SHIFT), I))
            Ds.append(D)
        if not Is:      # a rank without a group contributes padding only
            I = torch.full((q.shape[0], k), -1, dtype=torch.int64, device=q.device)
            D = torch.full((q.shape[0], k), float(np.finfo(np.float32).min), dtype=torch.float32, device=q.device)
        elif len(Is) == 1:
            I, D = Is[0], Ds[0]
        else:
            D, I = merge_topk(torch.stack(Ds), torch.stack(Is), k)
        if out is not None:
            out[0].copy_(I)
            out[1].copy_(D)
            return out
        return I, D


def _dist_state():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def embed_queries_sharded(cfg, queries, rank, world):
    """Each rank encodes its contiguous 1/world of the queries; the embeddings are all-gathered on the devices."""
    import torch.distributed as dist
    eval_args = cfg.evaluation
    per = (len(queries) + world - 1) // world
    lo, hi = min(len(queries), rank * per), min(len(queries), (rank + 1) * per)
    model, tokenizer = load_query_encoder(cfg)
    mine = embed_queries(eval_args.search, queries[lo:hi], model, tokenizer, cfg.model.query_encoder) if hi > lo else None
    d = int(cfg.datastore.index.projection_size)
    loc = torch.zeros((per, d), dtype=torch.float32, device=device)
    if mine is not None and len(mine):
        loc[: hi - lo] = torch.from_numpy(np.asarray(mine, dtype=np.float32)).to(device)
    allq = torch.empty((world * per, d), dtype=torch.float32, device=device)
    dist.all_gather_into_tensor(allq, loc)
    return allq[: len(queries)].cpu().numpy()


def search_dense_topk_distributed(cfg, rank, world):
    import torch.distributed as dist
    from .dist import ShardedSearcher
    from .indicies._common import DbIdMap
    index_args, eval_args = cfg.datastore.index, cfg.evaluation
    ds_domain = cfg.datastore.domain
    groups = _shard_groups(index_args)
    n_docs = int(eval_args.search.n_docs)
    merged_path = get_merged_search_output_path(cfg) if len(groups) > 1 else get_search_output_path(cfg, groups[0])
    overwrite = eval_args.search.get("overwrite", False)
    if os.path.exists(merged_path) and not overwrite:
        logging.info(f"{merged_path} exists, skipping searching.")
        return
    data = load_eval_data(cfg)
    queries, valid_query_idx = [], []
    for idx, ex in enumerate(data):
        if ex["raw_query"]:
            queries.append(ex["raw_query"])
            valid_query_idx.append(idx)
    cache = eval_args.search.get("query_embedding_save_path", "")
    if eval_args.search.get("cache_query_embedding", False) and cache and os.path.exists(cache):
        with open(cache, "rb") as fin:
            questions_embedding = pkl.load(fin)
    else:
        questions_embedding = embed_queries_sharded(cfg, queries, rank, world)
    mine = assign_groups_to_ranks(len(groups), world)[rank]
    logging.info(f"rank {rank}/{world}: index shard groups {[groups[g] for g in mine]}")
    indexers = [Indexer(cfg, index_shard_ids=groups[g]) for g in mine]
    local = GroupSearcher(indexers, mine, device=device)
    searcher = ShardedSearcher(local, world, rank, shard_coarse=False)
    q = torch.from_numpy(np.asarray(questions_embedding, dtype=np.float32)).to(device)
    I, D = searcher.search(q, n_docs)                     # replicated (ids, scores); ids carry the group position
    I, D = I.cpu().numpy(), D.cpu().numpy()
    # the reference's per-group artefacts: every rank writes the result files of the groups it owns
    for ix, g in zip(indexers, mine):
        out_g = get_search_output_path(cfg, groups[g])
        if len(groups) > 1 and (overwrite or not os.path.exists(out_g)):
            sc, psg, ids = ix.search(questions_embedding, n_docs)
            copied = copy.deepcopy(data)
            add_passages_to_eval_data(copied, psg, sc, ids, valid_query_idx, domain=ds_domain)
            os.makedirs(os.path.dirname(out_g), exist_ok=True)
            safe_write_jsonl(copied, out_g)
    if rank == 0:
        # passages of the merged rows: id -> (group, index id) -> [shard, chunk] through every group's .meta, text by
        # byte offset (the passage store is a shared directory; no index is loaded for groups of other ranks)
        gpos = (I >> GROUP_ID_SHIFT).astype(np.int64)
        local_id = I & ((1 << GROUP_ID_SHIFT) - 1)
        valid = I >= 0
        pairs = np.zeros(I.shape + (2,), dtype=np.int64)
        own = {g: ix.datastore for ix, g in zip(indexers, mine)}
        for g in range(len(groups)):
            sel = valid & (gpos == g)
            if not sel.any():
                continue
            if g in own:
                idmap = own[g].index_id_to_db_id
            else:
                idmap = DbIdMap.load(Indexer.artefact_paths(cfg, groups[g])["meta_file"])
            pairs[sel] = idmap.lookup(local_id[sel])
        any_store = indexers[0].datastore if indexers else None
        from .indicies import index_utils as iu
        pos_map = any_store.psg_pos_id_map if any_store is not None else None
        flat_pairs = pairs[valid]
        texts = [rec["text"] for rec in iu.fetch_passages(pos_map, flat_pairs)] if pos_map is not None else [None] * len(flat_pairs)
        all_scores, all_passages, db_ids, it = [], [], [], 0
        for row in range(I.shape[0]):
            nv = int(valid[row].sum())
            all_scores.append(D[row, :nv].tolist())
            all_passages.append(texts[it:it + nv])
            db_ids.append([[int(a), int(b)] for a, b in flat_pairs[it:it + nv]])
            it += nv
        merged = copy.deepcopy(data)
        add_passages_to_eval_data(merged, all_passages, all_scores, db_ids, valid_query_idx, domain=ds_domain)
        os.makedirs(os.path.dirname(merged_path), exist_ok=True)
        safe_write_jsonl(merged, merged_path)
    dist.barrier()


def search_dense_topk(cfg):
    rank, world = _dist_state()
    if world > 1:
        return search_dense_topk_distributed(cfg, rank, world)
    index_args, eval_args = cfg.datastore.index, cfg.evaluation
    ds_domain = cfg.datastore.domain
    groups = _shard_groups(index_args)
    overwrite = eval_args.search.get("overwrite", False)
    all_exist = all(os.path.exists(get_search_output_path(cfg, g)) for g in groups)
    if all_exist and not overwrite:
        logging.info(f"All search results for {index_args.index_shard_ids} exist, skipping searching.")
    else:
        data = load_eval_data(cfg)
        queries, valid_query_idx = [], []
        for idx, ex in enumerate(data):
            if ex["raw_query"]:
                queries.append(ex["raw_query"])
                valid_query_idx.append(idx)
        logging.info(f"Searching for {len(queries)} queries from {len(data)} total evaluation samples...")
        cache = eval_args.search.get("query_embedding_save_path", "")
        if eval_args.search.get("cache_query_embedding", False) and cache and os.path.exists(cache):
            with open(cache, "rb") as fin:
                questions_embedding = pkl.load(fin)
        else:
            model, tokenizer = load_query_encoder(cfg)
            questions_embedding = embed_queries(eval_args.search, queries, model, tokenizer, cfg.model.query_encoder)
        if eval_args.search.get("cache_query_embedding_only", False):
            return
        for g in groups:
            output_path = get_search_output_path(cfg, g)
            if os.path.exists(output_path) and not overwrite:
                logging.info(f"{output_path} exists, skipping searching.")
                continue
            copied = copy.deepcopy(data)
            logging.info("Loading or constructing the datastore...")
            index = Indexer(cfg, index_shard_ids=g)      # the reference drops `g` here (App. D quirk 1)
            logging.info("Searching for the queries...")
            all_scores, all_passages, db_ids = index.search(questions_embedding, eval_args.search.n_docs)
            add_passages_to_eval_data(copied, all_passages, all_scores, db_ids, valid_query_idx, domain=ds_domain)
            os.makedirs(os.path.dirname(output_path), exist_ok=True)
            safe_write_jsonl(copied, output_path)
    if eval_args.search.get("merge_multi_source_results", False) and eval_args.search.get("topk_subsample_p", None):
        post_hoc_merge_topk_multi_domain(cfg)
    elif eval_args.search.get("merge_multi_index_results", True):
        post_hoc_merge_topk(cfg)


def merge_ctxs(ctxs_per_shard: List[list], n_docs: int) -> list:
    """The reference's merge rule (`:357-367`): concat in shard order, stable sort by float(score) descending,
    keep n_docs.  (On the GPU path the same rule is `rsb_merge_topk`.)"""
    merged = [c for ctxs in ctxs_per_shard for c in ctxs if c is not None]
    merged.sort(key=lambda x: float(x["retrieval score"]), reverse=True)
    return merged[:n_docs]


def post_hoc_merge_topk(cfg):
    groups = _shard_groups(cfg.datastore.index)
    output_path = get_merged_search_output_path(cfg)
    if len(groups) <= 1:
        print("Single-index mode: no need to merge")
        return
    if os.path.exists(output_path) and not cfg.evaluation.search.get("overwrite", False):
        print(f"The merged path exists, skipping...\n{output_path}")
        return
    n_docs = cfg.evaluation.search.n_docs
    per_shard = [load_jsonl(get_search_output_path(cfg, g)) for g in groups]
    merged = per_shard[0]
    for rows in zip(*per_shard):
        assert all(r["raw_query"] == rows[0]["raw_query"] for r in rows)
    for i, ex in enumerate(merged):
        lists = [[c for c in (rows[i].get("ctxs") or []) if c is not None] for rows in per_shard]
        ex["ctxs"] = merge_ctxs(lists, n_docs)
    os.makedirs(os.path.dirname(output_path), exist_ok=True)
    safe_write_jsonl(merged, output_path)


# ----------------------------------------------------------------------------------------------------------
# multi-source merge + MinHash de-duplication + coin-flip subsampling (reference src/search.py:377-566)
# ----------------------------------------------------------------------------------------------------------
DATASTORE_DOMAIN = re.compile(r"/([^/]+)_datastore")


def merged_before_dedup_path(base_merged_path: str) -> str:
    """Where the merged, not yet de-duplicated results go (reference :395).  The reference takes
    `basename.strip('dedup_')`: str.strip removes any of the characters 'd', 'e', 'u', 'p', '_' from both ends of the
    name, not the prefix "dedup_".  'dedup_merged.jsonl' gives 'merged.jsonl', but 'dedup_dev.jsonl' gives 'v.jsonl'
    and 'pubmed' gives 'bm'.  Kept as is, so that existing merged files are found under their names."""
    return os.path.join(os.path.dirname(base_merged_path), os.path.basename(base_merged_path).strip("dedup_"))


def subsample_by_coin_flip(items, probability):
    return [item for item in items if random.random() < probability]


def additional_remove_short_chunk(ctxs):
    """Drops passages of 12 or fewer space-separated pieces (`split(' ')`, unlike the de-duplication's `split()`)."""
    return [ctx for ctx in ctxs if len(ctx["retrieval text"].split(" ")) > 12]


def merge_multi_domain(paths_to_merge: List[str], n_docs: int) -> list:
    """The per-source result files, merged query by query (reference :414-461): the passages of a source without a
    "source" field are tagged with the domain of its path (`.../<domain>_datastore...`), the lists concatenated in file
    order, stably sorted on "retrieval score" descending and cut to n_docs.  The sort compares the stored values as
    they are: the result files hold scores as strings, so the order is the strings' lexicographic order."""
    merged = []
    for domain_idx, path in enumerate(paths_to_merge):
        print(f"Adding {path}")
        matches = DATASTORE_DOMAIN.findall(path)
        ds_domain = matches[0] if matches else None
        rows = []
        with open(path) as f:
            for line in f:
                try:
                    ex = json.loads(line)
                except Exception:  # noqa: BLE001 -- the reference reports the file and raises AttributeError
                    print(f"Line read error when reading {path}")
                    raise AttributeError
                if not ex["ctxs"] or ex["ctxs"][0] is None:
                    ctxs = []
                else:
                    if "source" not in ex["ctxs"][0].keys() or not ex["ctxs"][0]["source"]:
                        for ctx in ex["ctxs"]:
                            ctx["source"] = ds_domain
                    ctxs = ex["ctxs"]
                ex["ctxs"] = ctxs
                rows.append(ex)
        if domain_idx == 0:
            merged = rows
            continue
        for id_, (_, ex) in enumerate(zip(merged, rows)):
            assert merged[id_]["raw_query"] == ex["raw_query"]
            merged[id_]["ctxs"].extend(ex["ctxs"])
            if merged[id_]["ctxs"] and merged[id_]["ctxs"][0] is not None:
                merged[id_]["ctxs"] = sorted(merged[id_]["ctxs"], key=lambda x: x["retrieval score"], reverse=True)[:n_docs]
                assert len(merged[id_]["ctxs"]) == n_docs
            else:
                assert id_ == 0 or id_ == 983      # the reference's allowance for queries without passages
    return merged


def _read_jsonl_strict(path):
    with open(path) as f:
        return [json.loads(line) for line in f]


def post_hoc_merge_topk_multi_domain(cfg, deduplicate=None):
    """Merge the results of several sources (`evaluation.search.paths_to_merge`, a text file with one result file per
    line), de-duplicate them on the GPU, subsample each query's passages with probability `topk_subsample_p` and write
    `full_subsampled_{p}_{seed}_{basename(merged_path)}` next to `merged_path` (reference :386-546).

    Files: the merged results go to `merged_before_dedup_path(merged_path)` and are read back from there when that file
    exists; the de-duplicated results go to `merged_path`, and with `use_saved_dedup_data` an existing `merged_path` is
    read instead of merging and de-duplicating again.  `deduplicate(examples)` (in place) defaults to
    `dedup.deduplicate`.  Returns the output path."""
    s = cfg.evaluation.search
    if s.get("rerank_method", None):
        raise NotImplementedError(f"rerank_method={s.rerank_method}: re-ranking (lexical / inclusion / unigram_f1) "
                                  f"needs the task answer files and is not implemented")
    if deduplicate is None:
        from .dedup import deduplicate
    base_merged_path = s.merged_path
    merged_path = merged_before_dedup_path(base_merged_path)
    use_saved = s.get("use_saved_dedup_data", False)

    if not os.path.exists(base_merged_path) or not use_saved:
        if not os.path.exists(merged_path):
            paths_to_merge = []
            with open(s.paths_to_merge) as f:
                for line in f:
                    path = line.strip()
                    paths_to_merge.append(path)
                    assert os.path.exists(path), f"{path}"
            print(f"Merging files:\n{paths_to_merge}")
            merged_data = merge_multi_domain(paths_to_merge, s.n_docs)
            if os.path.dirname(merged_path):    # the reference writes here before creating the directory (and fails)
                os.makedirs(os.path.dirname(merged_path), exist_ok=True)
            safe_write_jsonl(merged_data, merged_path)
        else:
            merged_data = _read_jsonl_strict(merged_path)
        deduplicate(merged_data)

    if os.path.exists(base_merged_path) and use_saved:
        merged_data = _read_jsonl_strict(base_merged_path)
    else:
        if os.path.dirname(base_merged_path):
            os.makedirs(os.path.dirname(base_merged_path), exist_ok=True)
        safe_write_jsonl(merged_data, base_merged_path)

    p = s.topk_subsample_p
    seed = s.get("subsample_seed", 1000)
    if p < 1:                                   # the draws of random.random() after random.seed(seed), query by query
        random.seed(seed)
        for ex in merged_data:
            ex["ctxs"] = subsample_by_coin_flip(ex["ctxs"], p)
    for ex in merged_data:
        ex["ctxs"] = additional_remove_short_chunk(ex["ctxs"])
    no_enough_data_count = 0
    for ex in merged_data:
        if len(ex["ctxs"]) < 3:
            no_enough_data_count += 1
            print(f"WARNING: the subsampled documents only have {len(ex['ctxs'])} left!")
    output_path = os.path.join(os.path.dirname(base_merged_path),
                               f"full_subsampled_{str(p)}_{seed}_{os.path.basename(base_merged_path)}")
    if os.path.dirname(output_path):
        os.makedirs(os.path.dirname(output_path), exist_ok=True)
    safe_write_jsonl(merged_data, output_path)
    print(f"Saved merged results to {output_path} with {no_enough_data_count} documents having less than 5 documents.")
    return output_path


# ----------------------------------------------------------------------------------------------------------
# BM25 (reference src/search.py:763-807): one index over every passage of the listed shards, on one GPU
# ----------------------------------------------------------------------------------------------------------
def check_sparse_retriever(cfg):
    """`model.sparse_retriever`: None (dense) or "bm25"; anything else raises NotImplementedError naming it.  BM25
    runs one index on one GPU: under torchrun with more than one process it raises NotImplementedError."""
    name = cfg.model.get("sparse_retriever", None)
    if name and name != "bm25":
        raise NotImplementedError(f"model.sparse_retriever={name}: only bm25 is implemented")
    if name and _dist_state()[1] > 1:
        raise NotImplementedError("model.sparse_retriever=bm25 searches one index on one GPU; run it without torchrun")
    return name


def search_sparse_topk(cfg):
    """BM25 top-n_docs for every eval example, written to get_search_output_path(cfg, flattened shard ids):
    ctxs = [{"retrieval text", "retrieval score" (a JSON number, as the reference writes it)}] best first, [None] for
    an empty raw_query, [] for a query without hits."""
    from . import bm25
    from .indicies import index_utils as iu
    eval_args = cfg.evaluation
    shard_ids = bm25.flat_shard_ids(cfg)
    output_path = get_search_output_path(cfg, shard_ids)
    if os.path.exists(output_path) and not eval_args.search.get("overwrite", False):
        logging.info(f"All search results for {cfg.datastore.index.index_shard_ids} exist, skipping searching.")
        return
    data = load_eval_data(cfg)
    logging.info(f"Searching for {len(data)} total evaluation samples...")
    path = bm25.index_dir(cfg, shard_ids)
    if not os.path.exists(os.path.join(path, "meta.json")):
        raise FileNotFoundError(f"The BM25 index does not exist, build it first (tasks.datastore.index=true)\n"
                                f"Missing: {path}")
    n_docs = int(eval_args.search.n_docs)
    bm25.check_k(n_docs)
    index = bm25.BM25Index.load(path, device=device)
    valid = [i for i, ex in enumerate(data) if ex["raw_query"]]
    D, I = index.search([data[i]["raw_query"] for i in valid], n_docs)
    hit = I >= 0
    passages_dir = cfg.datastore.embedding.passages_dir
    pos_map = iu.get_passage_pos_ids(passages_dir, os.path.join(os.path.dirname(path), "passage_pos_id_map.pkl"))
    records = iu.fetch_passages(pos_map, index.db_ids(I[hit]))
    it = 0
    for ex in data:
        ex["ctxs"] = [None]
    for row, i in enumerate(valid):
        nh = int(hit[row].sum())
        data[i]["ctxs"] = [{"retrieval text": rec["text"], "retrieval score": float(s)}
                           for rec, s in zip(records[it:it + nh], D[row, :nh])]
        it += nh
    os.makedirs(os.path.dirname(output_path), exist_ok=True)
    safe_write_jsonl(data, output_path)


def search_topk(cfg):
    if check_sparse_retriever(cfg):
        search_sparse_topk(cfg)
    else:
        search_dense_topk(cfg)
