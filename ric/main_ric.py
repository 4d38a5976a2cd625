#!/usr/bin/env python
"""Entry point with the reference's command line (`ric/main_ric.py:13-38`):

    PYTHONPATH=. python ric/main_ric.py --config-name <yaml> tasks.eval.search=true a.b=c ...

Hydra / OmegaConf are replaced by `retrieval_scaling_b200.config` (same YAML files, same dotted overrides).
Task switches: tasks.datastore.embedding (already-chunked passage shards -> embedding pickles, SURVEY §8f-4),
tasks.datastore.index (build or load the index; with model.sparse_retriever=bm25 the BM25 index of every listed shard
under {passages_dir}/bm25/{ids}/rsb_index), tasks.eval.search (query -> top-k, the hot path; dense, or BM25 on the GPU),
tasks.eval.merge_search (multi-source merge, MinHash de-duplication on the GPU and subsampling, reference :31-33),
tasks.eval.inference (task_name perplexity: reader-LM perplexity with concate_k retrieved documents prepended, the
Llama reader on the GPU, reference :35-38; perplexity_calibration and lm-eval raise NotImplementedError).
"""
import logging
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from retrieval_scaling_b200 import config as rcfg  # noqa: E402


def init_distributed() -> None:
    """`torchrun --nproc-per-node G ric/main_ric.py ...`: one process per GPU; the index shard groups of
    `datastore.index.index_shard_ids=[[0],[1],...]` are partitioned over the ranks and their top-k merged on the GPUs
    (retrieval_scaling_b200.search.search_dense_topk_distributed).  Without torchrun nothing changes."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world <= 1:
        return
    import torch
    import torch.distributed as dist
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if torch.cuda.is_available():
        torch.cuda.set_device(local)
        os.environ.setdefault("NCCL_NVLS_ENABLE", "0")     # a few MB per gather: NVLS set-up costs more than it saves
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    else:
        dist.init_process_group("gloo")


def main(cfg) -> None:
    init_distributed()
    logging.info("\n\n************** Experiment configuration ***********")
    logging.info("\n" + rcfg.to_yaml(cfg))

    if cfg.tasks.datastore.get("embedding", False):
        logging.info("\n\n************** Building Embedding ***********")
        from retrieval_scaling_b200.embed import generate_passage_embeddings
        generate_passage_embeddings(cfg)   # reference src/embed.py:110-167 (already-chunked passage shards only)

    if cfg.tasks.datastore.get("index", False):
        logging.info("\n\n************** Indexing ***********")
        from retrieval_scaling_b200.search import check_sparse_retriever
        if check_sparse_retriever(cfg):
            from retrieval_scaling_b200 import bm25
            bm25.build_index(cfg)   # reference src/index.py:164-207: one BM25 index over every listed shard
        else:
            from retrieval_scaling_b200.indicies.base import Indexer
            Indexer(cfg)   # reference src/index.py:46-57: constructing the Indexer builds / loads the index

    if cfg.tasks.eval.get("search", False):
        logging.info("\n\n************** Running Search ***********")
        from retrieval_scaling_b200.search import search_topk
        search_topk(cfg)

    if cfg.tasks.eval.get("merge_search", False):
        logging.info("\n\n************** Post Merging Searched Results from Multiple Domains ***********")
        from retrieval_scaling_b200.search import post_hoc_merge_topk_multi_domain
        post_hoc_merge_topk_multi_domain(cfg)
    if cfg.tasks.eval.get("inference", False):
        logging.info("\n\n************** Running Perplexity Evaluation ***********")
        from retrieval_scaling_b200.perplexity import evaluate_perplexity, log_results_separately
        outputs = evaluate_perplexity(cfg)     # reference :36-39; perplexity_calibration / lm-eval: NotImplementedError
        log_results_separately(cfg, outputs)


if __name__ == "__main__":
    name, path, overrides = rcfg.parse_cli(sys.argv[1:], os.path.join(os.path.dirname(os.path.abspath(__file__)), "conf"))
    logging.basicConfig(level=logging.INFO, stream=sys.stdout, format="%(asctime)s - %(name)s - %(levelname)s - %(message)s")
    main(rcfg.load_config(name, path, overrides))
