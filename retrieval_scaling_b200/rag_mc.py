"""Retrieval-augmented multiple-choice evaluation (MMLU, MedQA) by log-likelihood: the `multiple_choice` path of the
reference's lm-eval fork (`lm_eval --model hf --retrieval_file ... --concat_k K`, rag-evaluation-harness), restated as
host code around the GPU reader's `loglikelihood` (`reader.py`, `rsb_llm_loglikelihood`).

    samples     the harness's `--log_samples` output: one line {doc_id, doc, target, arguments} per document in
                samples_<task>_<date>.json, arguments = {gen_args_i: {arg_0: context, arg_1: continuation}}, one per
                choice (lm_eval/loggers/evaluation_tracker.py:237-285)
    retrieval   concat_k passages per question, prepended to the context as rag_qa does for generation
                (lm_eval/evaluator.py:479-514); retrieval_dir holds {task}_retrieved_results.jsonl per subtask
    encoding    _encode_pair (lm_eval/api/model.py:334-352), without special tokens
    scoring     the reader's loglikelihood, HFLM._loglikelihood_tokens (lm_eval/models/huggingface.py:948-1162)
    metric      acc (and acc_norm) of process_results (lm_eval/api/task.py:1356-1411); the mmlu group is the mean over
                every question of its subtasks (aggregate_subtask_metrics, size-weighted)

Few-shot prompts are not built here: the harness writes them into the samples, and the datasets are not read.
"""
from __future__ import annotations

import json
import logging
import os
import re
from typing import Dict, List, Optional, Sequence

import numpy as np

from . import rag_qa

CHOICES = ["A", "B", "C", "D"]                   # doc_to_choice of every task below
TARGET_DELIMITER = " "
GROUP = "mmlu"
# samples_<task>_<date>.json, date = datetime.now().isoformat() with ':' replaced by '-'
SAMPLES_NAME = re.compile(r"^samples_(?P<task>.+)_(?P<date>\d{4}-\d{2}-\d{2}T[0-9.\-]+)\.jsonl?$")


def task_metrics(task: str) -> Optional[tuple]:
    """The metric_list of a task of the table: medqa_4options acc and acc_norm, every mmlu_<subject> acc."""
    if task == "medqa_4options":
        return ("acc", "acc_norm")
    if task.startswith(GROUP + "_") and len(task) > len(GROUP) + 1:
        return ("acc",)
    return None


def is_mc_task(domain) -> bool:
    return isinstance(domain, str) and (domain == GROUP or task_metrics(domain) is not None)


# ---------------------------------------------------------------------------------------------------------------------
# samples (lm_eval/loggers/evaluation_tracker.py:237-285)
# ---------------------------------------------------------------------------------------------------------------------
def task_of_samples_file(name: str) -> Optional[str]:
    m = SAMPLES_NAME.match(os.path.basename(name))
    return m.group("task") if m else None


def samples_files(samples_dir: str, task: str) -> Dict[str, str]:
    """task -> samples file under samples_dir: `task` itself, or for the mmlu group every mmlu_<subject> found.  Two
    files of one task are refused, naming both."""
    found: Dict[str, str] = {}
    for name in sorted(os.listdir(samples_dir)):
        t = task_of_samples_file(name)
        if t is None or not (t == task or (task == GROUP and task_metrics(t) is not None and t.startswith(GROUP + "_"))):
            continue
        path = os.path.join(samples_dir, name)
        if t in found:
            raise ValueError(f"two samples files for task {t}: {found[t]} and {path}")
        found[t] = path
    if not found:
        raise FileNotFoundError(f"no samples_{task if task != GROUP else GROUP + '_*'}_<date>.json under {samples_dir}")
    return found


def read_samples(path: str) -> List[dict]:
    """One {doc_id, doc, target, context, choices} per logged document; every request must share one context and
    its continuation must be TARGET_DELIMITER + the choice, in choice order."""
    want = [TARGET_DELIMITER + c for c in CHOICES]
    docs = []
    with open(path) as f:
        for line in f:
            if not line.strip():
                continue
            s = json.loads(line)
            args = s["arguments"]
            reqs = [args[f"gen_args_{i}"] for i in range(len(args))]
            ctxs = {r["arg_0"] for r in reqs}
            conts = [r["arg_1"] for r in reqs]
            if len(ctxs) != 1 or conts != want:
                raise ValueError(f"{path}: doc {s.get('doc_id')}: the requests are not one context with the "
                                 f"continuations {want} (got {len(ctxs)} contexts, continuations {conts})")
            docs.append(dict(doc_id=s.get("doc_id"), doc=s.get("doc"), target=s.get("target"), context=ctxs.pop(),
                             choices=list(CHOICES)))
    return docs


# ---------------------------------------------------------------------------------------------------------------------
# encoding (lm_eval/api/model.py:334-352, lm_eval/models/huggingface.py)
# ---------------------------------------------------------------------------------------------------------------------
def prefix_token_id(tokenizer) -> int:
    """HFLM.prefix_token_id: BOS, else EOS (the eot token)."""
    return tokenizer.bos_token_id if tokenizer.bos_token_id is not None else tokenizer.eos_token_id


def encode_pair(tokenizer, context: str, continuation: str):
    """(context ids, continuation ids) of one request, without special tokens: an empty context is [prefix_token_id]
    (loglikelihood); otherwise the context's trailing whitespace moves to the continuation and the continuation is
    enc(context + continuation) past len(enc(context)), so a token merged across the boundary counts as continuation."""
    enc = lambda s: list(tokenizer.encode(s, add_special_tokens=False))   # noqa: E731
    if context == "":
        return [prefix_token_id(tokenizer)], enc(continuation)
    n_spaces = len(context) - len(context.rstrip())
    if n_spaces > 0:
        continuation = context[-n_spaces:] + continuation
        context = context[:-n_spaces]
    whole = enc(context + continuation)
    ctx = enc(context)
    return ctx, whole[len(ctx):]


# ---------------------------------------------------------------------------------------------------------------------
# metrics (lm_eval/api/task.py:1356-1411)
# ---------------------------------------------------------------------------------------------------------------------
def gold_index(target, choices: Sequence[str]) -> int:
    """The gold choice index, -100 when out of range (an int past the choices, a string that is not a choice)."""
    if isinstance(target, str) and target.strip().isdigit():
        target = int(target)
    if isinstance(target, (int, np.integer)) and not isinstance(target, bool):
        return int(target) if target < len(choices) else -100
    if isinstance(target, str):
        return choices.index(target) if target in choices else -100
    return -100


def score_doc(lls: Sequence[float], choices: Sequence[str], target) -> dict:
    """pred = argmax(lls), pred_norm = argmax(lls / len(choice)), np.argmax ties (the first); acc and acc_norm against
    the gold index, 0 for an out-of-range gold (with a warning)."""
    lls = np.asarray(lls, dtype=np.float64)
    pred = int(np.argmax(lls))
    pred_norm = int(np.argmax(lls / np.array([float(len(c)) for c in choices])))
    gold = gold_index(target, choices)
    if gold == -100:
        logging.warning(f"Label index was not in within range of available choices: target {target!r}")
    return dict(pred=pred, pred_norm=pred_norm, gold=gold, acc=1.0 if pred == gold else 0.0,
                acc_norm=1.0 if pred_norm == gold else 0.0)


class McOutput:
    """Accuracies of one task, or of the mmlu group with the per-subtask ones."""

    def __init__(self, cfg, task: str, n: int, metrics: Dict[str, float], subtasks: Dict[str, tuple]):
        self.cfg, self.task, self.n, self.metrics, self.subtasks = cfg, task, n, metrics, subtasks

    def log_message(self) -> str:
        m = "".join(f"\t{k} = {v:.4f}" for k, v in self.metrics.items())
        return f"Domain = {self.task}\tconcate_k = {self.cfg.evaluation.get('concate_k')}\tn = {self.n}{m}"


def aggregate(per_task: Dict[str, List[dict]], metrics: Sequence[str]) -> Dict[str, float]:
    """Size-weighted mean of each metric over the tasks' documents (aggregate_subtask_metrics), i.e. the mean over
    every document."""
    rows = [r for rs in per_task.values() for r in rs]
    return {k: (sum(r[k] for r in rows) / len(rows) if rows else float("nan")) for k in metrics}


# ---------------------------------------------------------------------------------------------------------------------
# the task
# ---------------------------------------------------------------------------------------------------------------------
def _args(cfg) -> dict:
    ev = cfg.evaluation.get("lm_eval", None) or {}
    return {k: ev.get(k, None) for k in ("samples_file", "samples_dir", "retrieval_file", "retrieval_dir",
                                         "predictions_file", "additional_system_prompt")}


def _tasks(task: str, args: dict) -> Dict[str, str]:
    if args["samples_dir"]:
        return samples_files(args["samples_dir"], task)
    if task == GROUP:
        raise ValueError("evaluation.lm_eval.samples_dir: the mmlu group reads every samples_mmlu_<subject>_<date>.json "
                         "under it")
    if not args["samples_file"]:
        raise ValueError("evaluation.lm_eval.samples_file (or samples_dir): the harness's --log_samples output is needed")
    return {task: args["samples_file"]}


def _prompts(cfg, args: dict, task: str, docs: List[dict], concat_k: int) -> List[str]:
    """Each document's context with its retrieved passages in front (lm_eval/evaluator.py:479-514).  With concat_k 0
    no retrieval file is read."""
    rows = [{"query": d["context"]} for d in docs]
    sys_prompt = args["additional_system_prompt"]
    if concat_k <= 0:
        return [(sys_prompt + r["query"]) if sys_prompt else r["query"] for r in rows]
    # retrieval_dir wins over retrieval_file (:483-486)
    path = os.path.join(args["retrieval_dir"], f"{task}_retrieved_results.jsonl") if args["retrieval_dir"] \
        else rag_qa.retrieval_path(cfg, args)
    if not os.path.exists(path):
        raise FileNotFoundError(f"retrieval path does not exist: {path}")
    hashed = rag_qa.hash_retrieval_results(rag_qa._load_jsonl(path), concat_k, task)
    return rag_qa.build_prompts(rows, hashed, sys_prompt)


def evaluate(cfg, model=None, tokenizer=None, model_config: Optional[dict] = None) -> McOutput:
    """`tasks.eval.inference` with task_name lm-eval on a multiple-choice task of the table (evaluation.domain)."""
    task = cfg.evaluation.get("domain")
    args = _args(cfg)
    files = _tasks(task, args)
    concat_k = int(cfg.evaluation.get("concate_k", 0) or 0)
    docs = {t: read_samples(p) for t, p in files.items()}
    prompts = {t: _prompts(cfg, args, t, docs[t], concat_k) for t in files}
    from .perplexity import load_lm_tokenizer
    from .reader import reader_dtype
    lm_dtype = (cfg.get("model") or {}).get("lm_dtype", None)
    try:
        dtype = reader_dtype("float16" if lm_dtype is None else lm_dtype)
    except ValueError as e:
        raise ValueError(f"model.lm_dtype: {e}") from None
    tokenizer = tokenizer or load_lm_tokenizer(cfg.model.lm_model)
    model_config = model_config or rag_qa.read_model_config(cfg.model.lm_model)
    if model is None:
        from .reader import load_reader
        model = load_reader(cfg.model.lm_model, dtype=dtype)
    max_len = rag_qa.max_length(model_config, tokenizer)
    requests, where, ctx_len = [], [], {}
    for t in files:
        for i, (d, p) in enumerate(zip(docs[t], prompts[t])):
            for c in d["choices"]:
                requests.append(encode_pair(tokenizer, p, TARGET_DELIMITER + c))
                where.append((t, i))
            ctx_len[(t, i)] = len(requests[-1][0])
    results = model.loglikelihood(requests, max_len)
    per_doc: Dict[tuple, list] = {}
    for key, r in zip(where, results):
        per_doc.setdefault(key, []).append(r)
    scored: Dict[str, List[dict]] = {t: [] for t in files}
    preds = []
    for t in files:
        for i, d in enumerate(docs[t]):
            lls, greedy = zip(*per_doc[(t, i)])
            s = score_doc(lls, d["choices"], d["target"])
            scored[t].append(s)
            keep = task_metrics(t)
            preds.append(dict(doc_id=d["doc_id"], task=t, prompt_tokens=ctx_len[(t, i)], loglikelihoods=list(lls),
                              is_greedy=list(greedy), pred=s["pred"], pred_norm=s["pred_norm"], gold=s["gold"],
                              **{k: s[k] for k in keep}))
    metrics = task_metrics(task) or ("acc",)
    subtasks = {t: (len(scored[t]), aggregate({t: scored[t]}, metrics)) for t in files}
    if task == GROUP:
        for t, (n, m) in subtasks.items():
            logging.info(f"{t}: n = {n}" + "".join(f"\t{k} = {v:.4f}" for k, v in m.items()))
    out = McOutput(cfg, task, sum(len(v) for v in scored.values()), aggregate(scored, metrics), subtasks)
    if args["predictions_file"]:
        d = os.path.dirname(args["predictions_file"])
        if d:
            os.makedirs(d, exist_ok=True)
        with open(args["predictions_file"], "w") as f:
            for p in preds:
                f.write(json.dumps(p) + "\n")
    logging.info(out.log_message())
    return out
