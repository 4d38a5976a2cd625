"""Retrieval-augmented open-domain QA with greedy generation: the `generate_until` path of the reference's lm-eval fork
(`lm_eval --model hf --retrieval_file ... --concat_k K --num_fewshot 5`, rag-evaluation-harness), restated as host
code around the GPU reader's `generate` (`reader.py`, `rsb_llm_generate`).

    prompts     the harness's saved inputs (`--answer_save_dir`): one row {query: <few-shot prompt>, answer: <gold>} per
                instance (lm_eval/evaluator.py:455-473)
    retrieval   hash_retrieval_results: concat_k passages per question from this repo's search output
                (lm_eval/evaluator.py:812-843), prepended to the few-shot prompt (:486-506)
    generation  greedy decoding until the model's EOS or max_gen_toks new tokens; the task's `until` terms only cut the
                decoded text afterwards (lm_eval/models/huggingface.py:1236-1296)
    metric      remove_whitespace, take_first, then exact_match with the task YAML's settings, any gold counts

The fork's quirks are kept; each carries a comment citing its line.  Few-shot prompts are not built here: the harness
writes them, and the datasets they come from are not read.
"""
from __future__ import annotations

import json
import logging
import os
import re
import string
from typing import Dict, List, Optional, Sequence

# generation_kwargs.until of both tasks (lm_eval/tasks/nq_open/nq_open.yaml, tasks/triviaqa/default.yaml)
UNTIL = ["\n", ".", ","]
# exact_match settings of each task's metric_list, keyed by evaluation.domain
DOMAINS: Dict[str, dict] = {
    "nq_open": dict(regexes_to_ignore=[r"\b(?:The |the |An |A |The |a |an )"], ignore_case=True,
                    ignore_punctuation=True),
    "triviaqa": dict(regexes_to_ignore=[], ignore_case=True, ignore_punctuation=True),
}
# description and doc_to_text of each task, for retrieval rows keyed by 'question' (lm_eval/evaluator.py:825-827)
QUESTION_PROMPTS: Dict[str, tuple] = {
    "nq_open": ("Answer these questions:\n\n", "Q: {question}?\nA:"),
    "triviaqa": ("", "Question: {question}?\nAnswer:"),
}
DEFAULT_MAX_LENGTH = 2048                        # HFLM._DEFAULT_MAX_LENGTH
HF_UNSET_MAX_LENGTH = 1000000000000000019884624838656   # transformers' "no limit" tokenizer.model_max_length


def domain_settings(domain: str) -> dict:
    if domain not in DOMAINS:
        raise NotImplementedError(f"lm-eval task {domain!r} is not implemented (only {', '.join(DOMAINS)})")
    return DOMAINS[domain]


# ---------------------------------------------------------------------------------------------------------------------
# retrieval context (lm_eval/evaluator.py:486-506, :803-843)
# ---------------------------------------------------------------------------------------------------------------------
def extract_question(prompt: str) -> str:
    """The 0-shot question of a few-shot prompt: its text after the last '\\n\\n', the few-shot delimiter (:803-810)."""
    return prompt.split("\n\n")[-1]


def hash_retrieval_results(rows: Sequence[dict], concat_k: int, domain: Optional[str] = None) -> Dict[str, str]:
    """question -> the concatenated text of its first concat_k passages (:812-843)."""
    out: Dict[str, str] = {}
    for row in rows:
        # the key is raw_query, else query, cut at the few-shot delimiter (:820-823); a row with only 'question' is
        # keyed by the task's description + doc_to_text of it (:825-827)
        if "raw_query" in row or "query" in row:
            key = extract_question(row["raw_query"] if "raw_query" in row else row["query"])
        else:
            if domain not in QUESTION_PROMPTS:
                raise NotImplementedError(f"retrieval rows keyed by 'question' need the task's prompt template; "
                                          f"{domain!r} has none here (only {', '.join(QUESTION_PROMPTS)})")
            description, template = QUESTION_PROMPTS[domain]
            key = extract_question(description + template.format(question=row["question"]))
        ctx = ""
        for i in range(concat_k):
            # each passage goes in front, so the most relevant is last; no separator (:829-830).  The fork's bare
            # try / except skips a missing passage, or one with neither key, and goes on with the next (:831-832)
            try:
                c = row["ctxs"][i]
                ctx = (c["retrieval text"] if "retrieval text" in c.keys() else c["text"]) + ctx
            except Exception:
                continue
        out[key] = ctx                           # a later duplicate row wins (:834-842)
    return out


def build_prompts(rows: Sequence[dict], hashed: Dict[str, str], additional_system_prompt: Optional[str] = None):
    """The generation prompt of each instance: its retrieved context, then the whole few-shot prompt (:488-506)."""
    prompts = []
    for row in rows:
        prompt_end = row["query"]
        question = extract_question(prompt_end)
        if question not in hashed:
            # the fork's non-interactive path raises (:492-500)
            raise RuntimeError(f"question {question!r} has no row in the retrieval file")
        ctx = hashed[question]
        prompt = ctx + prompt_end
        if additional_system_prompt:
            # (:505-506) builds on the prompt above, so the context appears twice
            prompt = ctx + "\n\n" + additional_system_prompt + prompt
        prompts.append(prompt)
    return prompts


# ---------------------------------------------------------------------------------------------------------------------
# tokenisation and post-processing (lm_eval/models/huggingface.py)
# ---------------------------------------------------------------------------------------------------------------------
def max_length(model_config: dict, tokenizer) -> int:
    """HFLM.max_length (:388-400): n_positions, max_position_embeddings or n_ctx of the model config, else the
    tokenizer's model_max_length unless unset, else 2048."""
    for attr in ("n_positions", "max_position_embeddings", "n_ctx"):
        if attr in model_config:
            return int(model_config[attr])
    if hasattr(tokenizer, "model_max_length"):
        if tokenizer.model_max_length == HF_UNSET_MAX_LENGTH:
            return DEFAULT_MAX_LENGTH
        return int(tokenizer.model_max_length)
    return DEFAULT_MAX_LENGTH


def encode_prompt(tokenizer, prompt: str, max_ctx_len: int) -> List[int]:
    """tok_encode without special tokens, no BOS even for Llama (:739-761), left-truncated to max_ctx_len =
    max_length - max_gen_toks (:1250-1261)."""
    if max_ctx_len <= 0:
        raise ValueError(f"max_length - max_gen_toks = {max_ctx_len}: no room for the prompt")
    ids = list(tokenizer.encode(prompt, add_special_tokens=False))
    return ids[-max_ctx_len:]


def cut_at_stop_terms(text: str, until: Sequence[str]) -> str:
    """For each term: keep the text before its first occurrence; when that piece is empty and the term occurred, keep
    the piece after it instead (:1285-1296)."""
    for term in until:
        if len(term) > 0:
            pieces = text.split(term)
            text = pieces[0]
            if not text and len(pieces) > 1:
                text = pieces[1]
    return text


def remove_whitespace(text: str) -> str:
    """The remove_whitespace filter: exactly one leading space is dropped (lm_eval/filters/extraction.py:54-74)."""
    return text[1:] if text.startswith(" ") else text


def postprocess(tokenizer, cont: Sequence[int], eos_string: str) -> tuple:
    """(raw generation, filtered prediction) of one continuation: decode without special tokens (:1283), cut at
    UNTIL + [eos string] (:1238-1243), then remove_whitespace and take_first."""
    raw = tokenizer.decode(list(cont), skip_special_tokens=True)
    return raw, remove_whitespace(cut_at_stop_terms(raw, UNTIL + [eos_string]))


# ---------------------------------------------------------------------------------------------------------------------
# metric (lm_eval/api/task.py:1446-1469 and HF evaluate's exact_match)
# ---------------------------------------------------------------------------------------------------------------------
def exact_match(prediction: str, reference: str, regexes_to_ignore=(), ignore_case=False,
                ignore_punctuation=False) -> float:
    """HF evaluate's exact_match on one pair, from its published definition: every regex removed from both strings,
    then lower-casing, then removal of string.punctuation, then string equality."""
    for r in regexes_to_ignore:
        prediction, reference = re.sub(r, "", prediction), re.sub(r, "", reference)
    if ignore_case:
        prediction, reference = prediction.lower(), reference.lower()
    if ignore_punctuation:
        table = str.maketrans("", "", string.punctuation)
        prediction, reference = prediction.translate(table), reference.translate(table)
    return float(prediction == reference)


def gold_targets(answer) -> List[str]:
    """The targets of one instance: a list as given, a string as one target, triviaqa's answer dict by its aliases
    (doc_to_target '{{answer.aliases}}')."""
    if isinstance(answer, dict):
        answer = answer["aliases"]
    if isinstance(answer, str):
        return [answer]
    return [str(a) for a in answer]


def score(prediction: str, answer, settings: dict) -> float:
    """1.0 when the prediction matches any target (multiple_target, api/task.py:1446-1469), else 0.0."""
    return 1.0 if any(exact_match(prediction, g, **settings) for g in gold_targets(answer)) else 0.0


# ---------------------------------------------------------------------------------------------------------------------
# the task
# ---------------------------------------------------------------------------------------------------------------------
class LmEvalOutput:
    def __init__(self, cfg, n: int, exact_match: float):
        self.cfg, self.n, self.exact_match = cfg, n, exact_match

    def log_message(self) -> str:
        ev = self.cfg.evaluation
        return (f"Domain = {ev.get('domain')}\tconcate_k = {ev.get('concate_k')}\tn = {self.n}"
                f"\texact_match = {self.exact_match:.4f}")


def _lm_eval_args(cfg) -> dict:
    ev = cfg.evaluation.get("lm_eval", None) or {}
    return {k: ev.get(k, d) for k, d in (("prompts_file", None), ("retrieval_file", None), ("max_gen_toks", 256),
                                         ("predictions_file", None), ("additional_system_prompt", None))}


def retrieval_path(cfg, args: dict) -> str:
    if args["retrieval_file"]:
        return args["retrieval_file"]
    path = (cfg.evaluation.get("search") or {}).get("merged_path", None)
    if path:
        return path
    from .search import get_merged_search_output_path
    return get_merged_search_output_path(cfg)


def eos_token_ids(model_config: dict, tokenizer) -> List[int]:
    """generate()'s stopping ids: the model config's eos_token_id, an int or a list, else the tokenizer's."""
    e = model_config.get("eos_token_id", None)
    if e is None:
        e = tokenizer.eos_token_id
    if e is None:
        return []
    return [int(e)] if isinstance(e, int) else [int(x) for x in e]


def read_model_config(name: str) -> dict:
    """config.json of `model.lm_model`, a local directory or HF cache name (never downloaded)."""
    from .encoder import _resolve_model_dir
    with open(os.path.join(_resolve_model_dir(name), "config.json")) as f:
        return json.load(f)


def _load_jsonl(path: str) -> List[dict]:
    with open(path) as f:
        return [json.loads(line) for line in f if line.strip()]


def evaluate_lm_eval(cfg, model=None, tokenizer=None, model_config: Optional[dict] = None) -> LmEvalOutput:
    """`tasks.eval.inference` with task_name lm-eval: the fork's generate_until on evaluation.domain's task."""
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        raise NotImplementedError("lm-eval inference runs in one process (the reader is single-GPU)")
    settings = domain_settings(cfg.evaluation.get("domain"))
    args = _lm_eval_args(cfg)
    if not args["prompts_file"]:
        raise ValueError("evaluation.lm_eval.prompts_file: the harness's saved prompts (--answer_save_dir) are needed")
    max_gen = int(args["max_gen_toks"])
    if max_gen <= 0:
        raise ValueError(f"evaluation.lm_eval.max_gen_toks {max_gen} must be positive")
    rows = _load_jsonl(args["prompts_file"])
    concat_k = int(cfg.evaluation.get("concate_k", 0) or 0)
    hashed = hash_retrieval_results(_load_jsonl(retrieval_path(cfg, args)), concat_k, cfg.evaluation.get("domain"))
    prompts = build_prompts(rows, hashed, args["additional_system_prompt"])
    from .perplexity import load_lm_tokenizer
    from .reader import reader_dtype
    lm_dtype = (cfg.get("model") or {}).get("lm_dtype", None)
    try:
        dtype = reader_dtype("float16" if lm_dtype is None else lm_dtype)
    except ValueError as e:
        raise ValueError(f"model.lm_dtype: {e}") from None
    tokenizer = tokenizer or load_lm_tokenizer(cfg.model.lm_model)
    model_config = model_config or read_model_config(cfg.model.lm_model)
    if model is None:
        from .reader import load_reader
        model = load_reader(cfg.model.lm_model, dtype=dtype)
    max_ctx_len = max_length(model_config, tokenizer) - max_gen
    ids = [encode_prompt(tokenizer, p, max_ctx_len) for p in prompts]
    eos = eos_token_ids(model_config, tokenizer)
    # generate() stops a sequence only at EOS (the fork passes stop=[eos] and comments out `until`, :1270-1275)
    conts = model.generate(ids, max_gen, eos)
    # the eos string appended to until (:1238-1243): tok_decode(eot_token_id, skip_special_tokens=False)
    eos_string = tokenizer.decode([tokenizer.eos_token_id], skip_special_tokens=False) \
        if tokenizer.eos_token_id is not None else ""
    preds, total = [], 0.0
    for row, p_ids, cont in zip(rows, ids, conts):
        raw, pred = postprocess(tokenizer, cont, eos_string)
        s = score(pred, row["answer"], settings)
        total += s
        preds.append({"query": row["query"], "prompt_tokens": len(p_ids), "generation": raw, "prediction": pred,
                      "gold": row["answer"], "exact_match": s})
    out = LmEvalOutput(cfg, len(rows), total / len(rows) if rows else float("nan"))
    if args["predictions_file"]:
        d = os.path.dirname(args["predictions_file"])
        if d:
            os.makedirs(d, exist_ok=True)
        with open(args["predictions_file"], "w") as f:
            for p in preds:
                f.write(json.dumps(p) + "\n")
    logging.info(out.log_message())
    return out


def log_results_separately(cfg, outputs: LmEvalOutput) -> None:
    path = cfg.evaluation.get("results_only_log_file", None)
    if path:
        if os.path.dirname(path):
            os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "a+") as f:
            f.write("\n")
            f.write(outputs.log_message())
