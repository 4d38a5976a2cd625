"""Perplexity evaluation with retrieved documents prepended: the reference's `task_name: perplexity`
(`src/data.py:271-366`, `src/evaluate_perplexity.py`, `src/decontamination.py`), restated as host code around the GPU
reader of `reader.py`.

    windows    prepare_ppl_eval_data / batch / batch_merged: the eval text cut into max_eval_data_seq_length-token
               windows every eval_stride tokens; the tokens scored by an earlier window become the window's query
    prompts    build_doc_prompts / extract_answer: concate_k retrieved documents, most relevant last, before the query;
               the answer is the window's text without the query
    decontam.  check_below_lexical_overlap_threshold: 'longest' common word run (ratio or word-count threshold) or
               13-word-gram 'jaccard'
    loss       evaluate_perplexity: context and answer tokenised separately, context labels -100, left truncation to
               max_position_embeddings, HF's per-window mean loss from `B200Llama.loss`, averaged over the windows

The reference's quirks are kept; each carries a comment citing its line.
"""
from __future__ import annotations

import json
import logging
import os
from typing import List, Optional, Sequence, Tuple

import numpy as np

IGNORE = -100


# ---------------------------------------------------------------------------------------------------------------------
# windows (src/data.py:332-436)
# ---------------------------------------------------------------------------------------------------------------------
def batch_merged(ids: np.ndarray, max_seq_length: int, stride: int, pad_token_id: int) -> Tuple[np.ndarray, np.ndarray]:
    """Windows of max_seq_length inputs starting every `stride` tokens of one id stream.  The targets are the inputs
    shifted by one; in each window only the targets past the previous window's end are kept, the rest are pad_token_id.
    The last window ends one token before the stream ends and is padded with pad_token_id to max_seq_length."""
    n = len(ids)
    last = n - 1                                 # the final id is only ever a target
    inputs, targets = [], []
    prev_end = 0
    begin = 0
    while begin < last:
        end = min(begin + max_seq_length, last)
        x = ids[begin:end].copy()
        y = ids[begin + 1:end + 1].copy()
        keep = end - prev_end
        if keep:                                 # already scored by the previous window; `[:-0]` pads nothing (src/data.py:403)
            y[:-keep] = pad_token_id
        if end == last and len(x) < max_seq_length:
            pad = np.full(max_seq_length - len(x), pad_token_id, dtype=x.dtype)
            x, y = np.concatenate([x, pad]), np.concatenate([y, pad])
        if len(x) != max_seq_length:
            raise ValueError(f"window [{begin}, {end}) of a {n}-token stream is not {max_seq_length} tokens")
        inputs.append(x)
        targets.append(y)
        prev_end = end
        if end == last:
            break
        begin += stride
    return np.stack(inputs), np.stack(targets)


def batch(input_ids: Sequence[Sequence[int]], max_seq_length: int, stride: int, pad_token_id: int):
    """batch_merged on each document on its own, concatenated in document order."""
    parts = [batch_merged(np.array(x), max_seq_length, stride, pad_token_id) for x in input_ids]
    return np.concatenate([p[0] for p in parts], 0), np.concatenate([p[1] for p in parts], 0)


def lm_pad_token_id(tokenizer) -> int:
    """The reference's pad id: eos when the tokenizer has one, else pad (src/data.py:337, evaluate_perplexity.py:110)."""
    return tokenizer.pad_token_id if tokenizer.eos_token_id is None else tokenizer.eos_token_id


def prepare_ppl_eval_data(data, tokenizer, max_seq_length: int, stride: int, merge: bool,
                          num_eval_samples: Optional[int] = None, seed: int = 310) -> List[dict]:
    """[{'raw_inputs', 'raw_query'}] per window: the window's inputs decoded, and its inputs whose target is the pad id
    (the tokens an earlier window already scored, plus the padding) decoded as the query."""
    ids = [tokenizer(ex["text"])["input_ids"] for ex in data]
    pad = lm_pad_token_id(tokenizer)
    if merge:
        flat = np.array([t for x in ids for t in x])
        all_inputs, all_targets = batch_merged(flat, max_seq_length, stride, pad)
    else:
        all_inputs, all_targets = batch(ids, max_seq_length, stride, pad)
    if num_eval_samples:
        # np.random.seed(seed) then np.random.permutation (src/data.py:350-352): the same legacy MT19937 stream
        order = np.random.RandomState(seed).permutation(len(all_inputs))[:num_eval_samples]
        all_inputs, all_targets = all_inputs[order], all_targets[order]
    out = []
    for x, y in zip(all_inputs.tolist(), all_targets.tolist()):
        query = [int(a) for a, b in zip(x, y) if b == pad]
        out.append({"raw_inputs": tokenizer.decode(x, skip_special_tokens=True),
                    "raw_query": tokenizer.decode(query, skip_special_tokens=True)})
    return out


# ---------------------------------------------------------------------------------------------------------------------
# decontamination (src/decontamination.py)
# ---------------------------------------------------------------------------------------------------------------------
def longest_common_run(a: Sequence[str], b: Sequence[str]) -> int:
    """Length of the longest run of equal consecutive words shared by a and b (dynamic programme over the end pair)."""
    best = 0
    prev = [0] * (len(b) + 1)
    for i in range(len(a)):
        cur = [0] * (len(b) + 1)
        ai = a[i]
        for j in range(len(b)):
            if ai == b[j]:
                cur[j + 1] = prev[j] + 1
                if cur[j + 1] > best:
                    best = cur[j + 1]
        prev = cur
    return best


def word_13grams(text: str) -> set:
    w = text.split()
    return {" ".join(w[i:i + 13]) for i in range(len(w) - 12)}


def jaccard(a: set, b: set) -> float:
    u = a | b
    return len(a & b) / len(u) if u else 0


def check_below_lexical_overlap_threshold(doc: str, gold_text: str, threshold=0.25, mode: str = "longest") -> bool:
    """True when `doc` may be prepended: its overlap with `gold_text` stays below the threshold.
    longest: the longest shared run of words (split on single spaces) is below int(threshold x gold words) for a
    threshold < 1, below `threshold` words otherwise; threshold 1 accepts every document.
    jaccard: the Jaccard similarity of the two texts' 13-word grams (split on whitespace) is at most threshold < 1."""
    if threshold == 1:
        return True
    if mode == "longest":
        gold_words = gold_text.split(" ")
        run = longest_common_run(doc.split(" "), gold_words)
        if threshold < 1:
            return run < int(len(gold_words) * threshold)
        return run < threshold
    if mode == "jaccard":
        if not threshold < 1:
            raise ValueError("jaccard decontamination takes a similarity threshold in [0, 1), not a word count")
        return not jaccard(word_13grams(doc), word_13grams(gold_text)) > threshold
    # any other mode falls through and returns None, which build_doc_prompts treats as "not below" (decontamination.py:13-33)
    return None


# ---------------------------------------------------------------------------------------------------------------------
# prompts (src/evaluate_perplexity.py:152-218)
# ---------------------------------------------------------------------------------------------------------------------
def extract_answer(raw_inputs: str, raw_query: str) -> str:
    """The window's text without its query, '<|endoftext|>' removed from both.  (The reference's fallbacks behind
    try / except cannot run: str.replace does not raise, evaluate_perplexity.py:207-217.)"""
    return raw_inputs.replace("<|endoftext|>", "").replace(raw_query.replace("<|endoftext|>", ""), "")


def build_doc_prompts(eval_data, args) -> Tuple[List[str], List[str], int]:
    """(contexts, answers, no_enough_docs_count).  Each context is up to concate_k retrieved texts, the most relevant
    nearest the query (each new document goes in front), then the query."""
    num_docs = args.get("concate_k", 0) or 0
    decontamination = args.get("decontamination", False)
    threshold = args.get("contamination_threshold", 0.5)
    method = args.get("decontamination_method", "longest")
    use_continuation = args.get("use_continuation", False)
    use_both = args.get("use_both_doc_and_continuation", False)
    contexts, answers = [], []
    no_enough_docs_count = 0
    for ex in eval_data[1:]:                     # the first example is skipped (evaluate_perplexity.py:162)
        answer = extract_answer(ex["raw_inputs"], ex["raw_query"])
        doc = ""
        no_enough_docs_count = 0                 # reset per example: the last example's value is returned (:165)
        if num_docs > 0:
            try:                                 # a missing / empty ctxs prepends nothing and is not counted (:166, :197-198)
                if ex["ctxs"][0] is not None:
                    added = idx = 0
                    while added < num_docs and idx < len(ex["ctxs"]):
                        c = ex["ctxs"][idx]
                        if use_both:
                            text = c["retrieval text"] + c["retrieval next text"] + " \n"
                        elif use_continuation:
                            text = c["retrieval next text"] + " \n"
                        else:
                            text = c["retrieval text"] + " \n"
                        if not decontamination or check_below_lexical_overlap_threshold(text, answer, threshold, method):
                            doc = text + doc
                            added += 1
                        idx += 1
                    if added == 0:
                        logging.info("No document prepended!")
                    if added < num_docs:
                        no_enough_docs_count += 1
            except (KeyError, IndexError, TypeError):
                logging.info("No document prepended!")
        contexts.append(doc + ex["raw_query"])
        answers.append(answer)
    return contexts, answers, no_enough_docs_count


def reader_inputs(tokenizer, context: str, answer: str, max_len: int, pad_token: int) -> Tuple[List[int], List[int]]:
    """(input_ids, labels) of one window as the reference builds them (evaluate_perplexity.py:121-132)."""
    # a tokenizer that adds BOS (Llama) adds it to both: the answer's BOS is scored; Pythia's adds none
    ctx = tokenizer(context, truncation=False)["input_ids"]
    ans = tokenizer(answer, truncation=False)["input_ids"]
    ids = list(ctx) + list(ans)
    labels = [IGNORE] * len(ctx) + list(ans)
    labels = [IGNORE if t == pad_token else t for t in labels]   # eos / pad answer tokens are not scored (:124)
    return ids[-max_len:], labels[-max_len:]                       # left truncation to max_position_embeddings (:127-128)


# ---------------------------------------------------------------------------------------------------------------------
# the task (src/evaluate_perplexity.py:35-149)
# ---------------------------------------------------------------------------------------------------------------------
class PplEvalOutput:
    def __init__(self, cfg, average_loss, perplexity, bit_per_byte, no_enough_docs_count=None):
        self.cfg = cfg
        self.average_loss = average_loss
        self.perplexity = perplexity
        self.bit_per_byte = bit_per_byte
        self.no_enough_docs_count = no_enough_docs_count

    def _g(self, *path):
        node = self.cfg
        for p in path:
            node = node.get(p) if hasattr(node, "get") else None
            if node is None:
                return None
        return node

    def log_message(self) -> str:
        c = self._g
        index_ids = c("datastore", "index", "index_shard_ids")
        msg = (f"Domain = {c('evaluation', 'domain')}\t DS_domain = {c('datastore', 'domain')}"
               f"\tconcate_k = {c('evaluation', 'concate_k')}\tavg Loss = {self.average_loss:.4f}"
               f"\tperplexity = {self.perplexity.item():.4f}\tbpb = {self.bit_per_byte.item():.4f}"
               f"\ttotal shards = {c('datastore', 'embedding', 'num_shards')}"
               f"\tsampled shards = {len(index_ids) if index_ids is not None else None}"
               f"\t#eval samples = {c('evaluation', 'data', 'num_eval_samples')}"
               f"\tds chunk size = {c('datastore', 'embedding', 'chunk_size')}"
               f"\teval chunk size = {c('evaluation', 'data', 'max_eval_data_seq_length')}"
               f"\teval stride = {c('evaluation', 'data', 'eval_stride')}\tall shards = {index_ids}")
        if self.no_enough_docs_count:
            msg += f"\tno enough docs = {self.no_enough_docs_count}"
        return msg

    def log_short_message(self) -> str:
        c = self._g
        return (f"Domain = {c('evaluation', 'domain')}\ttotal shards = {c('datastore', 'embedding', 'num_shards')}"
                f"\t#eval samples = {c('evaluation', 'data', 'num_eval_samples')}"
                f"\tconcate_k = {c('evaluation', 'concate_k')}\tavg Loss = {self.average_loss:.4f}"
                f"\tperplexity = {self.perplexity.item():.4f}\tbpb = {self.bit_per_byte.item():.4f}")


def load_lm_tokenizer(name: str):
    """The tokenizer of `model.lm_model` from a local directory or the HF cache (never downloaded)."""
    import transformers
    return transformers.AutoTokenizer.from_pretrained(name, local_files_only=True)


def summarize(cfg, losses: Sequence[float], no_enough_docs_count) -> PplEvalOutput:
    """Mean over windows of each window's mean loss (a NaN window makes it NaN, as in the reference), perplexity =
    exp in fp32 (`torch.tensor` of a Python float), bits per byte = log2(perplexity) / 8 (:141-145)."""
    import torch
    average_loss = sum(float(x) for x in losses) / len(losses)
    perplexity = torch.exp(torch.tensor(average_loss))
    return PplEvalOutput(cfg, average_loss, perplexity, torch.log2(perplexity) / 8, no_enough_docs_count)


def evaluate_perplexity(cfg, model=None, tokenizer=None) -> PplEvalOutput:
    """`tasks.eval.inference` with task_name perplexity.  concate_k 0 reads the eval windows; otherwise the merged
    search results (evaluation.search.merged_path, or the merged output path of the search)."""
    task = cfg.tasks.eval.get("task_name", "perplexity")
    if task == "perplexity_calibration":
        raise NotImplementedError("perplexity_calibration (src/evaluate_perplexity.py:220-297) is not implemented")
    if task != "perplexity":
        raise NotImplementedError(f"inference for task_name {task!r} is not implemented (lm-eval runs in its harness)")
    from .reader import reader_dtype
    lm_dtype = (cfg.get("model") or {}).get("lm_dtype", None)
    try:
        dtype = reader_dtype("float16" if lm_dtype is None else lm_dtype)
    except ValueError as e:
        raise ValueError(f"model.lm_dtype: {e}") from None
    args = cfg.evaluation
    if args.get("concate_k", 0):
        s = args.get("search") or {}
        path = s.get("merged_path", None)
        if not path:
            from .search import get_merged_search_output_path
            path = get_merged_search_output_path(cfg)
        with open(path) as f:
            eval_data = [json.loads(line) for line in f]
    else:
        from .search import load_eval_data
        eval_data = load_eval_data(cfg)
    contexts, answers, no_enough = build_doc_prompts(eval_data, args)
    tokenizer = tokenizer or load_lm_tokenizer(cfg.model.lm_model)
    if model is None:
        from .reader import load_reader
        model = load_reader(cfg.model.lm_model, dtype=dtype)
    pad = lm_pad_token_id(tokenizer)
    pairs = [reader_inputs(tokenizer, c, a, model.max_position_embeddings, pad) for c, a in zip(contexts, answers)]
    losses = model.loss([p[0] for p in pairs], [p[1] for p in pairs])
    out = summarize(cfg, losses, no_enough)
    logging.info(out.log_message())
    return out


def log_results_separately(cfg, outputs: PplEvalOutput) -> None:
    path = cfg.evaluation.get("results_only_log_file", None)
    if path:
        if os.path.dirname(path):
            os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "a+") as f:
            f.write("\n")
            f.write(outputs.log_message())
