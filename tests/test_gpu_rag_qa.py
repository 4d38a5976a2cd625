"""End to end: `ric/main_ric.py` search plus lm-eval inference (retrieval-augmented QA with greedy generation on the GPU
reader) against a CPU transformers fp32 restatement of the lm-eval fork's `generate_until`: prompts built from the
search output, no special tokens, left truncation to max_length - max_gen_toks, a left-padded batch, `model.generate`
greedy until every row has emitted EOS (finished rows filled with pad), then decode, the cut at the stop terms and
the EOS string, and remove_whitespace.  The reader stops each sequence at its own EOS instead; the texts must agree.
A byte-level BPE tokenizer is trained in the test, so "\\n", "." and "," are real tokens."""
import json
import os
import re
import string
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, ROOT)

import llama_fixture as LF  # noqa: E402

pytestmark = pytest.mark.gpu
MAX_GEN = 16
MAX_POS = 160
DELTA = 0.05                                     # fp16 reader against fp32: a smaller top-2 margin is a near-tie
UNTIL = ["\n", ".", ","]


def _bpe(corpus):
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers, trainers
    from transformers import PreTrainedTokenizerFast
    tok = Tokenizer(models.BPE())
    tok.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False)
    tok.decoder = decoders.ByteLevel()
    trainer = trainers.BpeTrainer(vocab_size=LF.CONFIG["vocab_size"], special_tokens=["<unk>", "<s>", "</s>"],
                                  initial_alphabet=pre_tokenizers.ByteLevel.alphabet())
    tok.train_from_iterator(corpus, trainer)
    assert tok.get_vocab_size() <= LF.CONFIG["vocab_size"] and tok.token_to_id("</s>") == 2
    return PreTrainedTokenizerFast(tokenizer_object=tok, unk_token="<unk>", bos_token="<s>", eos_token="</s>",
                                   pad_token="<unk>")


def _em(pred, gold):
    """nq_open's exact_match, written out: articles removed, lower case, no punctuation, equality."""
    def norm(s):
        s = re.sub(r"\b(?:The |the |An |A |The |a |an )", "", s).lower()
        return s.translate(str.maketrans("", "", string.punctuation))
    return float(any(norm(pred) == norm(g) for g in gold))


def _fork_generate_until(hf, tok, prompts):
    """(prediction, near_tie) per prompt, the fork's procedure with transformers fp32 on the CPU."""
    enc = [tok.encode(p, add_special_tokens=False)[-(MAX_POS - MAX_GEN):] for p in prompts]
    n = max(len(e) for e in enc)
    ids = torch.tensor([[0] * (n - len(e)) + e for e in enc])
    mask = torch.tensor([[0] * (n - len(e)) + [1] * len(e) for e in enc])
    with torch.no_grad():
        out = hf.generate(ids, attention_mask=mask, do_sample=False, num_beams=1, max_new_tokens=MAX_GEN,
                          eos_token_id=2, pad_token_id=0, output_scores=True, return_dict_in_generate=True)
    eos = tok.decode([2], skip_special_tokens=False)
    res = []
    for b in range(len(prompts)):
        cont = out.sequences[b, n:].tolist()
        s = tok.decode(cont, skip_special_tokens=True)
        for term in UNTIL + [eos]:
            ss = s.split(term)
            s = ss[0]
            if not s and len(ss) > 1:
                s = ss[1]
        s = s[1:] if s.startswith(" ") else s
        end = cont.index(2) + 1 if 2 in cont else len(cont)
        top2 = torch.stack([out.scores[k][b] for k in range(end)]).topk(2, dim=-1).values
        res.append((s, bool(((top2[:, 0] - top2[:, 1]) < DELTA).any()), 2 in cont, cont[:end]))
    return res


def test_main_ric_lm_eval_against_transformers(tmp_path):
    from golden import roberta_fixture as RF
    from safetensors.torch import save_file

    from retrieval_scaling_b200 import config as C
    from retrieval_scaling_b200.search import get_merged_search_output_path
    rng = np.random.default_rng(12)
    syll = ["ka", "ri", "to", "men", "sa", "lo", "vi", "dun", "pe", "qua", "zor", "bel"]
    words = ["".join(rng.choice(syll, int(rng.integers(1, 4)))) for _ in range(200)]

    def sentence(n):
        w = [str(x) for x in rng.choice(words, n)]
        return " ".join(w[:n // 2]) + ", " + " ".join(w[n // 2:]) + "."
    passages = [" ".join(sentence(int(rng.integers(4, 12))) for _ in range(3)) for _ in range(120)]
    tok = _bpe(passages + ["\n".join(passages[:20])])

    cfg = dict(LF.CONFIG, max_position_embeddings=MAX_POS)
    reader_dir = LF.build_dir(str(tmp_path / "reader"), cfg)
    sd = LF.seeded_state_dict(cfg)
    sd["lm_head.weight"][2] *= 2.2               # EOS wins often enough that some rows stop early
    save_file({k: v.contiguous() for k, v in sd.items()}, os.path.join(reader_dir, "model.safetensors"))
    tok.save_pretrained(reader_dir)
    enc = RF.build(str(tmp_path / "enc"))

    psg_dir = tmp_path / "passages" / "dom" / "1-shards"
    psg_dir.mkdir(parents=True)
    with open(psg_dir / "raw_passages-0-of-1.jsonl", "w") as f:
        for i, t in enumerate(passages):
            f.write(json.dumps({"id": i, "title": f"t{i % 7}", "text": t}) + "\n")
    questions = [f"Q: {' '.join(str(x) for x in rng.choice(words, int(rng.integers(2, 6))))}?\nA:" for _ in range(12)]
    shots = "Answer these questions:\n\n" + "".join(f"Q: {words[i]} {words[i + 1]}?\nA: {words[i + 2]}\n\n"
                                                     for i in range(0, 10, 3))
    with open(tmp_path / "questions.jsonl", "w") as f:
        for q in questions:
            f.write(json.dumps({"query": q}) + "\n")
    ov = [f"datastore.datastore_root_dir={tmp_path}", "datastore.domain=dom", "evaluation.domain=nq_open",
          "model.datastore_encoder=dragon-roberta", f"model.query_encoder={enc['query']['dir']}",
          f"datastore.embedding.model_name_or_path={enc['context']['dir']}", "datastore.index.index_type=Flat",
          "evaluation.search.n_docs=5", f"evaluation.data.eval_data={tmp_path / 'questions.jsonl'}",
          f"model.lm_model={reader_dir}", "evaluation.concate_k=2", "tasks.eval.task_name=lm-eval",
          f"evaluation.lm_eval.prompts_file={tmp_path / 'prompts.jsonl'}", f"evaluation.lm_eval.max_gen_toks={MAX_GEN}",
          f"evaluation.lm_eval.predictions_file={tmp_path / 'pred.jsonl'}",
          f"evaluation.results_only_log_file={tmp_path / 'results.log'}"]
    main = [sys.executable, os.path.join(ROOT, "ric", "main_ric.py"), "--config-name", "perplexity"]
    r = subprocess.run(main + ["tasks.datastore.embedding=true", "tasks.eval.search=true", *ov], cwd=ROOT,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]

    # the fork's prompts: the harness's few-shot prompt after the retrieved passages, most relevant last
    retrieved = {}
    for line in open(get_merged_search_output_path(C.load_config("perplexity", os.path.join(ROOT, "ric", "conf"), ov))):
        row = json.loads(line)
        retrieved[row["raw_query"].split("\n\n")[-1]] = "".join(c["retrieval text"] for c in row["ctxs"][:2][::-1])
    prompts = [retrieved[q] + shots + q for q in questions]
    hf = LF.hf_model(cfg)
    hf.load_state_dict(sd, strict=False)
    oracle = _fork_generate_until(hf, tok, prompts)
    # golds: the oracle's own prediction, re-cased with punctuation, for every other question
    golds = [[o[0].upper() + "!"] if i % 2 == 0 else ["nothing of the kind"] for i, o in enumerate(oracle)]
    with open(tmp_path / "prompts.jsonl", "w") as f:
        for q, g in zip(questions, golds):
            f.write(json.dumps({"query": shots + q, "answer": g}) + "\n")
    r = subprocess.run(main + ["tasks.eval.inference=true", *ov], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]

    preds = [json.loads(line) for line in open(tmp_path / "pred.jsonl")]
    assert len(preds) == len(questions)
    ties = sum(o[1] for o in oracle)
    stopped = sum(o[2] for o in oracle)
    same = sum(p["prediction"] == o[0] for p, o in zip(preds, oracle))
    for p, o in zip(preds, oracle):
        assert p["prompt_tokens"] <= MAX_POS - MAX_GEN
        if not o[1]:
            assert p["prediction"] == o[0], (p, o)
    em = float(re.search(r"exact_match = ([0-9.]+)", open(tmp_path / "results.log").read()).group(1))
    want = sum(_em(p["prediction"], g) for p, g in zip(preds, golds)) / len(preds)
    print(f"lm-eval end to end: {same} of {len(preds)} predictions equal to the fp32 fork restatement, {ties} items "
          f"flagged as near-ties (top-2 margin < {DELTA}), {stopped} rows ended at EOS in the batched HF run, "
          f"exact_match {em:.4f} (oracle metric {want:.4f})")
    assert ties <= len(preds) // 2
    assert em == pytest.approx(want, abs=1e-4)
