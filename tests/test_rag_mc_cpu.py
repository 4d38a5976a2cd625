"""CPU checks of the multiple-choice task (`rag_mc.py`) and of `_Reader.loglikelihood`'s host logic: samples parsing,
file-name -> task parsing, `_encode_pair` with a char tokenizer and a trained BPE, the empty-context prefix id,
windowing and truncation, grouping of identical windows, acc / acc_norm with ties, out-of-range golds, the mmlu
micro-average, retrieval precedence, and `main_ric` dispatch with a scripted reader."""
import json
import logging
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from retrieval_scaling_b200 import rag_mc as M  # noqa: E402
from retrieval_scaling_b200 import rag_qa as R  # noqa: E402

DATE = "2026-10-19T12-00-00.123456"


class _Tok:
    """One id per character; bos_token_id None makes EOS the prefix token."""
    model_max_length = R.HF_UNSET_MAX_LENGTH
    eos_token_id = 2
    bos_token_id = None

    def encode(self, s, add_special_tokens=True):
        assert add_special_tokens is False
        return [ord(c) for c in s]


def _sample(doc_id, ctx, target, conts=None):
    conts = conts or [" A", " B", " C", " D"]
    return {"doc_id": doc_id, "doc": {"q": ctx}, "target": target,
            "arguments": {f"gen_args_{i}": {"arg_0": ctx, "arg_1": c} for i, c in enumerate(conts)},
            "resps": [], "filtered_resps": []}


def _write_samples(path, samples):
    with open(path, "w") as f:
        for s in samples:
            f.write(json.dumps(s) + "\n")


def test_samples_parsing_and_task_names(tmp_path):
    assert M.task_of_samples_file(f"samples_mmlu_high_school_biology_{DATE}.json") == "mmlu_high_school_biology"
    assert M.task_of_samples_file(f"/x/samples_medqa_4options_{DATE}.json") == "medqa_4options"
    assert M.task_of_samples_file("results_2026-10-19T12-00-00.json") is None
    p = tmp_path / f"samples_mmlu_anatomy_{DATE}.json"
    _write_samples(p, [_sample(0, "Q1\nAnswer:", 2), _sample(1, "Q2\nAnswer:", 0)])
    docs = M.read_samples(str(p))
    assert [d["context"] for d in docs] == ["Q1\nAnswer:", "Q2\nAnswer:"] and [d["target"] for d in docs] == [2, 0]
    _write_samples(p, [_sample(0, "Q1\nAnswer:", 2, [" A", " B", " C", "D"])])
    with pytest.raises(ValueError, match="continuations"):
        M.read_samples(str(p))
    _write_samples(tmp_path / f"samples_mmlu_anatomy_{DATE}.json", [_sample(0, "Q", 0)])
    _write_samples(tmp_path / f"samples_mmlu_virology_{DATE}.json", [_sample(0, "Q", 0)])
    _write_samples(tmp_path / f"samples_medqa_4options_{DATE}.json", [_sample(0, "Q", 0)])
    (tmp_path / "results_x.json").write_text("{}")
    assert sorted(M.samples_files(str(tmp_path), "mmlu")) == ["mmlu_anatomy", "mmlu_virology"]
    assert list(M.samples_files(str(tmp_path), "medqa_4options")) == ["medqa_4options"]
    _write_samples(tmp_path / "samples_mmlu_virology_2026-10-20T01-02-03.000001.json", [_sample(0, "Q", 0)])
    with pytest.raises(ValueError, match="two samples files for task mmlu_virology:.*2026-10-19.*2026-10-20"):
        M.samples_files(str(tmp_path), "mmlu")


def test_encode_pair_char_tokenizer_and_prefix_id():
    tok = _Tok()
    ctx, cont = M.encode_pair(tok, "Answer: ", "A")     # the trailing space moves to the continuation
    assert ctx == [ord(c) for c in "Answer:"] and cont == [ord(" "), ord("A")]
    ctx, cont = M.encode_pair(tok, "Q\n\n", " B")
    assert ctx == [ord("Q")] and cont == [ord(c) for c in "\n\n B"]
    assert M.encode_pair(tok, "", " C") == ([2], [ord(" "), ord("C")])   # no BOS: EOS is the prefix token
    tok.bos_token_id = 1
    assert M.encode_pair(tok, "", " C")[0] == [1]


def test_encode_pair_bpe_merge_across_the_boundary():
    from tokenizers import Tokenizer, models, pre_tokenizers, trainers
    from transformers import PreTrainedTokenizerFast
    t = Tokenizer(models.BPE())
    t.pre_tokenizer = pre_tokenizers.Split(" ", "merged_with_next")   # words carry the space in front of them
    trainer = trainers.BpeTrainer(vocab_size=300, special_tokens=["<unk>", "<s>", "</s>"])
    t.train_from_iterator(["the answer is Axe", "Axe Axe answer", "the Axe"] * 50, trainer)
    tok = PreTrainedTokenizerFast(tokenizer_object=t, unk_token="<unk>", bos_token="<s>", eos_token="</s>")
    enc = lambda s: tok.encode(s, add_special_tokens=False)   # noqa: E731
    ctx, cont = M.encode_pair(tok, "the answer is Ax", "e")
    whole = enc("the answer is Axe")
    assert ctx == enc("the answer is Ax") and cont == whole[len(ctx):]
    assert whole != ctx + enc("e")                             # " Axe" is one token across the boundary
    # a context ending in a space: the space goes with the continuation, as the fork does
    ctx, cont = M.encode_pair(tok, "the answer is ", "Axe")
    assert ctx == enc("the answer is") and cont == enc("the answer is Axe")[len(ctx):]


def test_scores_ties_and_out_of_range_gold(caplog):
    s = M.score_doc([-1.0, -0.5, -0.5, -2.0], M.CHOICES, 2)        # exact tie: np.argmax takes the first
    assert s["pred"] == 1 and s["pred_norm"] == 1 and s["acc"] == 0.0 and s["acc_norm"] == 0.0
    s = M.score_doc([-3.0, -3.0, -3.0, -3.0], M.CHOICES, 0)
    assert s["pred"] == 0 and s["acc"] == 1.0
    # acc_norm divides by the choice's length in characters
    s = M.score_doc([-4.0, -3.0], ["long", "x"], 0)
    assert s["pred"] == 1 and s["pred_norm"] == 0 and s["acc_norm"] == 1.0
    assert M.score_doc([0.0, -1.0, -2.0, -3.0], M.CHOICES, "B")["gold"] == 1
    assert M.score_doc([0.0, -1.0, -2.0, -3.0], M.CHOICES, "1")["gold"] == 1
    with caplog.at_level(logging.WARNING):
        s = M.score_doc([0.0, -1.0, -2.0, -3.0], M.CHOICES, 4)
    assert s["gold"] == -100 and s["acc"] == 0.0 and s["acc_norm"] == 0.0 and "not in within range" in caplog.text
    assert M.score_doc([0.0, -1.0, -2.0, -3.0], M.CHOICES, "E")["gold"] == -100


def test_mmlu_micro_average():
    per = {"mmlu_a": [{"acc": 1.0}] * 3, "mmlu_b": [{"acc": 0.0}] * 1}
    assert M.aggregate(per, ("acc",))["acc"] == 0.75          # not the macro mean 0.5


class _ScriptedPacked:
    """Stands in for _Reader._loglikelihood_packed: records each call's windows and targets and returns, per target,
    the log-probability -(token + row / 1000) and a greedy flag when the token is even."""

    def __init__(self):
        self.calls = []

    def __call__(self, windows, targets):
        self.calls.append(([list(w) for w in windows], [list(t) for t in targets]))
        lp = np.array([-(t + r / 1000.0) for ts in targets for r, t in ts], dtype=np.float32)
        return lp, np.array([int(t % 2 == 0) for ts in targets for _, t in ts], dtype=np.int32)


def _host_reader(budget=16384):
    from retrieval_scaling_b200 import reader
    m = object.__new__(reader._Reader)
    m.token_budget = budget
    m._loglikelihood_packed = _ScriptedPacked()
    return m


def test_loglikelihood_windows_truncation_and_grouping():
    m = _host_reader()
    ctx = [5, 6, 7]
    res = m.loglikelihood([(ctx, [10]), (ctx, [12]), (ctx, [14]), (ctx, [11])], max_length=8)
    (windows, targets), = m._loglikelihood_packed.calls
    assert windows == [[5, 6, 7]]                              # four one-token requests, one window
    assert targets == [[(2, 10), (2, 12), (2, 14), (2, 11)]]
    assert [r[1] for r in res] == [True, True, True, False]
    assert res[0][0] == pytest.approx(-10.002) and res[3][0] == pytest.approx(-11.002)

    m = _host_reader()
    long_ctx = list(range(100, 110))
    res = m.loglikelihood([(long_ctx, [1, 2, 4]), ([9], [3]), (long_ctx, [2])], max_length=6)
    (windows, targets), = m._loglikelihood_packed.calls
    # (ctx + cont)[-(max_length + 1):][:-1], longest first
    assert windows == [[106, 107, 108, 109, 1, 2], [104, 105, 106, 107, 108, 109], [9]]
    assert targets[0] == [(3, 1), (4, 2), (5, 4)] and targets[1] == [(5, 2)] and targets[2] == [(0, 3)]
    want0 = -float(np.float32(1.003)) - float(np.float32(2.004)) - float(np.float32(4.005))
    assert res[0] == (pytest.approx(want0, abs=1e-12), False)  # 1 is odd: not greedy
    assert res[1][1] is False and res[2] == (pytest.approx(-float(np.float32(2.005))), True)


def test_loglikelihood_packing_order_and_refusals():
    m = _host_reader(budget=5)
    reqs = [([1], [2]), ([1, 2, 3], [4]), ([7, 8], [9]), ([1, 2, 3], [6])]
    res = m.loglikelihood(reqs, max_length=100)
    calls = m._loglikelihood_packed.calls
    assert [w for c in calls for w in c[0]] == [[1, 2, 3], [7, 8], [1]]   # longest first, packed up to 5 tokens
    assert [len(c[0]) for c in calls] == [2, 1]
    assert [r[1] for r in res] == [True, True, False, True]             # input order
    for bad, what in (([[], [1]], "empty context"), ([[1], []], "empty continuation"),
                      ([[1], [2, 3, 4]], "longer than max_length")):
        with pytest.raises(ValueError, match=what):
            m.loglikelihood([tuple(bad)], max_length=2)


def _cfg(tmp_path, domain, extra=()):
    from retrieval_scaling_b200 import config as C
    return C.load_config("perplexity", os.path.join(ROOT, "ric", "conf"), [
        "datastore.domain=d", f"evaluation.domain={domain}", "evaluation.data.eval_data=x.jsonl",
        "model.lm_model=/none", "tasks.eval.task_name=lm-eval", "tasks.eval.inference=true",
        f"evaluation.lm_eval.predictions_file={tmp_path / 'pred.jsonl'}",
        f"evaluation.results_only_log_file={tmp_path / 'results.log'}", *extra])


class _Reader:
    """Scripted reader: log-likelihood = -(position of the choice letter's distance to the gold letter in the
    context's last character), so the letter named at the end of the context wins."""

    def __init__(self):
        self.calls = []

    def loglikelihood(self, requests, max_length):
        self.calls.append((requests, max_length))
        return [(-abs(cont[-1] - ctx[-1]) * 1.0, False) for ctx, cont in requests]


def _run(tmp_path, monkeypatch, cfg):
    sys.path.insert(0, os.path.join(ROOT, "ric"))
    import main_ric
    from retrieval_scaling_b200 import perplexity as P
    from retrieval_scaling_b200 import reader as RD
    rd = _Reader()
    monkeypatch.setattr(RD, "load_reader", lambda *a, **k: rd)
    monkeypatch.setattr(P, "load_lm_tokenizer", lambda name: _Tok())
    monkeypatch.setattr(R, "read_model_config", lambda name: {"max_position_embeddings": 64})
    main_ric.main(cfg)
    return rd, [json.loads(line) for line in open(tmp_path / "pred.jsonl")], open(tmp_path / "results.log").read()


def test_main_ric_dispatch_medqa_without_retrieval(tmp_path, monkeypatch):
    """concate_k = 0 opens no retrieval file (the configured one does not exist); acc and acc_norm are logged."""
    p = tmp_path / f"samples_medqa_4options_{DATE}.json"
    # contexts end in the letter the scripted reader favours: B, D, A (gold 1, 3, 2)
    _write_samples(p, [_sample(0, "shot\n\nQ one B", 1), _sample(1, "shot\n\nQ two D", 3), _sample(2, "shot\n\nQ A", 2)])
    cfg = _cfg(tmp_path, "medqa_4options", [f"evaluation.lm_eval.samples_file={p}", "evaluation.concate_k=0",
                                            f"evaluation.lm_eval.retrieval_file={tmp_path / 'missing.jsonl'}"])
    rd, preds, log = _run(tmp_path, monkeypatch, cfg)
    (reqs, max_len), = rd.calls
    assert max_len == 64 and len(reqs) == 12
    assert reqs[0] == ([ord(c) for c in "shot\n\nQ one B"], [ord(" "), ord("A")])
    assert [p["pred"] for p in preds] == [1, 3, 0] and [p["acc"] for p in preds] == [1.0, 1.0, 0.0]
    assert all("acc_norm" in p and p["task"] == "medqa_4options" for p in preds)
    assert preds[0]["prompt_tokens"] == len("shot\n\nQ one B") and len(preds[0]["loglikelihoods"]) == 4
    assert "Domain = medqa_4options" in log and "n = 3" in log and "acc = 0.6667" in log and "acc_norm = 0.6667" in log


def _mmlu(tmp_path):
    sd = tmp_path / "samples"
    sd.mkdir()
    _write_samples(sd / f"samples_mmlu_anatomy_{DATE}.json", [_sample(0, "shots\n\nQ1 A", 0), _sample(1, "shots\n\nQ2 C", 1)])
    _write_samples(sd / f"samples_mmlu_virology_{DATE}.json", [_sample(0, "shots\n\nQ3 D", 3)])
    return sd


def _retrieved(path, questions, tag):
    with open(path, "w") as f:
        for q in questions:
            f.write(json.dumps({"query": q, "ctxs": [{"retrieval text": f"<{tag}{q[-1]}>"}]}) + "\n")


def test_main_ric_dispatch_mmlu_group_with_retrieval_dir(tmp_path, monkeypatch):
    """retrieval_dir wins over retrieval_file; the group's acc is the mean over all three questions."""
    sd = _mmlu(tmp_path)
    rdir = tmp_path / "ret"
    rdir.mkdir()
    _retrieved(rdir / "mmlu_anatomy_retrieved_results.jsonl", ["Q1 A", "Q2 C"], "dir")
    _retrieved(rdir / "mmlu_virology_retrieved_results.jsonl", ["Q3 D"], "dir")
    _retrieved(tmp_path / "file.jsonl", ["Q1 A", "Q2 C", "Q3 D"], "file")
    cfg = _cfg(tmp_path, "mmlu", [f"evaluation.lm_eval.samples_dir={sd}", "evaluation.concate_k=1",
                                  f"evaluation.lm_eval.retrieval_dir={rdir}",
                                  f"evaluation.lm_eval.retrieval_file={tmp_path / 'file.jsonl'}"])
    rd, preds, log = _run(tmp_path, monkeypatch, cfg)
    (reqs, _), = rd.calls
    assert reqs[0][0] == [ord(c) for c in "<dirA>shots\n\nQ1 A"]
    assert [(p["task"], p["pred"], p["gold"]) for p in preds] == [("mmlu_anatomy", 0, 0), ("mmlu_anatomy", 2, 1),
                                                                  ("mmlu_virology", 3, 3)]
    assert all("acc_norm" not in p for p in preds)
    assert "Domain = mmlu" in log and "n = 3" in log and "acc = 0.6667" in log


def test_main_ric_dispatch_mmlu_subject_with_retrieval_file_and_missing_question(tmp_path, monkeypatch):
    sd = _mmlu(tmp_path)
    _retrieved(tmp_path / "file.jsonl", ["Q1 A", "Q2 C"], "file")
    cfg = _cfg(tmp_path, "mmlu_anatomy", [f"evaluation.lm_eval.samples_dir={sd}", "evaluation.concate_k=1",
                                          f"evaluation.lm_eval.retrieval_file={tmp_path / 'file.jsonl'}"])
    rd, preds, log = _run(tmp_path, monkeypatch, cfg)
    assert rd.calls[0][0][4][0] == [ord(c) for c in "<fileC>shots\n\nQ2 C"]
    assert len(preds) == 2 and "Domain = mmlu_anatomy" in log and "acc = 0.5000" in log
    cfg = _cfg(tmp_path, "mmlu_virology", [f"evaluation.lm_eval.samples_dir={sd}", "evaluation.concate_k=1",
                                           f"evaluation.lm_eval.retrieval_file={tmp_path / 'file.jsonl'}"])
    with pytest.raises(RuntimeError, match="no row"):
        _run(tmp_path, monkeypatch, cfg)


def test_mc_refusals(tmp_path, monkeypatch):
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(NotImplementedError, match="one process"):
        R.evaluate_lm_eval(_cfg(tmp_path, "mmlu"))
    monkeypatch.setenv("WORLD_SIZE", "1")
    with pytest.raises(ValueError, match="samples_dir"):
        R.evaluate_lm_eval(_cfg(tmp_path, "mmlu"))
    with pytest.raises(ValueError, match="samples_file"):
        R.evaluate_lm_eval(_cfg(tmp_path, "medqa_4options"))
    with pytest.raises(NotImplementedError, match="mmlu"):
        R.domain_settings("mmlu")
    assert not M.is_mc_task("mmlu_") and not M.is_mc_task("squad") and M.is_mc_task("mmlu_anatomy")


@pytest.mark.parametrize("k", [0, 1, 2, 6, 7, 9, 10, 11])
def test_loglikelihood_abi_is_bound_and_refuses_null_pointers(k):
    """rsb_llm_loglikelihood is bound and exported; a null handle, batch, target, output or workspace pointer is
    RSB_ERR_INVALID before any device access (the other pointers are never read)."""
    import ctypes

    from retrieval_scaling_b200 import _lib
    L = _lib.lib()
    assert {"rsb_llm_loglikelihood", "rsb_llm_loglikelihood_workspace_bytes"} <= {n for n, _, _ in _lib.SIGNATURES}
    P = ctypes.c_void_p(16)
    args = [P, P, P, 1, 4, 4, P, P, 2, P, P, P, 1 << 20, None]
    args[k] = None
    assert L.rsb_llm_loglikelihood(*args) == _lib.RSB_ERR_INVALID
    assert b"null" in L.rsb_llm_last_error()
    assert L.rsb_llm_loglikelihood_workspace_bytes(None, 4, 2) == 0
