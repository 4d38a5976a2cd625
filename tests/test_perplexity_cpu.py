"""CPU checks of the perplexity task's host code (retrieval_scaling_b200.perplexity) against restatements of the
reference's functions written here in their original loop form: windows, prompts, extract_answer, both
decontamination modes, the reader inputs and the averaging, with the reference's quirks."""
import math
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import llama_fixture as F  # noqa: E402

from retrieval_scaling_b200 import perplexity as P  # noqa: E402


# ---- restatements in the reference's loop form (src/data.py:375-436, src/decontamination.py) ------------------------
def ref_batch_merged(flat, L, stride, pad):
    xs, ys, prev = [], [], 0
    for b in range(0, len(flat) - 1, stride):
        e = min(b + L, len(flat) - 1)
        k = e - prev
        x, y = flat[b:e].copy(), flat[b + 1:e + 1].copy()
        y[:-k] = pad
        if e == len(flat) - 1 and len(x) == len(y) < L:
            x = np.concatenate([x, np.full(L - len(x), pad)])
            y = np.concatenate([y, np.full(L - len(y), pad)])
        xs.append(x)
        ys.append(y)
        prev = e
        if e == len(flat) - 1:
            break
    return np.stack(xs), np.stack(ys)


def ref_overlap(a, b):
    best = 0
    for i in range(len(a)):
        for j in range(len(b)):
            if a[i] == b[j]:
                n = 0
                while i + n < len(a) and j + n < len(b) and a[i + n] == b[j + n]:
                    n += 1
                best = max(best, n)
    return best


@pytest.mark.parametrize("n, L, stride", [(50, 16, 8), (17, 16, 8), (100, 32, 32), (33, 8, 3), (200, 64, 16), (9, 16, 4)])
def test_batch_merged_matches_the_loop_form(n, L, stride):
    flat = np.random.default_rng(n).integers(3, 1000, n)
    x, y = P.batch_merged(flat, L, stride, 2)
    rx, ry = ref_batch_merged(flat, L, stride, 2)
    assert np.array_equal(x, rx) and np.array_equal(y, ry)
    # every target token after the first is scored exactly once over the windows
    assert sorted(y[y != 2].tolist()) == sorted(flat[1:][flat[1:] != 2].tolist())


def test_prepare_ppl_eval_data_merge_split_and_sampling():
    tok = F.tokenizer()
    rng = np.random.default_rng(0)
    data = [{"text": " ".join(f"w{i}" for i in rng.integers(3, 1000, n))} for n in (40, 7, 90)]
    for merge in (True, False):
        out = P.prepare_ppl_eval_data(data, tok, 32, 16, merge)
        ids = [tok(ex["text"])["input_ids"] for ex in data]
        if merge:
            X, Y = ref_batch_merged(np.array([t for x in ids for t in x]), 32, 16, 2)
        else:
            parts = [ref_batch_merged(np.array(x), 32, 16, 2) for x in ids]
            X, Y = np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
        assert len(out) == len(X)
        for ex, x, y in zip(out, X, Y):
            assert ex["raw_inputs"] == tok.decode(x.tolist(), skip_special_tokens=True)
            assert ex["raw_query"] == tok.decode([int(a) for a, b in zip(x, y) if b == 2], skip_special_tokens=True)
    full = P.prepare_ppl_eval_data(data, tok, 32, 16, True)
    np.random.seed(310)
    order = np.random.permutation(len(full))[:3]
    assert P.prepare_ppl_eval_data(data, tok, 32, 16, True, num_eval_samples=3, seed=310) == [full[i] for i in order]


def test_decontamination_both_modes():
    rng = np.random.default_rng(1)
    for _ in range(40):
        a = [f"w{i}" for i in rng.integers(0, 6, rng.integers(0, 30))]
        b = [f"w{i}" for i in rng.integers(0, 6, rng.integers(1, 30))]
        assert P.longest_common_run(a, b) == ref_overlap(a, b)
        doc, gold = " ".join(a), " ".join(b)
        run = ref_overlap(doc.split(" "), gold.split(" "))
        assert P.check_below_lexical_overlap_threshold(doc, gold, 0.5, "longest") == (run < int(len(b) * 0.5))
        assert P.check_below_lexical_overlap_threshold(doc, gold, 4, "longest") == (run < 4)
        assert P.check_below_lexical_overlap_threshold(doc, gold, 1, "longest") is True
    words = [f"w{i}" for i in range(40)]
    g = " ".join(words[:30])
    assert P.check_below_lexical_overlap_threshold(" ".join(words[:29]), g, 0.8, "jaccard") is False   # 17/18 grams shared
    assert P.check_below_lexical_overlap_threshold(" ".join(words[20:]), g, 0.8, "jaccard") is True
    assert P.check_below_lexical_overlap_threshold("a b", "c d", 0.5, "jaccard") is True               # no grams: 0
    with pytest.raises(ValueError):
        P.check_below_lexical_overlap_threshold("a", "b", 32, "jaccard")


def test_extract_answer():
    assert P.extract_answer("q1 q2 a1 a2<|endoftext|>", "q1 q2") == " a1 a2"
    assert P.extract_answer("a b a b", "a") == " b  b"             # every occurrence goes
    assert P.extract_answer("x y", "") == "x y"


class _Args(dict):
    def get(self, k, d=None):
        return dict.get(self, k, d)


def test_build_doc_prompts_quirks():
    ctx = lambda *t: [{"retrieval text": s, "retrieval next text": s + "+"} for s in t]   # noqa: E731
    data = [{"raw_inputs": "skipped", "raw_query": "", "ctxs": ctx("z")},
            {"raw_inputs": "q a b", "raw_query": "q", "ctxs": ctx("d1", "d2", "d3")},
            {"raw_inputs": "q2 c", "raw_query": "q2", "ctxs": ctx("e1")},
            {"raw_inputs": "q3 c", "raw_query": "q3", "ctxs": []}]
    c, a, n = P.build_doc_prompts(data, _Args(concate_k=2))
    assert a == [" a b", " c", " c"]                               # eval_data[1:]: the first example is skipped
    assert c == ["d2 \nd1 \nq", "e1 \nq2", "q3"]                   # most relevant nearest the query; empty ctxs: nothing
    assert n == 0                                                  # reset per example: the last one (no ctxs) is not counted
    c, a, n = P.build_doc_prompts(data[:3], _Args(concate_k=2))
    assert n == 1                                                  # the last example had one document of two
    c, _, _ = P.build_doc_prompts(data[:2], _Args(concate_k=2, use_continuation=True))
    assert c == ["d2+ \nd1+ \nq"]
    blocked = [data[0], {"raw_inputs": "q a b c d", "raw_query": "q", "ctxs": ctx("a b c", "x", "y z")}]
    c, _, _ = P.build_doc_prompts(blocked, _Args(concate_k=2, decontamination=True, contamination_threshold=2,
                                                 decontamination_method="longest"))
    assert c == ["y z \nx \nq"]                                    # "a b c" shares 3 >= 2 words with the answer
    c, _, n = P.build_doc_prompts(data, _Args(concate_k=0))
    assert c == ["q", "q2", "q3"] and n == 0


def test_reader_inputs_bos_pad_and_left_truncation():
    tok = F.tokenizer()
    ids, lab = P.reader_inputs(tok, "w5 w6", "w7 </s> w8", 100, 2)
    assert ids == [1, 5, 6, 1, 7, 2, 8]                            # BOS on the context and on the answer
    assert lab == [-100, -100, -100, 1, 7, -100, 8]                # the answer's BOS is a label; eos is masked
    ids, lab = P.reader_inputs(tok, "w5 w6", "w7 w8", 4, 2)
    assert ids == [6, 1, 7, 8] and lab == [-100, 1, 7, 8]


def test_hf_loss_without_labels_is_nan_and_the_average_keeps_it():
    cfg = dict(F.CONFIG, num_hidden_layers=1, max_position_embeddings=64)
    model = F.hf_model(cfg, seed=2)
    x = torch.tensor([[1, 5, 6, 7]])
    with torch.no_grad():
        assert math.isnan(float(model(x, labels=torch.full_like(x, -100)).loss))
        assert math.isnan(float(model(x[:, :1], labels=x[:, :1]).loss))
    out = P.summarize({}, [1.0, 2.0], 0)
    assert out.average_loss == 1.5 and out.perplexity.dtype == torch.float32
    assert float(out.perplexity) == float(torch.exp(torch.tensor(1.5)))
    assert float(out.bit_per_byte) == pytest.approx(math.log2(math.exp(1.5)) / 8, rel=1e-6)
    assert math.isnan(P.summarize({}, [1.0, float("nan")], 0).average_loss)


def test_other_inference_tasks_are_refused():
    from retrieval_scaling_b200 import config as C
    base = ["datastore.domain=d", "evaluation.domain=d", "evaluation.data.eval_data=x.jsonl", "model.lm_model=/none"]
    for task, what in (("perplexity_calibration", "perplexity_calibration"), ("lm-eval", "lm-eval")):
        cfg = C.load_config("perplexity", os.path.join(ROOT, "ric", "conf"), base + [f"tasks.eval.task_name={task}"])
        with pytest.raises(NotImplementedError, match=what):
            P.evaluate_perplexity(cfg)


def test_evaluate_perplexity_follows_the_reference_loop(tmp_path):
    """concate_k 0 through load_eval_data and the reader directory's tokenizer, with a model whose `loss` is HF's
    fp32 `lm(ids, labels=labels).loss` per window, against the reference's loop restated here."""
    import json

    from retrieval_scaling_b200 import config as C
    d = F.build_dir(str(tmp_path / "reader"), dict(num_hidden_layers=1, max_position_embeddings=40), seed=4)
    rng = np.random.default_rng(2)
    eval_path = tmp_path / "eval.jsonl"
    with open(eval_path, "w") as f:
        for n in (60, 30):
            f.write(json.dumps({"text": " ".join(f"w{i}" for i in rng.integers(2, 1000, n))}) + "\n")
    cfg = C.load_config("perplexity", os.path.join(ROOT, "ric", "conf"),
                        ["datastore.domain=d", "evaluation.domain=d", f"evaluation.data.eval_data={eval_path}",
                         f"model.lm_model={d}", "evaluation.data.max_eval_data_seq_length=24",
                         "evaluation.data.eval_stride=12"])
    hf = F.hf_model(dict(num_hidden_layers=1, max_position_embeddings=40), seed=4)

    class HFReader:
        max_position_embeddings = 40

        def loss(self, ids, labels):
            with torch.no_grad():
                return [float(hf(torch.tensor([i]), labels=torch.tensor([lb])).loss) for i, lb in zip(ids, labels)]

    out = P.evaluate_perplexity(cfg, model=HFReader())
    tok = F.tokenizer()
    data = P.prepare_ppl_eval_data([json.loads(line) for line in open(eval_path)], tok, 24, 12, True)
    total, count = 0.0, 0
    for ex in data[1:]:
        answer = ex["raw_inputs"].replace(ex["raw_query"], "")
        a = tok(answer, return_tensors="pt")["input_ids"]
        c = tok(ex["raw_query"], return_tensors="pt")["input_ids"]
        ids = torch.cat((c, a), 1)
        lab = torch.cat((torch.full(c.size(), -100), a), 1)
        lab = torch.where(lab == 2, torch.tensor(-100), lab)
        with torch.no_grad():
            total += hf(ids[:, -40:], labels=lab[:, -40:]).loss.item()
        count += 1
    assert out.average_loss == pytest.approx(total / count, rel=1e-12)
    assert "perplexity = " in out.log_message()
