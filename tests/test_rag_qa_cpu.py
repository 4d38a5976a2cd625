"""CPU checks of the retrieval-augmented QA task (`rag_qa.py`): the lm-eval fork's retrieval context, stop-term cutting,
whitespace filter, exact_match restated from its published definition, truncation, refusals, and `main_ric`
dispatch with a reader whose `generate` is scripted."""
import json
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

from retrieval_scaling_b200 import rag_qa as R  # noqa: E402

NQ = R.DOMAINS["nq_open"]
TQA = R.DOMAINS["triviaqa"]


def test_retrieval_context_order_separator_fallback_and_duplicates():
    rows = [
        {"raw_query": "Answer these questions:\n\nQ: who?\nA:", "query": "ignored",
         "ctxs": [{"retrieval text": "first. "}, {"retrieval text": "second. ", "text": "not this"}, {"text": "third. "}]},
        {"query": "shot\n\nQ: short?\nA:", "ctxs": [{"retrieval text": "only"}]},
        {"query": "Q: none?\nA:"},
        {"query": "Q: dup?\nA:", "ctxs": [{"text": "old"}]},
        {"query": "other shots\n\nQ: dup?\nA:", "ctxs": [{"text": "new"}]},
    ]
    h = R.hash_retrieval_results(rows, 3)
    assert h["Q: who?\nA:"] == "third. second. first. "      # most relevant last, no separator, 'text' fallback
    assert h["Q: short?\nA:"] == "only"                        # fewer passages than concat_k
    assert h["Q: none?\nA:"] == ""
    assert h["Q: dup?\nA:"] == "new"                           # a later duplicate row wins
    assert R.hash_retrieval_results(rows, 1)["Q: who?\nA:"] == "first. "
    assert R.hash_retrieval_results(rows, 0)["Q: who?\nA:"] == ""


def test_retrieval_context_skips_passages_without_text_and_keys_question_rows():
    """A passage with neither key is skipped and the next one used, as the fork's bare try / except does; rows with
    only 'question' are keyed by the task's description + doc_to_text."""
    rows = [{"query": "Q: x?\nA:", "ctxs": [{"retrieval text": "a"}, {"title": "no text"}, {"text": "c"}]},
            {"question": "who wrote it", "ctxs": [{"text": "p"}]}]
    h = R.hash_retrieval_results(rows, 3, "nq_open")
    assert h["Q: x?\nA:"] == "ca" and h["Q: who wrote it?\nA:"] == "p"
    assert R.hash_retrieval_results(rows[1:], 1, "triviaqa") == {"Question: who wrote it?\nAnswer:": "p"}
    with pytest.raises(NotImplementedError, match="question"):
        R.hash_retrieval_results(rows[1:], 1, None)


def test_prompts_prepend_the_context_to_the_whole_few_shot_prompt():
    hashed = {"Q: b?\nA:": "CTX "}
    rows = [{"query": "desc\n\nQ: a?\nA: x\n\nQ: b?\nA:", "answer": ["y"]}]
    assert R.build_prompts(rows, hashed) == ["CTX desc\n\nQ: a?\nA: x\n\nQ: b?\nA:"]
    # the fork's system-prompt branch builds on the prompt that already holds the context
    assert R.build_prompts(rows, hashed, "SYS ") == ["CTX \n\nSYS CTX desc\n\nQ: a?\nA: x\n\nQ: b?\nA:"]
    with pytest.raises(RuntimeError, match="no row"):
        R.build_prompts([{"query": "Q: missing?\nA:", "answer": []}], hashed)


@pytest.mark.parametrize("raw, want", [
    (" Paris", "Paris"),
    ("\nParis.", "Paris"),                   # empty first piece: the piece after the term
    (" Paris, France.", "Paris"),
    (" Paris\nLondon", "Paris"),
    ("\n\nParis", ""),                       # the piece after the first "\n" is empty too
    (".", ""),
    (" 3.5 million", "3"),
    ("  two spaces", " two spaces"),         # remove_whitespace drops exactly one space
    (" George Washington</s>x", "George Washington"),
    ("</s>Paris", "Paris"),
    ("", ""),
])
def test_stop_terms_and_whitespace(raw, want):
    assert R.remove_whitespace(R.cut_at_stop_terms(raw, R.UNTIL + ["</s>"])) == want


@pytest.mark.parametrize("pred, gold, settings, want", [
    ("The Beatles", "Beatles", NQ, 1.0),         # article removed by the regex
    ("the beatles", "The Beatles", NQ, 1.0),
    ("an apple", "apple", NQ, 1.0),
    ("The Beatles", "Beatles", TQA, 0.0),        # triviaqa keeps articles
    ("U.S.A.", "usa", TQA, 1.0),                 # punctuation and case
    ("Paris!", "paris", NQ, 1.0),
    ("Theodore", "odore", NQ, 0.0),              # \b: "The" inside a word is not an article
    ("1,000", "1000", NQ, 1.0),
    ("Paris ", "Paris", NQ, 0.0),                # whitespace is not stripped
    ("", "", NQ, 1.0),
])
def test_exact_match_hand_worked(pred, gold, settings, want):
    assert R.exact_match(pred, gold, **settings) == want


def test_multi_target_scores():
    assert R.score("Beatles", ["The Rolling Stones", "the Beatles"], NQ) == 1.0
    assert R.score("Stones", ["The Rolling Stones", "the Beatles"], NQ) == 0.0
    assert R.score("paris", "Paris", NQ) == 1.0
    tqa = {"aliases": ["J. F. K.", "Kennedy"], "value": "John F. Kennedy", "normalized_value": "john f kennedy"}
    assert R.score("JFK", tqa, TQA) == 0.0       # "J. F. K." becomes "j f k": the spaces stay
    assert R.score("J F K", tqa, TQA) == 1.0
    assert R.score("kennedy", tqa, TQA) == 1.0
    assert R.score("john f kennedy", tqa, TQA) == 0.0   # only the aliases are targets


class _Tok:
    model_max_length = R.HF_UNSET_MAX_LENGTH
    eos_token_id = 2

    def encode(self, s, add_special_tokens=True):
        assert add_special_tokens is False
        return [ord(c) for c in s]

    def decode(self, ids, skip_special_tokens=True):
        return "".join("</s>" if i == 2 else chr(i) for i in ids if not (skip_special_tokens and i == 2))


def test_truncation_and_max_length():
    tok = _Tok()
    assert R.max_length({"max_position_embeddings": 4096}, tok) == 4096
    assert R.max_length({"n_positions": 1024, "max_position_embeddings": 4096}, tok) == 1024
    assert R.max_length({}, tok) == 2048
    tok.model_max_length = 512
    assert R.max_length({}, tok) == 512
    assert R.encode_prompt(tok, "abcdef", 4) == [ord(c) for c in "cdef"]   # left truncation
    assert R.encode_prompt(tok, "ab", 4) == [ord("a"), ord("b")]
    with pytest.raises(ValueError, match="no room"):
        R.encode_prompt(tok, "ab", 0)


def test_refusals_and_eos_ids():
    with pytest.raises(NotImplementedError, match="mmlu"):
        R.domain_settings("mmlu")
    assert R.eos_token_ids({"eos_token_id": [5, 6]}, _Tok()) == [5, 6]
    assert R.eos_token_ids({"eos_token_id": 7}, _Tok()) == [7]
    assert R.eos_token_ids({}, _Tok()) == [2]


def _cfg(tmp_path, domain="nq_open", extra=()):
    from retrieval_scaling_b200 import config as C
    return C.load_config("perplexity", os.path.join(ROOT, "ric", "conf"), [
        "datastore.domain=d", f"evaluation.domain={domain}", "evaluation.data.eval_data=x.jsonl",
        "model.lm_model=/none", "tasks.eval.task_name=lm-eval", "evaluation.concate_k=2",
        f"evaluation.lm_eval.prompts_file={tmp_path / 'prompts.jsonl'}",
        f"evaluation.lm_eval.retrieval_file={tmp_path / 'retrieved.jsonl'}",
        f"evaluation.lm_eval.predictions_file={tmp_path / 'pred.jsonl'}",
        f"evaluation.results_only_log_file={tmp_path / 'results.log'}", "evaluation.lm_eval.max_gen_toks=8", *extra])


def _write(tmp_path):
    prompts = [{"query": "Answer these questions:\n\nQ: a?\nA: x\n\nQ: capital?\nA:", "answer": ["Paris"]},
               {"query": "Answer these questions:\n\nQ: a?\nA: x\n\nQ: band?\nA:", "answer": ["The Beatles", "Beatles"]},
               {"query": "Answer these questions:\n\nQ: a?\nA: x\n\nQ: none?\nA:", "answer": "no"}]
    with open(tmp_path / "prompts.jsonl", "w") as f:
        for p in prompts:
            f.write(json.dumps(p) + "\n")
    with open(tmp_path / "retrieved.jsonl", "w") as f:
        for q in ("capital", "band", "none"):
            f.write(json.dumps({"raw_query": f"Q: {q}?\nA:", "ctxs": [{"retrieval text": f"<{q}1>"},
                                                                       {"retrieval text": f"<{q}2>"}]}) + "\n")
    return prompts


def test_main_ric_dispatch_with_a_scripted_reader(tmp_path, monkeypatch):
    """`tasks.eval.inference` with task_name lm-eval runs rag_qa: prompt ids truncated to max_length - max_gen_toks,
    the config's EOS ids, the fork's post-processing, the score and both outputs."""
    sys.path.insert(0, os.path.join(ROOT, "ric"))
    import main_ric
    from retrieval_scaling_b200 import perplexity as P
    from retrieval_scaling_b200 import reader as RD
    prompts = _write(tmp_path)
    conts = [[ord(c) for c in " Paris, France"], [ord(c) for c in "\nthe Beatles."] + [2], [ord(c) for c in " yes"]]
    calls = []

    class Reader:
        def generate(self, ids, max_new, eos):
            calls.append((ids, max_new, eos))
            return conts

    monkeypatch.setattr(RD, "load_reader", lambda *a, **k: Reader())
    monkeypatch.setattr(P, "load_lm_tokenizer", lambda name: _Tok())
    monkeypatch.setattr(R, "read_model_config", lambda name: {"max_position_embeddings": 40, "eos_token_id": [2, 3]})
    cfg = _cfg(tmp_path, extra=["tasks.eval.inference=true"])
    main_ric.main(cfg)
    (ids, max_new, eos), = calls
    assert max_new == 8 and eos == [2, 3]
    want = ["<capital2><capital1>" + prompts[0]["query"], "<band2><band1>" + prompts[1]["query"]]
    assert ids[0] == [ord(c) for c in want[0]][-32:] and ids[1] == [ord(c) for c in want[1]][-32:]
    preds = [json.loads(line) for line in open(tmp_path / "pred.jsonl")]
    assert [p["prediction"] for p in preds] == ["Paris", "the Beatles", "yes"]
    assert [p["exact_match"] for p in preds] == [1.0, 1.0, 0.0]
    assert preds[1]["generation"] == "\nthe Beatles." and all(p["prompt_tokens"] == 32 for p in preds)
    log = open(tmp_path / "results.log").read()
    assert "Domain = nq_open" in log and "concate_k = 2" in log and "n = 3" in log and "exact_match = 0.6667" in log


def test_evaluate_perplexity_still_refuses_lm_eval_and_torchrun_is_refused(tmp_path, monkeypatch):
    _write(tmp_path)
    from retrieval_scaling_b200 import perplexity as P
    with pytest.raises(NotImplementedError, match="lm-eval"):
        P.evaluate_perplexity(_cfg(tmp_path))
    monkeypatch.setenv("WORLD_SIZE", "2")
    with pytest.raises(NotImplementedError, match="one process"):
        R.evaluate_lm_eval(_cfg(tmp_path))
    monkeypatch.setenv("WORLD_SIZE", "1")
    with pytest.raises(NotImplementedError, match="'squad'"):
        R.evaluate_lm_eval(_cfg(tmp_path, domain="squad"))
