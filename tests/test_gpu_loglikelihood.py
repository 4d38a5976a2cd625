"""GPU checks of multiple-choice scoring (`rsb_llm_loglikelihood`, `_Reader.loglikelihood`, `rag_mc`) on the seeded
reader fixtures (Llama GQA 4:1, GPT-NeoX, OLMo and OLMo-2, fp16 and bf16):

  against nll     every target's log-probability is bit for bit -rsb_llm_nll of the same (row, token), computed on the
                  window cut after that row with the token as its last label; the prefill, norms and LM-head GEMM are
                  per row, so the cut changes nothing
  greedy          the flag equals "token == the id rsb_llm_generate chooses after the same prefix"
  layouts         4 and 1 000 targets on one row, duplicates, shuffled order, rows 0 and last, 1-token windows, and more
                  distinct rows than chunk_rows() on the chunked LM head of test_gpu_generate's batch-invariance case
  oracle          logits made exact by construction (all-ones final LayerNorm output, one non-zero per LM-head row)
                  against oracle/loglik_oracle.py's fp64 value, within its fp32 bound
  refusals        outputs pre-filled with NaN stay untouched
  transformers    reader.loglikelihood against a CPU fp32 restatement of the fork's _loglikelihood_tokens
  end to end      main_ric with medqa_4options and a two-subject mmlu group against the same restatement"""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, ROOT)

import llama_fixture as LF  # noqa: E402
import neox_fixture as NF  # noqa: E402
import olmo_fixture as OF  # noqa: E402

from oracle import loglik_oracle as LO  # noqa: E402

pytestmark = pytest.mark.gpu

CASES = {
    "llama-gqa4": ("B200Llama", LF, LF.CONFIG),
    "neox-d128": ("B200NeoX", NF, dict(NF.CONFIG, num_attention_heads=4)),
    "olmo": ("B200Olmo", OF, OF.CONFIGS["olmo"]),
    "olmo2": ("B200Olmo", OF, OF.CONFIGS["olmo2"]),
}
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
DELTA = {"fp16": 0.05, "bf16": 0.3}              # test_gpu_generate.py's near-tie margin: several times the logit error
# |log-likelihood - transformers fp32| per scored token: in fp16 test_gpu_generate.py's LP_TOL.  In bf16 its LP_TOL
# (0.1) bounds decode against prefill, two computations rounded to bf16 alike; against fp32 the bf16 logit error itself
# enters, so the bound is DELTA's
LL_TOL = {"fp16": 2e-2, "bf16": DELTA["bf16"]}
# a one-layer Llama whose LM head runs in 128-row chunks (test_gpu_generate.py's CHUNKED_HEAD)
CHUNKED_HEAD = dict(hidden_size=128, num_attention_heads=1, num_key_value_heads=1, intermediate_size=128,
                    num_hidden_layers=1, vocab_size=(1 << 20) - 99)


def _reader(name, dtype, load=True, sd=None, **change):
    from retrieval_scaling_b200 import reader
    cls, FX, base = CASES[name]
    cfg = dict(base, **change)
    sd = FX.seeded_state_dict(cfg) if sd is None else sd
    m = getattr(reader, cls)(cfg, dtype=DTYPES[dtype])
    if load:
        m.load_state_dict(sd)
    return m, cfg, sd


def _call(m, windows, rows, toks, short=0):
    """rsb_llm_loglikelihood on packed windows: (rc, logprob, greedy) with the outputs pre-filled with NaN / 7."""
    lens = [len(w) for w in windows]
    cu = [0] + np.cumsum(lens).tolist()
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device="cuda")   # noqa: E731
    ids, d_cu, d_row, d_tok = i32([v for w in windows for v in w]), i32(cu), i32(rows), i32(toks)
    lp = torch.full((len(rows),), float("nan"), device="cuda")
    gr = torch.full((len(rows),), 7, dtype=torch.int32, device="cuda")
    need = m.L.rsb_llm_loglikelihood_workspace_bytes(m._h, cu[-1], len(rows))
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())   # noqa: E731
    rc = m.L.rsb_llm_loglikelihood(m._h, p(ids), p(d_cu), len(lens), cu[-1], max(lens), p(d_row), p(d_tok), len(rows),
                                   p(lp), p(gr), p(ws), need - short,
                                   ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return rc, lp.cpu(), gr.cpu()


def _check_targets(m, windows, targets):
    """targets: (window, row, token).  Bit-equality with -nll and greedy against generate, per target."""
    cu = [0] + np.cumsum([len(w) for w in windows]).tolist()
    rows = [cu[w] + r for w, r, _ in targets]
    toks = [t for _, _, t in targets]
    rc, lp, gr = _call(m, windows, rows, toks)
    assert rc == 0, m.L.rsb_llm_last_error()
    cut = [windows[w][:r + 1] + [t] for w, r, t in targets]
    nll = m.nll(cut, [[-100] * (len(c) - 1) + [c[-1]] for c in cut])
    want = torch.stack([-n[-1] for n in nll])
    diff = (lp - want).abs()
    assert torch.equal(lp, want), f"{int((diff > 0).sum())} of {len(rows)} differ, max {float(diff.max()):.3e}"
    prefixes = sorted({(w, r) for w, r, _ in targets})
    chosen = dict(zip(prefixes, (t[0] for t in m.generate([windows[w][:r + 1] for w, r in prefixes], 1, []))))
    want_g = torch.tensor([int(t == chosen[(w, r)]) for w, r, t in targets], dtype=torch.int32)
    assert torch.equal(gr, want_g)
    return lp, gr


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("name", list(CASES))
def test_against_nll_and_greedy(name, dtype):
    m, cfg, _ = _reader(name, dtype)
    V = cfg["vocab_size"]
    rng = np.random.default_rng(3)
    windows = [rng.integers(0, V, n).tolist() for n in (1, 5, 64, 130, 1)]
    # the tokens each prefix's generate chooses, so some flags are 1
    pre = [(0, 0), (1, 4), (2, 63), (3, 0), (3, 129), (4, 0)]
    chosen = [t[0] for t in m.generate([windows[w][:r + 1] for w, r in pre], 1, [])]
    targets = [(w, r, t) for (w, r), t in zip(pre, chosen)]
    targets += [(2, 17, int(t)) for t in rng.integers(0, V, 4)]              # 4 on one row
    targets += [(3, 65, int(t)) for t in rng.integers(0, V, 1000)]           # 1 000 on one row, duplicates among them
    targets += [(1, 2, 9), (1, 2, 9), (0, 0, V - 1), (4, 0, 0), (3, 129, chosen[4])]   # repeats, first and last ids
    order = rng.permutation(len(targets))
    targets = [targets[i] for i in order]
    lp, gr = _check_targets(m, windows, targets)
    print(f"{name} {dtype}: {len(targets)} targets bit-equal to -nll, {int(gr.sum())} greedy")
    assert int(gr.sum()) >= len(pre) and bool((lp <= 0).all())


def test_more_rows_than_one_head_chunk():
    m, cfg, _ = _reader("llama-gqa4", "fp16", **CHUNKED_HEAD)
    rng = np.random.default_rng(4)
    windows = [rng.integers(0, cfg["vocab_size"], n).tolist() for n in (120, 200)]
    targets = [(w, r, int(rng.integers(0, cfg["vocab_size"]))) for w in range(2) for r in range(len(windows[w]))]
    targets = [targets[i] for i in rng.permutation(len(targets))]
    _check_targets(m, windows, targets)          # 320 distinct rows: three 128-row chunks


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_exact_logits_against_the_fp64_oracle(dtype):
    """Final LayerNorm weight 0 and bias 1 make every normed row all ones; each embed_out row has one non-zero, so
    each logit is that value exactly, whatever the GEMM's order.  Ties at the top, two near-maximal ids, -8 .. 8."""
    cfg = dict(NF.CONFIG, num_attention_heads=4)
    sd = NF.seeded_state_dict(cfg)
    V, H = cfg["vocab_size"], cfg["hidden_size"]
    sd["gpt_neox.final_layer_norm.weight"].zero_()
    sd["gpt_neox.final_layer_norm.bias"].fill_(1.0)
    g = torch.Generator().manual_seed(9)
    vals = (torch.rand(V, generator=g) * 16 - 8).to(DTYPES[dtype]).float()
    vals[[77, 412]] = 9.0                          # an exact tie: the lower id wins
    head = torch.zeros(V, H)
    head[torch.arange(V), torch.arange(V) % H] = vals
    sd["embed_out.weight"] = head
    m, _, _ = _reader("neox-d128", dtype, sd=sd)
    rng = np.random.default_rng(5)
    windows = [rng.integers(0, V, n).tolist() for n in (3, 70)]
    rows = [0, 2, 3, 40, 72, 72, 72]
    toks = [77, 412, int(rng.integers(0, V)), 0, V - 1, 77, 5]
    rc, lp, gr = _call(m, windows, rows, toks)
    assert rc == 0
    x = vals.numpy()[None, :].repeat(len(rows), 0)
    want, greedy, bound = LO.choices(x, V, np.arange(len(rows)), toks)
    err = np.abs(lp.double().numpy() - want)
    print(f"[oracle {dtype}] max |err| / bound {float((err / bound).max()):.3f}")
    assert (err <= bound).all(), (err, bound)
    assert gr.tolist() == greedy.astype(int).tolist() and gr.tolist()[0] == 1 and gr.tolist()[1] == 0


def test_refusals_leave_the_outputs_untouched():
    m, cfg, sd = _reader("llama-gqa4", "fp16")
    V = cfg["vocab_size"]
    windows = [[1, 2, 3], [4, 5]]
    for rows, toks, short, code in (([0, -1], [1, 1], 0, 1), ([5], [1], 0, 1), ([0], [V], 0, 1), ([4], [3], 1, None)):
        rc, lp, gr = _call(m, windows, rows, toks, short)
        from retrieval_scaling_b200 import _lib
        want = _lib.RSB_ERR_OOM if code is None else _lib.RSB_ERR_INVALID
        assert rc == want, (rows, toks, short, m.L.rsb_llm_last_error())
        assert bool(torch.isnan(lp).all()) and bool((gr == 7).all())
    empty, _, _ = _reader("llama-gqa4", "fp16", load=False)
    rc, lp, gr = _call(empty, windows, [0], [1])
    from retrieval_scaling_b200 import _lib
    assert rc == _lib.RSB_ERR_STATE and bool(torch.isnan(lp).all()) and bool((gr == 7).all())
    with pytest.raises(ValueError, match="empty context"):
        m.loglikelihood([([], [1])], 16)


def _fork_loglikelihood(hf, requests, max_length, delta):
    """(ll, is_greedy, near_tie) per request: HFLM._loglikelihood_tokens with transformers fp32 on the CPU, one
    request at a time (a right-padded batch gives the same rows for a causal model)."""
    out = []
    with torch.no_grad():
        for ctx, cont in requests:
            inp = (ctx + cont)[-(max_length + 1):][:-1]
            logits = torch.log_softmax(hf(torch.tensor([inp])).logits[0].float(), dim=-1)[len(inp) - len(cont):]
            top2 = logits.topk(2, dim=-1).values
            c = torch.tensor(cont)
            out.append((float(logits.gather(1, c[:, None]).sum()), bool((logits.argmax(-1) == c).all()),
                        bool(((top2[:, 0] - top2[:, 1]) < delta).any())))
    return out


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_reader_loglikelihood_against_transformers(dtype):
    m, cfg, sd = _reader("llama-gqa4", dtype)
    hf = LF.hf_model(cfg)
    hf.load_state_dict(sd, strict=False)
    rng = np.random.default_rng(6)
    V, ML = cfg["vocab_size"], 48
    reqs = []
    for _ in range(24):
        ctx = rng.integers(0, V, int(rng.integers(1, 80))).tolist()       # many past max_length: truncated
        for k in (1, 1, 3, 6):
            reqs.append((ctx, rng.integers(0, V, k).tolist()))
    got = m.loglikelihood(reqs, ML)
    want = _fork_loglikelihood(hf, reqs, ML, DELTA[dtype])
    worst, ties = 0.0, 0
    for (ll, g), (wl, wg, tie), (_, cont) in zip(got, want, reqs):
        err = abs(ll - wl)
        worst = max(worst, err / len(cont))
        assert err <= LL_TOL[dtype] * len(cont), (ll, wl, len(cont))
        ties += tie
        if not tie:
            assert g == wg
    print(f"loglikelihood {dtype}: |d ll| / token max {worst:.2e}; {ties} of {len(reqs)} near-ties excused")


def _bpe(corpus, vocab):
    from tokenizers import Tokenizer, decoders, models, pre_tokenizers, trainers
    from transformers import PreTrainedTokenizerFast
    tok = Tokenizer(models.BPE())
    tok.pre_tokenizer = pre_tokenizers.ByteLevel(add_prefix_space=False)
    tok.decoder = decoders.ByteLevel()
    trainer = trainers.BpeTrainer(vocab_size=vocab, special_tokens=["<unk>", "<s>", "</s>"],
                                  initial_alphabet=pre_tokenizers.ByteLevel.alphabet())
    tok.train_from_iterator(corpus, trainer)
    return PreTrainedTokenizerFast(tokenizer_object=tok, unk_token="<unk>", bos_token="<s>", eos_token="</s>",
                                   pad_token="<unk>")


def test_main_ric_multiple_choice_against_transformers(tmp_path):
    from golden import roberta_fixture as RF
    from safetensors.torch import save_file

    from retrieval_scaling_b200 import config as C
    from retrieval_scaling_b200 import rag_mc
    from retrieval_scaling_b200.search import get_merged_search_output_path
    rng = np.random.default_rng(13)
    syll = ["ka", "ri", "to", "men", "sa", "lo", "vi", "dun", "pe", "qua", "zor", "bel"]
    words = ["".join(rng.choice(syll, int(rng.integers(1, 4)))) for _ in range(200)]
    sentence = lambda n: " ".join(str(x) for x in rng.choice(words, n)) + "."   # noqa: E731
    passages = [" ".join(sentence(int(rng.integers(4, 12))) for _ in range(3)) for _ in range(120)]
    tok = _bpe(passages + ["Answer: A B C D"] * 5, LF.CONFIG["vocab_size"])
    cfg = dict(LF.CONFIG, max_position_embeddings=256)
    reader_dir = LF.build_dir(str(tmp_path / "reader"), cfg)
    sd = LF.seeded_state_dict(cfg)
    save_file({k: v.contiguous() for k, v in sd.items()}, os.path.join(reader_dir, "model.safetensors"))
    tok.save_pretrained(reader_dir)
    enc = RF.build(str(tmp_path / "enc"))
    psg_dir = tmp_path / "passages" / "dom" / "1-shards"
    psg_dir.mkdir(parents=True)
    with open(psg_dir / "raw_passages-0-of-1.jsonl", "w") as f:
        for i, t in enumerate(passages):
            f.write(json.dumps({"id": i, "title": f"t{i % 7}", "text": t}) + "\n")
    shots = "The following are questions.\n\n" + "".join(
        f"{sentence(5)}\nA. {words[i]}\nB. {words[i + 1]}\nC. {words[i + 2]}\nD. {words[i + 3]}\nAnswer: "
        f"{'ABCD'[i % 4]}\n\n" for i in range(0, 8, 4))
    tasks = {"medqa_4options": 10, "mmlu_anatomy": 7, "mmlu_virology": 5}
    questions, samples = [], {}
    for t, n in tasks.items():
        rows = []
        for i in range(n):
            q = f"{sentence(int(rng.integers(3, 8)))}\nA. {words[i]}\nB. {words[i + 5]}\nC. {words[i + 9]}\nD. x\nAnswer:"
            questions.append(q)
            ctx = shots + q
            rows.append({"doc_id": i, "doc": {"question": q}, "target": int(rng.integers(0, 4)),
                         "arguments": {f"gen_args_{j}": {"arg_0": ctx, "arg_1": " " + c} for j, c in enumerate("ABCD")}})
        samples[t] = rows
    sdir = tmp_path / "samples"
    sdir.mkdir()
    for t, rows in samples.items():
        with open(sdir / f"samples_{t}_2026-10-19T12-00-00.000001.json", "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")
    with open(tmp_path / "questions.jsonl", "w") as f:
        for q in questions:
            f.write(json.dumps({"query": q}) + "\n")
    ov = [f"datastore.datastore_root_dir={tmp_path}", "datastore.domain=dom", "model.datastore_encoder=dragon-roberta",
          f"model.query_encoder={enc['query']['dir']}", f"datastore.embedding.model_name_or_path={enc['context']['dir']}",
          "datastore.index.index_type=Flat", "evaluation.search.n_docs=3",
          f"evaluation.data.eval_data={tmp_path / 'questions.jsonl'}", f"model.lm_model={reader_dir}",
          "evaluation.concate_k=2", "tasks.eval.task_name=lm-eval", f"evaluation.lm_eval.samples_dir={sdir}",
          f"evaluation.lm_eval.predictions_file={tmp_path / 'pred.jsonl'}",
          f"evaluation.results_only_log_file={tmp_path / 'results.log'}"]
    main = [sys.executable, os.path.join(ROOT, "ric", "main_ric.py"), "--config-name", "perplexity"]
    r = subprocess.run(main + ["evaluation.domain=nq_open", "tasks.datastore.embedding=true", "tasks.eval.search=true",
                               *ov], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    merged = get_merged_search_output_path(C.load_config("perplexity", os.path.join(ROOT, "ric", "conf"),
                                                         ov + ["evaluation.domain=nq_open"]))
    retrieved = {}
    for line in open(merged):
        row = json.loads(line)
        retrieved[row["raw_query"].split("\n\n")[-1]] = "".join(c["retrieval text"] for c in row["ctxs"][:2][::-1])
    hf = LF.hf_model(cfg)
    hf.load_state_dict(sd, strict=False)

    for domain in ("medqa_4options", "mmlu"):
        r = subprocess.run(main + [f"evaluation.domain={domain}", f"evaluation.lm_eval.retrieval_file={merged}",
                                   "tasks.eval.inference=true", *ov], cwd=ROOT, capture_output=True, text=True,
                           timeout=900)
        assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
        preds = [json.loads(line) for line in open(tmp_path / "pred.jsonl")]
        docs = [(t, d) for t in (["medqa_4options"] if domain != "mmlu" else ["mmlu_anatomy", "mmlu_virology"])
                for d in samples[t]]
        assert len(preds) == len(docs)
        same = ties = correct = 0
        for p, (t, d) in zip(preds, docs):
            ctx = retrieved[d["doc"]["question"]] + shots + d["doc"]["question"]
            reqs = [rag_mc.encode_pair(tok, ctx, " " + c) for c in "ABCD"]
            fork = _fork_loglikelihood(hf, reqs, 256, DELTA["fp16"])
            lls = np.array([f[0] for f in fork])
            top = np.sort(lls)[::-1]
            near = top[0] - top[1] < DELTA["fp16"]
            pred = int(np.argmax(lls))
            ties += near
            same += p["pred"] == pred
            if not near:
                assert p["pred"] == pred, (p, lls)
            assert p["task"] == t and p["gold"] == d["target"]
            correct += p["pred"] == d["target"]
        import re
        acc = float(re.search(r"Domain = " + domain + r"\t.*?acc = ([0-9.]+)", open(tmp_path / "results.log").read())
                    .group(1))
        print(f"{domain}: {same} of {len(docs)} preds equal to the fp32 fork restatement, {ties} near-ties excused, "
              f"acc {acc:.4f}")
        assert acc == pytest.approx(correct / len(docs), abs=1e-4)
        assert ties <= len(docs) // 2
