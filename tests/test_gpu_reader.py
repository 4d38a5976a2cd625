"""GPU checks of the Llama reader (rsb_llm_*): per-token NLL against the committed fp64 golden at the attention kernel's
tile edges and at max_position_embeddings, held to the precision of HF's own bf16 forward (the reference's reader
dtype) on the same inputs; label masks; packing; determinism; refusals."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import llama_fixture as F  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    from retrieval_scaling_b200.reader import B200Llama
    m = B200Llama(F.CONFIG)
    m.load_state_dict(F.seeded_state_dict())
    return m


@pytest.fixture(scope="module")
def golden():
    g = np.load(F.GOLDEN)
    cu = g["cu_seqlens"]
    return [g["ids"][cu[b]:cu[b + 1]] for b in range(len(cu) - 1)], [g["nll"][cu[b]:cu[b + 1]] for b in range(len(cu) - 1)]


@pytest.fixture(scope="module")
def hf_bf16(golden):
    m = F.hf_model(dtype=torch.bfloat16, attn_implementation="sdpa").cuda()
    out = [F.hf_token_nll(m, w) for w in golden[0]]
    del m
    torch.cuda.empty_cache()
    return out


def _masks(ids, kind, seed):
    lab = np.array(ids, np.int64)
    if kind == "none":
        lab[:] = -100
    elif kind == "partial":
        rng = np.random.default_rng(seed)
        lab[rng.random(len(ids)) < 0.5] = -100
        lab[: len(ids) // 3] = -100                # a masked prefix, as a retrieved context before the answer
    return lab


def test_nll_against_fp64_golden_within_hf_bf16_precision(model, golden, hf_bf16):
    windows, gold = golden
    ours = model.nll(windows, windows)           # full labels, every window in one packed forward
    err_ours, err_bf16, mean_ours, mean_bf16 = [], [], [], []
    for w, o, g, b in zip(windows, ours, gold, hf_bf16):
        o = o.numpy().astype(np.float64)
        assert np.all(np.isfinite(o)) and o[0] == 0.0
        if len(w) < 2:
            assert np.all(o == 0)
            continue
        err_ours.append(np.abs(o[1:] - g[1:]))
        err_bf16.append(np.abs(b[1:] - g[1:]))
        mean_ours.append(abs(o[1:].mean() - g[1:].mean()))
        mean_bf16.append(abs(b[1:].mean() - g[1:].mean()))
    e_o, e_b = np.concatenate(err_ours), np.concatenate(err_bf16)
    p99_o, p99_b = np.percentile(e_o, 99), np.percentile(e_b, 99)
    print(f"per-token |err| p99: ours {p99_o:.3e}, HF bf16 {p99_b:.3e}; max ours {e_o.max():.3e}; "
          f"sample-mean |err| max: ours {max(mean_ours):.3e}, HF bf16 {max(mean_bf16):.3e}")
    assert p99_o <= p99_b
    assert max(mean_ours) <= max(mean_bf16)
    assert np.mean(mean_ours) <= np.mean(mean_bf16)


@pytest.mark.parametrize("budget", [None, 1, 300])
def test_label_masks_packing_and_determinism(model, golden, budget):
    windows, _ = golden
    kinds = ["full", "partial", "none"]
    labels = [_masks(w, kinds[i % 3], i) for i, w in enumerate(windows)]
    full = model.nll(windows, windows)
    masked = model.nll(windows, labels, max_tokens=budget)
    again = model.nll(windows, labels, max_tokens=budget)
    for w, f, m, a, lb in zip(windows, full, masked, again, labels):
        assert torch.equal(m, a)                                    # bit-identical runs
        scored = np.zeros(len(w), bool)
        scored[1:] = lb[1:] != -100
        assert torch.equal(m[scored], f[scored])                   # a token's NLL does not depend on the others' labels
        assert torch.all(m[~scored] == 0)


def test_packed_equals_one_at_a_time(model, golden):
    windows, _ = golden
    order = [7, 0, 3, 1, 5, 2, 6, 4]                                # mixed lengths in one pack (all but 4096)
    packed = model.nll([windows[i] for i in order], [windows[i] for i in order])
    for i, p in zip(order, packed):
        assert torch.equal(p, model.nll([windows[i]], [windows[i]])[0])


def test_loss_is_hf_mean_and_nan_without_labels(model, golden):
    windows, _ = golden
    w = windows[4]
    lab = _masks(w, "partial", 3)
    nll = model.nll([w], [lab])[0].double()
    pos = [t for t in range(1, len(w)) if lab[t] != -100]
    losses = model.loss([w, w, windows[0]], [lab, _masks(w, "none", 0), windows[0]])
    assert losses[0] == pytest.approx(float(nll[pos].mean()), rel=1e-12)
    assert np.isnan(losses[1]) and np.isnan(losses[2])


def test_gqa_1to1_and_tied_reader_within_hf_bf16_precision():
    """MHA with rope_theta 5e5, and tied embeddings: against the fp64 oracle, held to HF bf16's own error on the same
    windows (per-token 99th percentile and the worst window mean), as the golden test is."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import llama_oracle as O
    from retrieval_scaling_b200.reader import B200Llama
    for cfg in (dict(F.CONFIG, num_key_value_heads=4, rope_theta=500000.0, max_position_embeddings=512),
                dict(F.CONFIG, tie_word_embeddings=True, num_hidden_layers=1, max_position_embeddings=512)):
        sd = F.seeded_state_dict(cfg, seed=11)
        m = B200Llama(cfg)
        m.load_state_dict(sd)
        hf = F.hf_model(cfg, dtype=torch.bfloat16, seed=11, attn_implementation="sdpa").cuda()
        rng = np.random.default_rng(5)
        windows = [rng.integers(0, cfg["vocab_size"], S) for S in (5, 64, 200, 512)]
        e_o, e_b, m_o, m_b = [], [], [], []
        for w, o in zip(windows, m.nll(windows, windows)):
            ref = O.token_nll(sd, cfg, w)[1:]
            o, b = o.numpy().astype(np.float64)[1:], F.hf_token_nll(hf, w)[1:]
            e_o.append(np.abs(o - ref)); e_b.append(np.abs(b - ref))
            m_o.append(abs(o.mean() - ref.mean())); m_b.append(abs(b.mean() - ref.mean()))
        p_o, p_b = np.percentile(np.concatenate(e_o), 99), np.percentile(np.concatenate(e_b), 99)
        print(f"{cfg['num_key_value_heads']} kv heads, tied {cfg['tie_word_embeddings']}: p99 ours {p_o:.3e} "
              f"HF bf16 {p_b:.3e}; worst window mean ours {max(m_o):.3e} HF bf16 {max(m_b):.3e}")
        assert p_o <= p_b and max(m_o) <= max(m_b), cfg
        del hf, m
        torch.cuda.empty_cache()


def test_refusals_before_any_launch(model):
    from retrieval_scaling_b200.reader import B200Llama
    V, P = F.CONFIG["vocab_size"], F.CONFIG["max_position_embeddings"]
    with pytest.raises(ValueError, match="token id"):
        model.nll([[1, V]], [[1, 2]])
    with pytest.raises(ValueError, match="label"):
        model.nll([[1, 2]], [[1, -5]])
    with pytest.raises(ValueError, match="label"):
        model.nll([[1, 2]], [[1, V]])
    with pytest.raises(NotImplementedError, match="max_position_embeddings"):
        model.nll([[1] * (P + 1)], [[1] * (P + 1)])
    with pytest.raises(ValueError, match="empty"):
        model.nll([[]], [[]])
    part = B200Llama(dict(F.CONFIG, num_hidden_layers=1))
    part.load_weight("model.norm.weight", torch.ones(512))
    with pytest.raises(RuntimeError, match="not loaded"):
        part.nll([[1, 2]], [[1, 2]])
    with pytest.raises(ValueError, match="finite"):
        part.load_weight("model.norm.weight", torch.full((512,), 1e5, dtype=torch.bfloat16))
    # fp16 overflow of the residual stream is reported, not returned as inf / NaN
    cfg1 = dict(F.CONFIG, num_hidden_layers=1)
    sd = F.seeded_state_dict(cfg1)
    sd["model.embed_tokens.weight"].fill_(65000.0)
    sd["model.layers.0.self_attn.o_proj.weight"] *= 1e4       # o_proj rows ~1e4: 65000 + 1e4 > 65504
    hot = B200Llama(cfg1)
    hot.load_state_dict(sd)
    with pytest.raises(FloatingPointError, match="overflow"):
        hot.nll([[5, 6, 7]], [[5, 6, 7]])
    from retrieval_scaling_b200 import _lib
    L = _lib.lib()
    x = torch.zeros(4, dtype=torch.int32, device="cuda")
    bad_cu = torch.tensor([0, 3, 2], dtype=torch.int32, device="cuda")
    out = torch.zeros(4, dtype=torch.float32, device="cuda")
    ws = torch.empty(L.rsb_llm_workspace_bytes(model._h, 4, 4), dtype=torch.uint8, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())   # noqa: E731
    assert L.rsb_llm_nll(model._h, p(x), p(bad_cu), 2, 4, 4, p(x), p(out), p(ws), ws.numel(), None) == _lib.RSB_ERR_INVALID
    assert L.rsb_llm_nll(model._h, p(x), p(bad_cu), 2, 4, 4, p(x), p(out), p(ws), 16, None) == _lib.RSB_ERR_INVALID


@pytest.mark.parametrize("concate_k", [0, 3])
def test_main_ric_perplexity_end_to_end(tmp_path, concate_k):
    """`ric/main_ric.py --config-name perplexity tasks.eval.search=true tasks.eval.inference=true` on a tiny seeded
    datastore (passage embedding and search with the DRAGON-RoBERTa fixture encoders, the seeded Llama reader, 'longest'
    decontamination on), against the reference's loop restated here on the CPU with transformers in fp32."""
    import json
    import re
    import subprocess

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from golden import roberta_fixture as RF
    from retrieval_scaling_b200 import config as C
    from retrieval_scaling_b200 import perplexity as P
    enc = RF.build(str(tmp_path / "enc"))
    reader_dir = F.build_dir(str(tmp_path / "reader"))
    rng = np.random.default_rng(9)
    texts = [" ".join(f"w{i}" for i in rng.integers(3, 1000, n)) for n in (300, 200)]
    words = " ".join(texts).split()
    psg_dir = tmp_path / "passages" / "dom" / "1-shards"
    psg_dir.mkdir(parents=True)
    with open(psg_dir / "raw_passages-0-of-1.jsonl", "w") as f:
        for i in range(150):
            if i % 5 == 0:                                         # copies of eval text: decontamination removes some
                s = int(rng.integers(0, len(words) - 60))
                t = " ".join(words[s:s + 60])
            else:
                t = " ".join(f"w{j}" for j in rng.integers(3, 1000, int(rng.integers(10, 60))))
            f.write(json.dumps({"id": i, "title": f"t{i % 5}", "text": t}) + "\n")
    eval_path = tmp_path / "ppl.jsonl"
    with open(eval_path, "w") as f:
        for t in texts:
            f.write(json.dumps({"text": t}) + "\n")
    log = tmp_path / f"results_{concate_k}.log"
    ov = [f"datastore.datastore_root_dir={tmp_path}", "datastore.domain=dom", "evaluation.domain=dom",
          "model.datastore_encoder=dragon-roberta", f"model.query_encoder={enc['query']['dir']}",
          f"datastore.embedding.model_name_or_path={enc['context']['dir']}", "datastore.index.index_type=Flat",
          "evaluation.search.n_docs=10", f"evaluation.data.eval_data={eval_path}", f"model.lm_model={reader_dir}",
          "evaluation.data.max_eval_data_seq_length=128", "evaluation.data.eval_stride=64",
          f"evaluation.concate_k={concate_k}", "evaluation.decontamination=true", "evaluation.contamination_threshold=0.5",
          f"evaluation.results_only_log_file={log}"]
    cmd = [sys.executable, os.path.join(ROOT, "ric", "main_ric.py"), "--config-name", "perplexity",
           "tasks.datastore.embedding=true", "tasks.eval.search=true", "tasks.eval.inference=true", *ov]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    ppl_gpu = float(re.search(r"perplexity = ([0-9.]+)", open(log).read()).group(1))

    cfg = C.load_config("perplexity", os.path.join(ROOT, "ric", "conf"), ov)
    tok = F.tokenizer()
    if concate_k:
        from retrieval_scaling_b200.search import get_merged_search_output_path
        eval_data = [json.loads(line) for line in open(get_merged_search_output_path(cfg))]
        assert all(len(ex["ctxs"]) == 10 for ex in eval_data if ex["raw_query"])   # an empty query is not searched
    else:
        eval_data = P.prepare_ppl_eval_data([json.loads(line) for line in open(eval_path)], tok, 128, 64, True)
    contexts, answers, _ = P.build_doc_prompts(eval_data, cfg.evaluation)
    if concate_k:
        assert sum(c.count(" \n") for c in contexts) > 0
    hf = F.hf_model(dtype=torch.float32)
    total, count = 0.0, 0
    for context, answer in zip(contexts, answers):                # src/evaluate_perplexity.py:117-139
        a = tok(answer, return_tensors="pt")["input_ids"]
        c = tok(context, return_tensors="pt")["input_ids"]
        ids = torch.cat((c, a), 1)
        lab = torch.cat((torch.full(c.size(), -100), a), 1)
        lab = torch.where(lab == 2, torch.tensor(-100), lab)
        with torch.no_grad():
            total += hf(ids[:, -4096:], labels=lab[:, -4096:]).loss.item()
        count += 1
    ppl_cpu = float(torch.exp(torch.tensor(total / count)))
    print(f"concate_k {concate_k}: {count} windows, perplexity GPU {ppl_gpu:.4f} CPU fp32 {ppl_cpu:.4f}")
    assert ppl_gpu == pytest.approx(ppl_cpu, rel=1e-3)
