"""GPU checks of greedy generation (`rsb_llm_generate`, `_Reader.generate`) on the seeded reader fixtures: Llama with
GQA 4:1, GPT-NeoX at head_dim 64 / 80 / 128 / 256, OLMo and OLMo-2, each in fp16 and bf16.  Each decoded token's
log-probability against the prefill NLL of the same text, the tokens against the fp64 oracles' argmax, batch
invariance, and the edges: context lengths around the 16- and 64-position tiles, a context ending at
max_pos - max_new_tokens, one new token, EOS at step 0 and a list of EOS ids, and a head whose real logits are all
negative."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import llama_fixture as LF  # noqa: E402
import llama_oracle as LO  # noqa: E402
import neox_fixture as NF  # noqa: E402
import neox_oracle as NO  # noqa: E402
import olmo_fixture as OF  # noqa: E402
import olmo_oracle as OO  # noqa: E402

pytestmark = pytest.mark.gpu

CASES = {
    "llama-gqa4": ("B200Llama", LF, LF.CONFIG),
    "neox-d64": ("B200NeoX", NF, dict(NF.CONFIG, num_attention_heads=8)),
    "neox-d80": ("B200NeoX", NF, dict(NF.CONFIG, hidden_size=640, num_attention_heads=8)),
    "neox-d128": ("B200NeoX", NF, dict(NF.CONFIG, num_attention_heads=4)),
    "neox-d256": ("B200NeoX", NF, NF.CONFIG),
    "olmo": ("B200Olmo", OF, OF.CONFIGS["olmo"]),
    "olmo2": ("B200Olmo", OF, OF.CONFIGS["olmo2"]),
}
DTYPES = {"fp16": torch.float16, "bf16": torch.bfloat16}
# decode log-probability against the prefill NLL of the same text: both round to the dtype at the same points and
# differ in the attention's order of summation (split-KV chunks against 64-key blocks)
LP_TOL = {"fp16": 2e-2, "bf16": 1e-1}
# oracle top-2 logit margin below which a step is a near-tie: several times the dtype's logit error on the fixtures
DELTA = {"fp16": 0.05, "bf16": 0.3}
LENS = [1, 63, 64, 65, 127, 128, 129, 300]


def _sd(FX, cfg, seed=None):
    if FX is OF:
        return OF.seeded_state_dict(cfg) if seed is None else OF.seeded_state_dict(cfg, seed)
    return FX.seeded_state_dict(cfg) if seed is None else FX.seeded_state_dict(cfg, seed)


def _reader(name, dtype, **change):
    from retrieval_scaling_b200 import reader
    cls, FX, base = CASES[name]
    cfg = dict(base, **change)
    sd = _sd(FX, cfg)
    m = getattr(reader, cls)(cfg, dtype=DTYPES[dtype])
    m.load_state_dict(sd)
    return m, cfg, sd, FX


def _prompts(vocab, lens, seed):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, vocab, n).tolist() for n in lens]


def _oracle_logits(FX, sd, cfg, ids):
    """fp64 logits [S, vocab] of one sequence."""
    dev = "cuda"
    f = lambda k: sd[k].to(device=dev, dtype=torch.float64)   # noqa: E731
    if FX is LF:
        x = LO.hidden_rows(sd, cfg, ids, dev)[-1]
        x = LO._rms(x, f("model.norm.weight"), cfg["rms_norm_eps"])
        head = f("lm_head.weight")
    elif FX is NF:
        x = NO.hidden_rows(sd, cfg, ids, dev)[-1]
        x = NO._ln(x, f("gpt_neox.final_layer_norm.weight"), f("gpt_neox.final_layer_norm.bias"), cfg["layer_norm_eps"])
        head = f("embed_out.weight")
    else:
        x = OO.hidden_rows(sd, cfg, ids, dev)[-1]
        x = OO.rms_norm(x, f("model.norm.weight"), OO.eps(cfg)) if OO.version(cfg) == 2 else OO.layer_norm(x)
        head = f("model.embed_tokens.weight") if cfg.get("tie_word_embeddings") else f("lm_head.weight")
    return x @ head.T


@pytest.mark.parametrize("dtype", list(DTYPES))
@pytest.mark.parametrize("name", list(CASES))
def test_decode_against_prefill_and_oracle(name, dtype):
    """Every generated token's log-probability matches rsb_llm_nll over [context + generated] within LP_TOL; every
    token is the fp64 oracle's argmax at each step whose top-2 margin is at least DELTA (teacher-forced on the
    generated prefix), and most steps are compared."""
    m, cfg, sd, FX = _reader(name, dtype)
    prompts = _prompts(cfg["vocab_size"], LENS, 11)
    max_new = 24
    toks, lps = m.generate(prompts, max_new, [], return_logprobs=True)
    full = [p + t for p, t in zip(prompts, toks)]
    nll = m.nll(full, full)
    compared = steps = 0
    first_tie = []
    worst = 0.0
    for p, t, lp, n in zip(prompts, toks, lps, nll):
        assert len(t) == max_new and all(0 <= v < cfg["vocab_size"] for v in t)
        want = -n[len(p):len(p) + max_new].double()
        err = float((lp.double() - want).abs().max())
        worst = max(worst, err)
        assert err <= LP_TOL[dtype], (len(p), err)
        logits = _oracle_logits(FX, sd, cfg, p + t[:-1])[len(p) - 1:]
        top2 = logits.topk(2, dim=-1)
        margin = (top2.values[:, 0] - top2.values[:, 1]).cpu().numpy()
        arg = top2.indices[:, 0].cpu().numpy()
        tie = [s for s in range(max_new) if margin[s] < DELTA[dtype]]
        first_tie.append(tie[0] if tie else max_new)
        for s in range(max_new):
            steps += 1
            if margin[s] >= DELTA[dtype]:
                compared += 1
                assert t[s] == arg[s], (len(p), s, t[s], int(arg[s]), float(margin[s]))
    print(f"{name} {dtype}: decode vs prefill |dlogp| max {worst:.2e}; oracle argmax compared at {compared} of {steps} "
          f"steps (margin >= {DELTA[dtype]}); equal up to the first near-tie in every sequence, first near-tie at "
          f"steps {first_tie}")
    assert compared >= 0.5 * steps


@pytest.mark.parametrize("name, dtype", [("llama-gqa4", "fp16"), ("llama-gqa4", "bf16"), ("neox-d256", "fp16"),
                                         ("olmo2", "bf16")])
def test_batch_invariance(name, dtype):
    """A sequence decoded alone and inside a batch of 37 mixed-length prompts gives bit-identical ids and
    log-probabilities."""
    m, cfg, _, _ = _reader(name, dtype)
    rng = np.random.default_rng(5)
    lens = rng.integers(1, 400, 37).tolist()
    prompts = _prompts(cfg["vocab_size"], lens, 6)
    toks, lps = m.generate(prompts, 20, [], return_logprobs=True)
    for i in (0, 7, 19, 36, int(np.argmin(lens)), int(np.argmax(lens))):
        t, lp = m.generate([prompts[i]], 20, [], return_logprobs=True)
        assert t[0] == toks[i] and torch.equal(lp[0], lps[i]), i


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_edges(dtype):
    m, cfg, _, _ = _reader("llama-gqa4", dtype, max_position_embeddings=512)
    V = cfg["vocab_size"]
    prompts = _prompts(V, [1, 63, 64, 65, 127, 128, 129, 512 - 8], 3)
    toks = m.generate(prompts, 8, [])
    assert all(len(t) == 8 for t in toks)                       # the last context ends exactly at max_pos - 8
    with pytest.raises(NotImplementedError, match="max_position_embeddings"):
        m.generate(_prompts(V, [512 - 7], 3), 8, [])
    one = m.generate(prompts, 1, [])
    assert one == [t[:1] for t in toks]
    eos0 = m.generate(prompts[:3], 8, toks[0][0])                # EOS at step 0 of the first sequence
    assert eos0[0] == toks[0][:1]
    stop = [toks[1][3], V + 5]                                   # a list of EOS ids, one outside the vocabulary
    got = m.generate(prompts[:3], 8, stop)
    for t, g in zip(toks[:3], got):
        cut = next((s + 1 for s, v in enumerate(t) if v in stop), len(t))
        assert g == t[:cut]
    assert len(got[1]) <= 4
    with pytest.raises(ValueError, match="empty"):
        m.generate([[]], 4, [])
    with pytest.raises(ValueError, match="outside the vocabulary"):
        m.generate([[V]], 4, [])


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_pad_logits_never_win(dtype):
    """A head whose real logits are all negative: the LM head's zero pad rows (vocab 1000 -> 1024) score 0, above
    every real logit, and are never chosen.  The final LayerNorm's zero weight and unit bias make every normed row all
    ones; each embed_out row has a negative sum."""
    from retrieval_scaling_b200 import reader
    cfg = dict(NF.CONFIG, num_attention_heads=4)
    sd = NF.seeded_state_dict(cfg)
    sd["gpt_neox.final_layer_norm.weight"].zero_()
    sd["gpt_neox.final_layer_norm.bias"].fill_(1.0)
    sd["embed_out.weight"] = -sd["embed_out.weight"].abs() * 0.1
    m = reader.B200NeoX(cfg, dtype=DTYPES[dtype])
    m.load_state_dict(sd)
    toks, lps = m.generate(_prompts(cfg["vocab_size"], [1, 40, 130], 2), 6, [], return_logprobs=True)
    ids = {v for t in toks for v in t}
    assert len(ids) == 1 and 0 <= ids.pop() < cfg["vocab_size"]   # every row has the same logits
    assert all(bool((lp <= 0).all()) for lp in lps)


@pytest.mark.parametrize("dtype", list(DTYPES))
def test_query_groups_wider_than_one_tile(dtype):
    """20 query heads on one KV head (multi-query attention): the decode kernel takes the group in two 16-row tiles.
    Every token's log-probability matches the prefill NLL of the same text."""
    m, cfg, _, _ = _reader("llama-gqa4", dtype, hidden_size=20 * 128, num_attention_heads=20, num_key_value_heads=1,
                           intermediate_size=256, num_hidden_layers=1)
    prompts = _prompts(cfg["vocab_size"], [1, 65, 200], 8)
    toks, lps = m.generate(prompts, 12, [], return_logprobs=True)
    full = [p + t for p, t in zip(prompts, toks)]
    for p, lp, n in zip(prompts, lps, m.nll(full, full)):
        err = float((lp.double() + n[len(p):len(p) + 12].double()).abs().max())
        assert err <= LP_TOL[dtype], (len(p), err)


def test_c_abi_refusals():
    """rsb_llm_generate's own refusals, called directly: an empty context RSB_ERR_INVALID and a workspace below
    rsb_llm_generate_workspace_bytes RSB_ERR_OOM, both before any launch (the outputs stay untouched)."""
    import ctypes

    from retrieval_scaling_b200 import _lib
    m, cfg, _, _ = _reader("llama-gqa4", "fp16")
    L = m.L
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def call(ids, cu, max_seqlen, ws_bytes):
        B, T = len(cu) - 1, len(ids)
        d_ids = torch.tensor(ids, dtype=torch.int32, device="cuda")
        d_cu = torch.tensor(cu, dtype=torch.int32, device="cuda")
        toks = torch.full((B, 4), 7, dtype=torch.int32, device="cuda")
        lens = torch.full((B,), 7, dtype=torch.int32, device="cuda")
        ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device="cuda")
        rc = L.rsb_llm_generate(m._h, ctypes.c_void_p(d_ids.data_ptr()), ctypes.c_void_p(d_cu.data_ptr()), B, T,
                                max_seqlen, 4, None, 0, ctypes.c_void_p(toks.data_ptr()),
                                ctypes.c_void_p(lens.data_ptr()), None, ctypes.c_void_p(ws.data_ptr()), ws_bytes,
                                stream)
        torch.cuda.synchronize()
        untouched = bool((toks == 7).all()) and bool((lens == 7).all())
        return rc, L.rsb_llm_last_error().decode(), untouched

    need = L.rsb_llm_generate_workspace_bytes(m._h, 2, 5, 3, 4)
    rc, msg, untouched = call([1, 2, 3, 4, 5], [0, 0, 5], 5, L.rsb_llm_generate_workspace_bytes(m._h, 2, 5, 5, 4))
    assert rc == _lib.RSB_ERR_INVALID and "empty" in msg and untouched
    rc, msg, untouched = call([1, 2, 3, 4, 5], [0, 2, 5], 3, need - 1)
    assert rc == _lib.RSB_ERR_OOM and "workspace" in msg and untouched
    rc, _, untouched = call([1, 2, 3, 4, 5], [0, 2, 5], 3, need)
    assert rc == _lib.RSB_OK and not untouched
