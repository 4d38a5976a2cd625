"""GPU checks of the GPT-NeoX reader (rsb_llm_create, then rsb_llm_*): per-token NLL against the committed fp64
golden held to HF bf16's own error, label masks, packing and determinism, partial RoPE bit for bit, causal attention
per element at head_dim 64 / 80 / 128 / 256, production widths against transformers, pickle loading and the overflow
check.  Every per-element comparison also has to reject a deliberately wrong reference."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import neox_fixture as F  # noqa: E402

pytestmark = pytest.mark.gpu


def _must_fail(name, ok):
    assert not bool(np.all(ok)), f"the comparison also accepts the wrong reference {name!r}: its tolerance is too loose"


def _r16(x):
    return x.half().double()


def _i32(a):
    return torch.as_tensor(np.asarray(a), dtype=torch.int32, device="cuda")


def _ulp16(x):
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e.clamp_min(-14) - 10)


@pytest.fixture(scope="module")
def model():
    from retrieval_scaling_b200.reader import B200NeoX
    m = B200NeoX(F.CONFIG)
    m.load_state_dict(F.seeded_state_dict())
    return m


@pytest.fixture(scope="module")
def golden():
    g = np.load(F.GOLDEN)
    cu = g["cu_seqlens"]
    return [g["ids"][cu[b]:cu[b + 1]] for b in range(len(cu) - 1)], [g["nll"][cu[b]:cu[b + 1]] for b in range(len(cu) - 1)]


def test_nll_against_fp64_golden_within_hf_bf16_precision(model, golden):
    windows, gold = golden
    hf = F.hf_model(dtype=torch.bfloat16, attn_implementation="sdpa").cuda()
    bf16 = [F.hf_token_nll(hf, w) for w in windows]
    del hf
    torch.cuda.empty_cache()
    ours = model.nll(windows, windows)
    err_o, err_b, mean_o, mean_b = [], [], [], []
    for w, o, g, b in zip(windows, ours, gold, bf16):
        o = o.numpy().astype(np.float64)
        assert np.all(np.isfinite(o)) and o[0] == 0.0
        if len(w) < 2:
            continue
        err_o.append(np.abs(o[1:] - g[1:]))
        err_b.append(np.abs(b[1:] - g[1:]))
        mean_o.append(abs(o[1:].mean() - g[1:].mean()))
        mean_b.append(abs(b[1:].mean() - g[1:].mean()))
    p99_o, p99_b = np.percentile(np.concatenate(err_o), 99), np.percentile(np.concatenate(err_b), 99)
    print(f"per-token |err| p99: ours {p99_o:.3e}, HF bf16 {p99_b:.3e}; window-mean |err| max: ours {max(mean_o):.3e}, "
          f"HF bf16 {max(mean_b):.3e}")
    assert p99_o <= p99_b
    assert max(mean_o) <= max(mean_b)


@pytest.mark.parametrize("budget", [None, 1, 300])
def test_label_masks_packing_and_determinism(model, golden, budget):
    windows, _ = golden
    rng = np.random.default_rng(5)
    labels = []
    for i, w in enumerate(windows):
        lab = np.array(w, np.int64)
        if i % 3 == 1:
            lab[rng.random(len(w)) < 0.5] = -100
        elif i % 3 == 2:
            lab[:] = -100
        labels.append(lab)
    full = model.nll(windows, windows)
    masked = model.nll(windows, labels, max_tokens=budget)
    again = model.nll(windows, labels, max_tokens=budget)
    for w, f, m, a, lb in zip(windows, full, masked, again, labels):
        assert torch.equal(m, a)
        scored = np.zeros(len(w), bool)
        scored[1:] = lb[1:] != -100
        assert torch.equal(m[scored], f[scored])
        assert torch.all(m[~scored] == 0)


def test_packed_equals_one_at_a_time(model, golden):
    windows, _ = golden
    order = [9, 0, 3, 11, 1, 5, 2, 6, 4, 12]
    packed = model.nll([windows[i] for i in order], [windows[i] for i in order])
    for i, p in zip(order, packed):
        assert torch.equal(p, model.nll([windows[i]], [windows[i]])[0])


def _neox(heads, head_dim, rot, max_pos=2048):
    from retrieval_scaling_b200.reader import B200NeoX
    H = heads * head_dim
    return B200NeoX(dict(F.CONFIG, hidden_size=H, num_attention_heads=heads, intermediate_size=max(128, H),
                         rotary_pct=rot / head_dim, num_hidden_layers=1, max_position_embeddings=max_pos))


def _rope_ref(x, pos, rot, base=10000.0, pairing="half"):
    """HF GPT-NeoX partial rotary in fp16 order on x [n, nh, d] fp16 at positions pos: (fp16 result, near-boundary
    mask of cos / sin)."""
    inv = (1.0 / (base ** (torch.arange(0, rot, 2, dtype=torch.int64).float() / rot))).double().cuda()
    f = (torch.as_tensor(pos, dtype=torch.float64, device="cuda")[:, None] * inv[None]).float().double()
    c64, s64 = torch.cos(f), torch.sin(f)
    ulp32 = lambda v: torch.exp2(torch.floor(torch.log2(v.abs().clamp_min(2.0 ** -126))) - 23)   # noqa: E731
    near = ((_r16(c64 - 2 * ulp32(c64)) != _r16(c64 + 2 * ulp32(c64))) | (_r16(s64 - 2 * ulp32(s64)) != _r16(s64 + 2 * ulp32(s64))))
    c, s = _r16(c64)[:, None], _r16(s64)[:, None]
    xd = x.double()
    h = rot // 2
    if pairing == "half":
        x1, x2 = xd[..., :h], xd[..., h:rot]
    else:
        x1, x2 = xd[..., 0:rot:2], xd[..., 1:rot:2]
    o1, o2 = _r16(_r16(x1 * c) + _r16(-x2 * s)), _r16(_r16(x2 * c) + _r16(x1 * s))
    out = xd.clone()
    if pairing == "half":
        out[..., :h], out[..., h:rot] = o1, o2
    else:
        out[..., 0:rot:2], out[..., 1:rot:2] = o1, o2
    nm = torch.zeros(xd.shape, dtype=torch.bool, device="cuda")
    nm[..., :h] = near[:, None]
    nm[..., h:rot] = near[:, None]
    return out.half(), nm


def _attention_ref(qkv, cu, heads, d, mask_shift=0):
    """ctx float64 and a per-element bound (the terms of oracle.attention_oracle.causal_attention with head_dim d) for
    rotated rows qkv [T, 3 heads d] fp16 in [Q | K | V] head order."""
    T, hid = int(cu[-1]), heads * d
    out = torch.zeros((T, hid), dtype=torch.float64, device="cuda")
    bnd = torch.zeros_like(out)
    for b in range(len(cu) - 1):
        t0, S = int(cu[b]), int(cu[b + 1] - cu[b])
        if S == 0:
            continue
        x = qkv[t0:t0 + S].double()
        q, k, v = (x[:, i * hid:(i + 1) * hid].view(S, heads, d).transpose(0, 1) for i in range(3))
        sc = q @ k.transpose(1, 2) / d ** 0.5
        i = torch.arange(S, device="cuda")
        vis = i[None, :] <= i[:, None] + mask_shift
        p = torch.softmax(sc.masked_fill(~vis, -torch.inf), dim=-1)
        ctx = p @ v
        E = p @ v.abs()
        svis = vis.sum(-1).double()[None, :, None]
        qk = (q.abs() @ k.abs().transpose(1, 2)).masked_fill(~vis, 0).amax(-1, keepdim=True) / d ** 0.5
        smax = sc.abs().masked_fill(~vis, 0).amax(-1, keepdim=True)
        a = 2.0 ** -20 + 2.0 ** -22 * smax + svis * 2.0 ** -24 + d * 2.0 ** -23 * qk
        vmax = v.abs().amax(1, keepdim=True)
        bd = (2.0 ** -11 + (svis + 32) * 2.0 ** -24) * E + svis * 2.0 ** -25 * vmax + 2 * a * (E + ctx.abs()) \
            + 0.5 * _ulp16(ctx)
        out[t0:t0 + S] = ctx.transpose(0, 1).reshape(S, hid)
        bnd[t0:t0 + S] = bd.transpose(0, 1).reshape(S, hid)
    return out, bnd


@pytest.mark.parametrize("heads, head_dim", [(8, 64), (8, 80), (4, 128), (2, 256)])
def test_partial_rope_and_attention_per_element(heads, head_dim):
    rot = head_dim // 4
    m = _neox(heads, head_dim, rot)
    lens = [1, 15, 16, 17, 0, 63, 64, 65, 127, 129, 300, 2048]
    cu = np.concatenate([[0], np.cumsum(lens)])
    T = int(cu[-1]) + 5                                             # rows past cu[B] stay untouched
    g = torch.Generator(device="cuda").manual_seed(head_dim)
    qkv0 = (torch.randn(T, 3 * heads * head_dim, generator=g, device="cuda") * 2.0).half()
    qkv = qkv0.clone()
    ctx = torch.full((T, heads * head_dim), 7.0, dtype=torch.float16, device="cuda")
    m.attention(qkv, _i32(cu), max(lens), ctx)
    torch.cuda.synchronize()
    n = int(cu[-1])
    pos = np.concatenate([np.arange(L) for L in lens])
    hid = heads * head_dim
    qk0 = qkv0[:n, :2 * hid].view(n, 2 * heads, head_dim)
    ref, near = _rope_ref(qk0, pos, rot)
    got = qkv[:n, :2 * hid].view(n, 2 * heads, head_dim)
    eq = (got == ref) | near
    assert bool(eq.all()), f"{int((~eq).sum())} rotated elements differ"
    assert torch.equal(got[..., rot:], qk0[..., rot:])                 # pass-through dims bit-identical
    assert torch.equal(qkv[:, 2 * hid:], qkv0[:, 2 * hid:]) and torch.equal(qkv[n:], qkv0[n:])
    assert torch.all(ctx[n:] == 7.0)
    wrong, _ = _rope_ref(qk0, pos, rot, pairing="adjacent")
    _must_fail("GPT-J adjacent-pair rotation", ((got == wrong) | near).cpu().numpy())
    want, bound = _attention_ref(qkv, cu, heads, head_dim)
    err = (ctx[:n].double() - want).abs()
    print(f"head_dim {head_dim}: attention error / bound max {float((err / bound).max()):.3f}")
    assert bool((err <= bound).all())
    w1, _ = _attention_ref(qkv, cu, heads, head_dim, mask_shift=1)
    _must_fail("causal mask one key too far", ((ctx[:n].double() - w1).abs() <= bound).cpu().numpy())


def _ln_ref(x, w, b, eps, order="torch"):
    """float64 LayerNorm of fp16 rows x with fp16 w / b, and the fp32 evaluation error an exact-then-rounded result may
    carry besides its final rounding.  order="rms": the deliberately wrong RMSNorm order, normalised rows rounded to
    fp16 before the weight multiply (and after it, before the bias)."""
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    xh = (xd - mean) / torch.sqrt((xd - mean).pow(2).mean(-1, keepdim=True) + eps)
    if order == "rms":
        return _r16(_r16(_r16(xh) * w.double()) + b.double())
    y = xh * w.double() + b.double()
    # fp32 evaluation error, which exceeds half an fp16 ulp only where y cancels to near zero.  The mean is a sum of at
    # most 45 rounded adds deep (32 per thread, 5 shuffles, 8 warp partials): |d mean| <= 45 2^-24 mean|x|, which enters
    # y as |w| rstd |d mean|; the variance's own sum and rsqrt put a relative 2^-24 x ~24 on xh; then the product and
    # the fma.  Rounded up: 32 2^-24 (|xh w| + |b|) + 64 2^-24 |w| rstd mean|x|.
    rstd = 1.0 / torch.sqrt((xd - mean).pow(2).mean(-1, keepdim=True) + eps)
    extra = 2.0 ** -24 * (32 * ((xh * w.double()).abs() + b.double().abs())
                          + 64 * w.double().abs() * rstd * xd.abs().mean(-1, keepdim=True))
    return y, extra


@pytest.mark.parametrize("hidden", [512, 1024, 2048, 2560, 4096, 5120, 8192])
def test_layernorm_per_element(hidden):
    """rsb_llm_layernorm (the forward's ln_rows_kernel) against float64 on the same fp16 inputs, in its three modes:
    the parallel residual's add then both norms; the row-gathered final norm; the add alone.  Each normed element is
    within 1 fp16 ulp of the float64 value plus the derived fp32 evaluation error of `_ln_ref` (which matters only where
    the result cancels to near zero); the add is bit-equal to fp16(x + a).  Rejected: RMSNorm's rounding order, statistics taken before
    the add."""
    import ctypes
    from retrieval_scaling_b200 import _lib
    L = _lib.lib()
    g = torch.Generator(device="cuda").manual_seed(hidden)
    n, eps = 300, 1e-5
    rnd = lambda *sh, std=1.0, mu=0.0: (torch.randn(*sh, generator=g, device="cuda") * std + mu).half()   # noqa: E731
    x0 = rnd(n, hidden, std=3.0, mu=2.0)
    x0[::7] *= 20                                                      # rows of several magnitudes
    a = rnd(n, hidden, std=2.0)
    w1, b1, w2, b2 = rnd(hidden, std=0.5, mu=1.0), rnd(hidden, std=1.0), rnd(hidden, std=0.5, mu=1.0), rnd(hidden)
    ptr = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None   # noqa: E731
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    def run(x, add, rows, m, with2, w=w1, b=b1):
        o1 = torch.full((m, hidden), 7.0, dtype=torch.float16, device="cuda")
        o2 = torch.full((m, hidden), 7.0, dtype=torch.float16, device="cuda")
        rc = L.rsb_llm_layernorm(hidden, ctypes.c_float(eps), ptr(x), ptr(add), ptr(rows), m, ptr(w), ptr(b),
                                 ptr(w2) if with2 else None, ptr(b2) if with2 else None,
                                 ptr(o1) if w is not None else None, ptr(o2) if with2 else None, st)
        assert rc == _lib.RSB_OK, L.rsb_llm_last_error()
        torch.cuda.synchronize()
        return o1, o2

    def check(got, x, w, b, name):
        want, extra = _ln_ref(x, w, b, eps)
        ok = (got.double() - want).abs() <= _ulp16(want) + extra
        assert bool(ok.all()), f"{name}: {int((~ok).sum())} elements beyond 1 ulp"
        wrong = _ln_ref(x, w, b, eps, order="rms")
        _must_fail(f"{name}: RMSNorm rounding order", ((got.double() - wrong).abs() <= _ulp16(wrong) + extra).cpu().numpy())
        return float(((got.double() - want).abs() / (_ulp16(want) + extra)).max())

    # 1. the layer step: x += a, then ln1 and ln2 of the new x from one set of statistics
    x = x0.clone()
    o1, o2 = run(x, a, None, n, True)
    xs = (x0.double() + a.double()).half()
    assert torch.equal(x, xs)
    worst = max(check(o1, xs, w1, b1, "ln1"), check(o2, xs, w2, b2, "ln2"))
    want_old, _ = _ln_ref(x0, w1, b1, eps)
    _must_fail("statistics before the add", ((o1.double() - want_old).abs() <= _ulp16(want_old)).cpu().numpy())
    # 2. the final norm on gathered rows: x is read, not written
    rows = torch.randperm(n, generator=g, device="cuda")[:n // 2].int()
    x = xs.clone()
    o1, o2 = run(x, None, rows, len(rows), False)
    assert torch.equal(x, xs) and torch.all(o2 == 7.0)
    worst = max(worst, check(o1, xs[rows.long()], w1, b1, "gathered"))
    # 3. the last layer's add alone
    x = x0.clone()
    o1, _ = run(x, a, None, n, False, w=None, b=None)
    assert torch.equal(x, xs) and torch.all(o1 == 7.0)
    print(f"hidden {hidden}: LayerNorm |err| / (1 ulp + fp32 term) max {worst:.3f}")


def _hf_err(cfg, sd, ids):
    """(NLL fp64 of transformers fp32, |fp16 - fp32| per token, pre-final-norm rows fp64 of fp32, |fp16 - fp32| per
    row element) on the GPU."""
    out, rows = {}, {}
    for dt in (torch.float32, torch.float16):
        hf = F.hf_model(cfg, dtype=dt, sd=sd).cuda()
        cap = []
        hk = hf.gpt_neox.final_layer_norm.register_forward_hook(lambda mod, a, o: cap.append(a[0][0].double()))
        out[dt] = F.hf_token_nll(hf, ids)
        hk.remove()
        rows[dt] = cap[0]
        del hf
        torch.cuda.empty_cache()
    return (out[torch.float32], np.abs(out[torch.float16] - out[torch.float32]), rows[torch.float32],
            (rows[torch.float16] - rows[torch.float32]).abs())


@pytest.mark.parametrize("name, layers", [("410m", 1), ("1b", 1), ("1b", 2), ("1.4b", 1), ("2.8b", 2)])
def test_rows_and_nll_at_production_width(name, layers):
    """One 700-token window at a released Pythia width (vocabulary 50304) against transformers fp32 on the device: every
    hidden row before final_layer_norm, and the NLL (worst and mean token), within twice transformers fp16's error."""
    from retrieval_scaling_b200.reader import B200NeoX
    H, nh, I = {"410m": (1024, 16, 4096), "1b": (2048, 8, 8192), "1.4b": (2048, 16, 8192), "2.8b": (2560, 32, 10240)}[name]
    cfg = dict(F.CONFIG, hidden_size=H, num_attention_heads=nh, intermediate_size=I, num_hidden_layers=layers,
               vocab_size=50304)
    sd = F.seeded_state_dict(cfg, seed=H + layers)
    ids = np.random.default_rng(layers).integers(0, 50304, 700)
    ref, err16, h32, herr16 = _hf_err(cfg, sd, ids)
    m = B200NeoX(cfg)
    m.load_state_dict(sd)
    ours = m.nll([ids], [ids])[0].numpy().astype(np.float64)
    rows = m.hidden_states(_i32(ids), _i32([0, len(ids)]), len(ids)).double()
    del m
    # every row of rsb_llm_hidden_states: max |err| <= 2x transformers fp16's own max |err| on that row (floor: 1 fp16
    # ulp of the row's largest element); the rows shifted by one must be rejected
    err = (rows - h32).abs().max(1).values
    lim = torch.maximum(2 * herr16.max(1).values, _ulp16(h32.abs().max(1).values))
    print(f"pythia-{name} x{layers}: hidden rows max err / bound {float((err / lim).max()):.3f}")
    assert bool((err <= lim).all())
    _must_fail("rows shifted by one", ((rows - torch.roll(h32, 1, 0)).abs().max(1).values <= lim).cpu().numpy())
    torch.cuda.empty_cache()
    e = np.abs(ours - ref)[1:]
    print(f"pythia-{name} x{layers}: max |ours - fp32| {e.max():.3e}, max |HF fp16 - fp32| {err16.max():.3e}")
    assert e.max() <= 2 * err16[1:].max()
    assert np.mean(e) <= 2 * np.mean(err16[1:])


def test_pickle_directory_matches_safetensors(tmp_path):
    from retrieval_scaling_b200.reader import load_reader, B200NeoX
    a = load_reader(F.build_dir(str(tmp_path / "st")))
    b = load_reader(F.build_dir(str(tmp_path / "bin"), pickle=True))
    assert isinstance(a, B200NeoX) and isinstance(b, B200NeoX)
    ids = F.window_ids()[9]
    assert torch.equal(a.nll([ids], [ids])[0], b.nll([ids], [ids])[0])
    m = B200NeoX(F.CONFIG)                                          # strict: the legacy buffers are not unexpected
    assert m.load_state_dict(dict(F.seeded_state_dict(), **F.legacy_buffers())) == []


def test_refusals_and_overflow(model):
    ids = F.window_ids()[5]
    with pytest.raises(ValueError, match="outside the vocabulary"):
        model.nll([[0, 1000]], [[0, 1000]])
    with pytest.raises(NotImplementedError, match="max_position_embeddings"):
        model.nll([np.zeros(2049, np.int64)], [np.zeros(2049, np.int64)])
    from retrieval_scaling_b200.reader import B200NeoX
    sd = F.seeded_state_dict()
    sd["gpt_neox.layers.0.mlp.dense_4h_to_h.bias"] = torch.full_like(sd["gpt_neox.layers.0.mlp.dense_4h_to_h.bias"], 6e4)
    sd["gpt_neox.layers.0.attention.dense.bias"] = torch.full_like(sd["gpt_neox.layers.0.attention.dense.bias"], 6e4)
    m = B200NeoX(F.CONFIG)
    m.load_state_dict(sd)
    with pytest.raises(FloatingPointError):
        m.nll([ids], [ids])


@pytest.mark.parametrize("concate_k", [0, 3])
def test_main_ric_perplexity_end_to_end(tmp_path, concate_k):
    """`ric/main_ric.py --config-name perplexity` with the NeoX fixture reader, against the reference's loop restated on
    the CPU with transformers fp32 (no BOS: Pythia's tokenizer adds none; eos 0 is the masked pad id)."""
    import json
    import re
    import subprocess

    from golden import roberta_fixture as RF
    from retrieval_scaling_b200 import config as C
    from retrieval_scaling_b200 import perplexity as P
    enc = RF.build(str(tmp_path / "enc"))
    reader_dir = F.build_dir(str(tmp_path / "reader"))
    rng = np.random.default_rng(9)
    texts = [" ".join(f"w{i}" for i in rng.integers(1, 1000, n)) for n in (300, 200)]
    words = " ".join(texts).split()
    psg_dir = tmp_path / "passages" / "dom" / "1-shards"
    psg_dir.mkdir(parents=True)
    with open(psg_dir / "raw_passages-0-of-1.jsonl", "w") as f:
        for i in range(150):
            if i % 5 == 0:
                s = int(rng.integers(0, len(words) - 60))
                t = " ".join(words[s:s + 60])
            else:
                t = " ".join(f"w{j}" for j in rng.integers(1, 1000, int(rng.integers(10, 60))))
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
    else:
        eval_data = P.prepare_ppl_eval_data([json.loads(line) for line in open(eval_path)], tok, 128, 64, True)
    contexts, answers, _ = P.build_doc_prompts(eval_data, cfg.evaluation)
    hf = F.hf_model(dtype=torch.float32)
    total, count = 0.0, 0
    for context, answer in zip(contexts, answers):                # src/evaluate_perplexity.py:117-139
        a = tok(answer, return_tensors="pt")["input_ids"]
        c = tok(context, return_tensors="pt")["input_ids"]
        ids = torch.cat((c, a), 1)
        lab = torch.cat((torch.full(c.size(), -100), a), 1)
        lab = torch.where(lab == 0, torch.tensor(-100), lab)        # eos <|endoftext|> = 0 is the pad id
        with torch.no_grad():
            total += hf(ids[:, -2048:], labels=lab[:, -2048:]).loss.item()
        count += 1
    ppl_cpu = float(torch.exp(torch.tensor(total / count)))
    print(f"concate_k {concate_k}: {count} windows, perplexity GPU {ppl_gpu:.4f} CPU fp32 {ppl_cpu:.4f}")
    assert ppl_gpu == pytest.approx(ppl_cpu, rel=1e-3)
