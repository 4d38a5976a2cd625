"""GPU checks of the OLMo / OLMo-2 reader (rsb_llm_create, then rsb_llm_*): per-token NLL against the committed
fp64 golden held to HF bf16's own error, packing and determinism, the attention prologue (clip_qkv clamp, whole-
projection QK-norm, fp32-cos / sin RoPE) per element, the two norms per element, production widths against
transformers, the refusals, the overflow check and `main_ric.py` end to end.  Every per-element comparison also has
to reject a deliberately wrong reference."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import olmo_fixture as F  # noqa: E402
import olmo_oracle as O  # noqa: E402

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


def _round_bound(want, extra):
    """Largest |fp16(want + e) - want| over |e| <= extra: half an fp16 ulp (at the larger magnitude) plus extra."""
    return 0.5 * _ulp16(want.abs() + extra) + extra


def _model(kind, **change):
    from retrieval_scaling_b200.reader import B200Olmo
    cfg = F.config(kind, **change)
    m = B200Olmo(cfg)
    m.load_state_dict(F.seeded_state_dict(cfg))
    return m


@pytest.fixture(scope="module")
def models():
    return {k: _model(k) for k in F.CONFIGS}


def _golden(kind):
    g = np.load(F.GOLDEN)
    cu, nll = g[f"{kind}_cu_seqlens"], g[f"{kind}_nll"].astype(np.float64)
    return F.window_ids(kind), [nll[cu[b]:cu[b + 1]] for b in range(len(cu) - 1)]


@pytest.mark.parametrize("kind", ["olmo", "olmo2"])
def test_nll_against_fp64_golden_within_hf_bf16_precision(models, kind):
    """The OLMo fixture has a tied head and an active clamp; the OLMo-2 fixture GQA 4:1 and rope_theta 5e5."""
    windows, gold = _golden(kind)
    hf = F.hf_model(F.CONFIGS[kind], dtype=torch.bfloat16, attn_implementation="sdpa").cuda()
    bf16 = [F.hf_token_nll(hf, w) for w in windows]
    del hf
    torch.cuda.empty_cache()
    ours = models[kind].nll(windows, windows)
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
    print(f"{kind}: per-token |err| p99: ours {p99_o:.3e}, HF bf16 {p99_b:.3e}; window-mean |err| max: ours "
          f"{max(mean_o):.3e}, HF bf16 {max(mean_b):.3e}")
    assert p99_o <= p99_b
    assert max(mean_o) <= max(mean_b)


@pytest.mark.parametrize("kind", ["olmo", "olmo2"])
def test_packed_equals_one_at_a_time_and_deterministic(models, kind):
    windows, _ = _golden(kind)
    m = models[kind]
    order = [9, 0, 3, 11, 1, 5, 2, 6, 4, 12]
    packed = m.nll([windows[i] for i in order], [windows[i] for i in order])
    again = m.nll([windows[i] for i in order], [windows[i] for i in order], max_tokens=300)
    for i, p, a in zip(order, packed, again):
        assert torch.equal(p, m.nll([windows[i]], [windows[i]])[0])
        assert torch.equal(p, a)


def _powf(x, y):
    """glibc powf, the function the handle's inv_freq is computed with on the host."""
    libm = ctypes.CDLL("libm.so.6")
    libm.powf.restype, libm.powf.argtypes = ctypes.c_float, [ctypes.c_float, ctypes.c_float]
    return libm.powf(x, y)


def _cos_sin(pos, theta):
    """float64 cos / sin [n, 1, 64] of the kernel's fp32 angles fp32(inv_freq[i] * pos)."""
    inv = torch.tensor([np.float32(1) / np.float32(_powf(theta, 2 * i / 128)) for i in range(64)], dtype=torch.float32)
    f = torch.as_tensor(np.asarray(pos), dtype=torch.float32)[:, None] * inv[None, :]
    f = f.double().cuda()
    return f.cos()[:, None], f.sin()[:, None]


def _rope_check(got, xin, near, c, s, name):
    """got [n, h, 128] fp16 against the fp32-cos / sin RoPE of xin [n, h, 128] (the fp16 inputs RoPE read, float64) with
    one rounding; near marks inputs that may sit one fp16 ulp away (a norm's result at a rounding boundary).  A
    reference in Llama's order (fp16 cos / sin, every product and the sum rounded) must be rejected.  Returns the
    worst error / bound."""
    h = 64
    x1, x2 = xin[..., :h], xin[..., h:]
    y = torch.cat((x1 * c - x2 * s, x2 * c + x1 * s), -1)
    # fp32 evaluation: cosf / sinf within 2 fp32 ulps, each product and the sum one fp32 rounding
    d = 2.0 ** -21 * torch.cat((x1.abs() + x2.abs(), x2.abs() + x1.abs()), -1)
    w1, w2 = near[..., :h] * _ulp16(x1), near[..., h:] * _ulp16(x2)
    d = d + torch.cat((w1 * c.abs() + w2 * s.abs(), w2 * c.abs() + w1 * s.abs()), -1)
    bound = _round_bound(y, d)
    err = (got.double() - y).abs()
    assert bool((err <= bound).all()), f"{name}: {int((err > bound).sum())} rotated elements beyond the bound"
    c16, s16 = _r16(c), _r16(s)
    llama = torch.cat((_r16(_r16(x1 * c16) + _r16(-x2 * s16)), _r16(_r16(x2 * c16) + _r16(x1 * s16))), -1)
    _must_fail(f"{name}: Llama's fp16 cos / sin order", ((got.double() - llama).abs() <= bound).cpu().numpy())
    return float((err / bound).max())


@pytest.mark.parametrize("version, heads, kv_heads, theta", [(1, 32, 32, 1e4), (1, 8, 2, 5e5), (2, 32, 8, 5e5),
                                                              (2, 40, 40, 5e5), (2, 16, 4, 1e4)])
def test_attention_prologue_per_element(version, heads, kv_heads, theta):
    """rsb_llm_attention on an OLMo handle runs layer 0's prologue in place.  Windows of one token isolate the clamp
    and the norm (RoPE at position 0 is the identity); every row checks RoPE.  OLMo: the clamp is bit-exact on Q, K
    and V.  OLMo-2: each Q / K element is within half an fp16 ulp plus the fp32 term of the float64 whole-projection
    RMSNorm, V is untouched, and a per-head norm is rejected."""
    from retrieval_scaling_b200 import _lib
    from retrieval_scaling_b200.reader import B200Olmo
    kind, clip = ("olmo", 3.0) if version == 1 else ("olmo2", None)
    H, KV = heads * 128, kv_heads * 128
    cfg = F.config(kind, hidden_size=H, num_attention_heads=heads, num_key_value_heads=kv_heads, intermediate_size=128,
                   num_hidden_layers=1, rope_theta=theta, max_position_embeddings=4096, clip_qkv=clip)
    m = B200Olmo(cfg)
    lens = [1] * 48 + [15, 17, 0, 64, 65, 129, 1000, 4096]
    cu = np.concatenate([[0], np.cumsum(lens)])
    n = int(cu[-1])
    T = n + 5                                                      # rows past cu[B] stay untouched
    g = torch.Generator(device="cuda").manual_seed(heads * 100 + version)
    qkv0 = (torch.randn(T, H + 2 * KV, generator=g, device="cuda") * 2.0).half()
    qkv0[::11] *= 4                                                # rows of several magnitudes
    ctx = torch.empty((T, H), dtype=torch.float16, device="cuda")
    qn = kn = None
    eps = 1e-5 if version == 1 else float(cfg["rms_norm_eps"])
    if version == 2:
        qkv = qkv0.clone()
        with pytest.raises(_lib.RsbError, match="q_norm"):           # RSB_ERR_STATE before layer 0's norms are loaded
            m.attention(qkv, _i32(cu), max(lens), ctx)
        qn = (1.0 + 0.3 * torch.randn(H, generator=g, device="cuda")).half()
        kn = (1.0 + 0.3 * torch.randn(KV, generator=g, device="cuda")).half()
        m.load_weight("model.layers.0.self_attn.q_norm.weight", qn)
        m.load_weight("model.layers.0.self_attn.k_norm.weight", kn)
    qkv = qkv0.clone()
    m.attention(qkv, _i32(cu), max(lens), ctx)
    torch.cuda.synchronize()
    assert torch.equal(qkv[n:], qkv0[n:])
    pos = np.concatenate([np.arange(L) for L in lens])
    first = torch.as_tensor(pos == 0, device="cuda")
    x = qkv0[:n].double()
    q, k, v = x[:, :H], x[:, H:H + KV], x[:, H + KV:]
    got_qk, got_v = qkv[:n, :H + KV], qkv[:n, H + KV:]
    if version == 1:
        cl = [t.clamp(-clip, clip) for t in (q, k, v)]
        assert float((v.abs() > clip).double().mean()) > 0.01      # the clamp acts
        assert torch.equal(got_v, cl[2].half())                    # V: the clamp alone, bit for bit
        assert torch.equal(got_qk[first], torch.cat(cl[:2], 1)[first].half())   # position 0: the clamp alone
        xin = torch.cat(cl[:2], 1)                                  # exact fp16 values
        near = torch.zeros_like(xin)
        _must_fail("no clamp", (got_v == v.half()).cpu().numpy())
    else:
        assert torch.equal(got_v, qkv0[:n, H + KV:])               # OLMo-2 leaves V as it is
        nq, nk = O.rms_norm(q, qn.double(), eps), O.rms_norm(k, kn.double(), eps)
        want = torch.cat((nq, nk), 1)
        extra = 64 * 2.0 ** -24 * want.abs()                       # the fp32 statistics, rsqrt and two products
        bound = _round_bound(want, extra)
        err = (got_qk[first].double() - want[first]).abs()
        assert bool((err <= bound[first]).all()), f"{int((err > bound[first]).sum())} normed elements beyond the bound"
        print(f"v2 {heads}:{kv_heads}: QK-norm |err| / bound max {float((err / bound[first]).max()):.3f}")
        ph = torch.cat((O.rms_norm(q.view(n, heads, 128), qn.double().view(heads, 128), eps).view(n, H),
                        O.rms_norm(k.view(n, kv_heads, 128), kn.double().view(kv_heads, 128), eps).view(n, KV)), 1)
        _must_fail("per-head norm", ((got_qk[first].double() - ph[first]).abs() <= bound[first]).cpu().numpy())
        xin = _r16(want)
        near = (_r16(want - extra) != _r16(want + extra)).double()
    c, s = _cos_sin(pos, theta)
    nh = heads + kv_heads
    worst = _rope_check(got_qk.view(n, nh, 128), xin.view(n, nh, 128), near.view(n, nh, 128), c, s,
                        f"v{version} {heads}:{kv_heads}")
    print(f"v{version} {heads}:{kv_heads} theta {theta:g}: RoPE |err| / bound max {worst:.3f}")


def _ln_ref(x, eps):
    """float64 OlmoLayerNorm of fp16 rows and the fp32 evaluation error a rounded result may carry besides its final
    rounding (the statistics' sums and rsqrt; see test_gpu_reader_neox._ln_ref with unit weight and zero bias)."""
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt((xd - mean).pow(2).mean(-1, keepdim=True) + eps)
    y = (xd - mean) * rstd
    return y, 2.0 ** -24 * (32 * y.abs() + 64 * rstd * xd.abs().mean(-1, keepdim=True))


@pytest.mark.parametrize("hidden", [2048, 4096, 5120, 8192])
def test_norms_per_element(hidden):
    """The two norm steps of the forward on the same fp16 inputs.
    OLMo: rsb_llm_layernorm with unit weight and zero bias, as the forward runs it, all rows and gathered rows.
    OLMo-2: rsb_llm_olmo2_norm (rms_post_kernel) in its two modes, the post-norm add x += norm(a) and the gathered
    final norm.  Each normed element is within half an fp16 ulp of float64 plus the fp32 evaluation term; each sum is
    fp16(x + normed).  Rejected: LlamaRMSNorm's two roundings (fp16 before the weight) and the pre-norm placement
    x + a (the block output added without its norm)."""
    from retrieval_scaling_b200 import _lib
    L = _lib.lib()
    g = torch.Generator(device="cuda").manual_seed(hidden)
    n, eps = 300, 1e-6
    rnd = lambda *sh, std=1.0, mu=0.0: (torch.randn(*sh, generator=g, device="cuda") * std + mu).half()   # noqa: E731
    x0, a = rnd(n, hidden, std=3.0, mu=1.0), rnd(n, hidden, std=2.0)
    x0[::7] *= 20
    a[::5] *= 30                                                   # rows of several magnitudes
    w = rnd(hidden, std=0.5, mu=1.0)
    ptr = lambda t: ctypes.c_void_p(t.data_ptr()) if t is not None else None   # noqa: E731
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    rows = torch.randperm(n, generator=g, device="cuda")[:n // 2].int()
    worst = 0.0

    # OLMo's LayerNorm
    ones, zeros = torch.ones(hidden, dtype=torch.float16, device="cuda"), torch.zeros(hidden, dtype=torch.float16, device="cuda")
    for rsel in (None, rows):
        m = n if rsel is None else len(rsel)
        out = torch.full((m, hidden), 7.0, dtype=torch.float16, device="cuda")
        x = x0.clone()
        rc = L.rsb_llm_layernorm(hidden, ctypes.c_float(1e-5), ptr(x), None, ptr(rsel), m, ptr(ones), ptr(zeros), None,
                                 None, ptr(out), None, st)
        assert rc == _lib.RSB_OK, L.rsb_llm_last_error()
        torch.cuda.synchronize()
        assert torch.equal(x, x0)
        want, extra = _ln_ref(x0 if rsel is None else x0[rsel.long()], 1e-5)
        bound = _round_bound(want, extra)
        err = (out.double() - want).abs()
        assert bool((err <= bound).all()), f"LayerNorm: {int((err > bound).sum())} elements beyond the bound"
        worst = max(worst, float((err / bound).max()))

    # OLMo-2's RMSNorm
    def rms(v, order="olmo2"):
        vd = v.double()
        r = 1.0 / torch.sqrt(vd.pow(2).mean(-1, keepdim=True) + eps)
        if order == "llama":
            return _r16(w.double() * _r16(vd * r))
        return w.double() * vd * r

    def extra_of(want):
        return 64 * 2.0 ** -24 * want.abs()

    x = x0.clone()
    rc = L.rsb_llm_olmo2_norm(hidden, ctypes.c_float(eps), ptr(x), ptr(a), None, n, ptr(w), None, st)   # x += norm(a)
    assert rc == _lib.RSB_OK, L.rsb_llm_last_error()
    torch.cuda.synchronize()
    nw = rms(a)
    ne = extra_of(nw)
    # fp16(x + n16) with n16 within the rounding bound of nw: |got - (x + nw)| <= that bound + half an ulp of the sum
    s = x0.double() + nw
    bound = _round_bound(s, _round_bound(nw, ne))
    err = (x.double() - s).abs()
    assert bool((err <= bound).all()), f"post-norm add: {int((err > bound).sum())} elements beyond the bound"
    worst = max(worst, float((err / bound).max()))
    _must_fail("pre-norm placement (x + a)", ((x.double() - (x0.double() + a.double())).abs() <= bound).cpu().numpy())

    out = torch.full((len(rows), hidden), 7.0, dtype=torch.float16, device="cuda")
    xs = x.clone()
    rc = L.rsb_llm_olmo2_norm(hidden, ctypes.c_float(eps), ptr(xs), None, ptr(rows), len(rows), ptr(w), ptr(out), st)
    assert rc == _lib.RSB_OK, L.rsb_llm_last_error()
    torch.cuda.synchronize()
    assert torch.equal(xs, x)
    want = rms(x[rows.long()])
    bound = _round_bound(want, extra_of(want))
    err = (out.double() - want).abs()
    assert bool((err <= bound).all()), f"final RMSNorm: {int((err > bound).sum())} elements beyond the bound"
    worst = max(worst, float((err / bound).max()))
    _must_fail("LlamaRMSNorm's order", ((out.double() - rms(x[rows.long()], "llama")).abs() <= bound).cpu().numpy())
    print(f"hidden {hidden}: norms |err| / bound max {worst:.3f}")


def _hf_err(cfg, sd, ids):
    """(NLL fp64 of transformers fp32, |fp16 - fp32| per token, pre-final-norm rows fp64 of fp32, |fp16 - fp32| per
    row element) on the GPU."""
    out, rows = {}, {}
    for dt in (torch.float32, torch.float16):
        hf = F.hf_model(cfg, dtype=dt, sd=sd).cuda()
        cap = []
        hk = hf.model.norm.register_forward_hook(lambda mod, a, o: cap.append(a[0][0].double()))
        out[dt] = F.hf_token_nll(hf, ids)
        hk.remove()
        rows[dt] = cap[0]
        del hf
        torch.cuda.empty_cache()
    return (out[torch.float32], np.abs(out[torch.float16] - out[torch.float32]), rows[torch.float32],
            (rows[torch.float16] - rows[torch.float32]).abs())


# (model_type, hidden, heads, kv heads, intermediate, extra config) at published widths
WIDTHS = {"olmo-1b": ("olmo", 2048, 16, 16, 8192, dict(tie_word_embeddings=True, clip_qkv=None)),
          "olmo-7b-0424": ("olmo", 4096, 32, 32, 11008, dict(tie_word_embeddings=False, clip_qkv=8.0)),
          "olmo2-7b": ("olmo2", 4096, 32, 32, 11008, dict(rms_norm_eps=1e-6)),
          "olmo2-32b-gqa": ("olmo2", 5120, 40, 8, 27648, dict(rms_norm_eps=1e-6))}


@pytest.mark.parametrize("name, layers", [("olmo-1b", 1), ("olmo-1b", 2), ("olmo-7b-0424", 1), ("olmo2-7b", 1),
                                          ("olmo2-7b", 2), ("olmo2-32b-gqa", 1)])
def test_rows_and_nll_at_production_width(name, layers):
    """One 700-token window at a published OLMo width (vocabulary 50304) against transformers fp32 on the device: every
    hidden row before the final norm, and the NLL (worst and mean token), within twice transformers fp16's error."""
    from retrieval_scaling_b200.reader import B200Olmo
    kind, H, nh, kv, I, extra = WIDTHS[name]
    cfg = F.config(kind, hidden_size=H, num_attention_heads=nh, num_key_value_heads=kv, intermediate_size=I,
                   num_hidden_layers=layers, vocab_size=50304, **extra)
    sd = F.seeded_state_dict(cfg, seed=H + layers)
    ids = np.random.default_rng(layers).integers(0, 50304, 700)
    ref, err16, h32, herr16 = _hf_err(cfg, sd, ids)
    m = B200Olmo(cfg)
    m.load_state_dict(sd)
    ours = m.nll([ids], [ids])[0].numpy().astype(np.float64)
    rows = m.hidden_states(_i32(ids), _i32([0, len(ids)]), len(ids)).double()
    del m
    err = (rows - h32).abs().max(1).values
    lim = torch.maximum(2 * herr16.max(1).values, _ulp16(h32.abs().max(1).values))
    print(f"{name} x{layers}: hidden rows max err / bound {float((err / lim).max()):.3f}")
    assert bool((err <= lim).all())
    _must_fail("rows shifted by one", ((rows - torch.roll(h32, 1, 0)).abs().max(1).values <= lim).cpu().numpy())
    torch.cuda.empty_cache()
    e = np.abs(ours - ref)[1:]
    print(f"{name} x{layers}: max |ours - fp32| {e.max():.3e}, max |HF fp16 - fp32| {err16.max():.3e}")
    assert e.max() <= 2 * err16[1:].max()
    assert np.mean(e) <= 2 * np.mean(err16[1:])


@pytest.mark.parametrize("kind", ["olmo", "olmo2"])
def test_refusals_and_overflow(models, kind):
    from retrieval_scaling_b200.reader import B200Olmo
    m = models[kind]
    with pytest.raises(ValueError, match="outside the vocabulary"):
        m.nll([[0, 1000]], [[0, 1000]])
    with pytest.raises(NotImplementedError, match="max_position_embeddings"):
        m.nll([np.zeros(2049, np.int64)], [np.zeros(2049, np.int64)])
    bare = B200Olmo(F.CONFIGS[kind])
    assert bare.missing_keys()
    with pytest.raises(Exception, match="not loaded"):
        bare.nll([[1, 2, 3]], [[1, 2, 3]])
    ids = F.window_ids(kind)[5]
    sd = F.seeded_state_dict(F.CONFIGS[kind])
    sd["model.layers.0.mlp.down_proj.weight"] = torch.full_like(sd["model.layers.0.mlp.down_proj.weight"], 6e4)
    bad = B200Olmo(F.CONFIGS[kind])
    bad.load_state_dict(sd)
    with pytest.raises(FloatingPointError):
        bad.nll([ids], [ids])


def test_tied_head_reads_the_embedding(models):
    """The OLMo fixture ties its head: it needs no lm_head.weight, its NLL differs from the same weights with an untied
    head, and a second handle loaded from the same state dict reproduces it bit for bit."""
    m = models["olmo"]
    assert "lm_head.weight" not in m.missing_keys() and F.CONFIGS["olmo"]["tie_word_embeddings"]
    ids = F.window_ids("olmo")[9]
    before = m.nll([ids], [ids])[0]
    untied = _model("olmo", tie_word_embeddings=False)
    assert not torch.equal(untied.nll([ids], [ids])[0], before)
    sd = F.seeded_state_dict(F.CONFIGS["olmo"])
    from retrieval_scaling_b200.reader import B200Olmo
    m2 = B200Olmo(F.CONFIGS["olmo"])
    m2.load_state_dict(sd)
    assert torch.equal(m2.nll([ids], [ids])[0], before)


@pytest.mark.parametrize("concate_k", [0, 3])
def test_main_ric_perplexity_end_to_end(tmp_path, concate_k):
    """`ric/main_ric.py --config-name perplexity` with the OLMo-2 fixture reader, against the reference's loop restated
    on the CPU with transformers fp32 (no BOS: OLMo's tokenizers add none; eos 0 is the masked pad id)."""
    import json
    import re
    import subprocess

    from golden import roberta_fixture as RF
    from retrieval_scaling_b200 import config as C
    from retrieval_scaling_b200 import perplexity as P
    cfg2 = F.CONFIGS["olmo2"]
    enc = RF.build(str(tmp_path / "enc"))
    reader_dir = F.build_dir(str(tmp_path / "reader"), cfg2)
    tok = F.tokenizer()
    assert tok("w5 w6")["input_ids"] == [5, 6]                    # no BOS is added
    rng = np.random.default_rng(9)
    texts = [" ".join(f"w{i}" for i in rng.integers(2, 1000, n)) for n in (300, 200)]
    words = " ".join(texts).split()
    psg_dir = tmp_path / "passages" / "dom" / "1-shards"
    psg_dir.mkdir(parents=True)
    with open(psg_dir / "raw_passages-0-of-1.jsonl", "w") as f:
        for i in range(150):
            if i % 5 == 0:
                s = int(rng.integers(0, len(words) - 60))
                t = " ".join(words[s:s + 60])
            else:
                t = " ".join(f"w{j}" for j in rng.integers(2, 1000, int(rng.integers(10, 60))))
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
    if concate_k:
        from retrieval_scaling_b200.search import get_merged_search_output_path
        eval_data = [json.loads(line) for line in open(get_merged_search_output_path(cfg))]
    else:
        eval_data = P.prepare_ppl_eval_data([json.loads(line) for line in open(eval_path)], tok, 128, 64, True)
    contexts, answers, _ = P.build_doc_prompts(eval_data, cfg.evaluation)
    hf = F.hf_model(cfg2, dtype=torch.float32)
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
