"""GPU checks of the readers in bf16 (`load_reader(..., dtype=torch.bfloat16)`, `model.lm_dtype=bfloat16`): the four
fp64 goldens held to 1.5x the error of transformers' own bf16 forward (both sides round to bf16 at the same points),
the fp16 overflow fixture evaluated, the attention prologues bit for bit against torch's bf16 operation sequence,
attention per element, hidden rows at published widths, packing, and `main_ric.py` perplexity end to end against
transformers bf16 sdpa, the reference's configuration."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import llama_fixture as LF  # noqa: E402
import neox_fixture as NF  # noqa: E402
import olmo_fixture as OF  # noqa: E402

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
# librsb bf16 against HF bf16 sdpa: both round to bf16 at the same points, in different orders of summation
RATIO = 1.5


def _i32(a):
    return torch.as_tensor(np.asarray(a), dtype=torch.int32, device="cuda")


def _ulpb(x):
    """Spacing of bf16 at |x| (float64)."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -126)))
    return torch.exp2(e.clamp_min(-126) - 7)


def _reader(cls_name, cfg, sd):
    from retrieval_scaling_b200 import reader
    m = getattr(reader, cls_name)(cfg, dtype=BF)
    m.load_state_dict(sd)
    return m


def _golden_cases():
    g = np.load(LF.GOLDEN)
    cu = g["cu_seqlens"]
    llama = ([g["ids"][cu[b]:cu[b + 1]] for b in range(len(cu) - 1)], [g["nll"][cu[b]:cu[b + 1]] for b in range(len(cu) - 1)])
    g = np.load(NF.GOLDEN)
    cu = g["cu_seqlens"]
    neox = ([g["ids"][cu[b]:cu[b + 1]] for b in range(len(cu) - 1)], [g["nll"][cu[b]:cu[b + 1]] for b in range(len(cu) - 1)])
    g = np.load(OF.GOLDEN)
    olmo = {}
    for k in ("olmo", "olmo2"):
        cu, nll = g[f"{k}_cu_seqlens"], g[f"{k}_nll"].astype(np.float64)
        olmo[k] = (OF.window_ids(k), [nll[cu[b]:cu[b + 1]] for b in range(len(cu) - 1)])
    return {"llama": ("B200Llama", LF, LF.CONFIG, llama), "neox": ("B200NeoX", NF, NF.CONFIG, neox),
            "olmo": ("B200Olmo", OF, OF.CONFIGS["olmo"], olmo["olmo"]),
            "olmo2": ("B200Olmo", OF, OF.CONFIGS["olmo2"], olmo["olmo2"])}


def _fixture_sd(FX, cfg):
    return FX.seeded_state_dict(cfg) if FX is OF else FX.seeded_state_dict()


def _hf(FX, cfg, dtype, **kw):
    return (FX.hf_model(cfg, dtype=dtype, **kw) if FX is OF else FX.hf_model(dtype=dtype, **kw)).cuda()


@pytest.mark.parametrize("kind", ["llama", "neox", "olmo", "olmo2"])
def test_golden_within_hf_bf16_precision(kind):
    """Per-token p99 and worst window-mean error against the fp64 golden: at most 1.5x HF bf16 sdpa's on the same
    windows; packed equals one window at a time, bit for bit; two runs are bit-identical."""
    cls, FX, cfg, (windows, gold) = _golden_cases()[kind]
    hf = _hf(FX, cfg, BF, attn_implementation="sdpa")
    hf_nll = [FX.hf_token_nll(hf, w) for w in windows]
    del hf
    torch.cuda.empty_cache()
    m = _reader(cls, cfg, _fixture_sd(FX, cfg))
    ours = m.nll(windows, windows)
    e_o, e_b, m_o, m_b = [], [], [], []
    for w, o, g, b in zip(windows, ours, gold, hf_nll):
        o = o.numpy().astype(np.float64)
        assert np.all(np.isfinite(o)) and o[0] == 0.0
        if len(w) < 2:
            continue
        e_o.append(np.abs(o[1:] - g[1:]))
        e_b.append(np.abs(b[1:] - g[1:]))
        m_o.append(abs(o[1:].mean() - g[1:].mean()))
        m_b.append(abs(b[1:].mean() - g[1:].mean()))
    p_o, p_b = np.percentile(np.concatenate(e_o), 99), np.percentile(np.concatenate(e_b), 99)
    print(f"{kind} bf16: per-token |err| p99 ours {p_o:.3e} HF bf16 {p_b:.3e} ({p_o / p_b:.2f}x); worst window mean "
          f"ours {max(m_o):.3e} HF bf16 {max(m_b):.3e} ({max(m_o) / max(m_b):.2f}x)")
    assert p_o <= RATIO * p_b
    assert max(m_o) <= RATIO * max(m_b)
    order = list(range(len(windows)))[::-1]
    packed = m.nll([windows[i] for i in order], [windows[i] for i in order], max_tokens=700)
    for i, p in zip(order, packed):
        assert torch.equal(p, ours[i])
        if len(windows[i]) <= 130:
            assert torch.equal(p, m.nll([windows[i]], [windows[i]])[0])


def test_label_masks_do_not_change_other_tokens():
    cls, FX, cfg, (windows, _) = _golden_cases()["llama"]
    m = _reader(cls, cfg, _fixture_sd(FX, cfg))
    rng = np.random.default_rng(3)
    labels = []
    for w in windows:
        lb = np.array(w, np.int64)
        lb[rng.random(len(w)) < 0.5] = -100
        labels.append(lb)
    full, masked = m.nll(windows, windows), m.nll(windows, labels, max_tokens=300)
    for f, mk, lb in zip(full, masked, labels):
        scored = np.zeros(len(lb), bool)
        scored[1:] = lb[1:] != -100
        assert torch.equal(mk[scored], f[scored]) and torch.all(mk[~scored] == 0)


def test_overflow_raises_in_fp16_and_evaluates_in_bf16():
    """Embedding 65000 and o_proj x 1e4: the fp16 residual stream passes 65504; in bf16 the same weights give a finite
    NLL within the bf16 tolerance of the float64 oracle.  A final-norm weight of 1e5 loads in bf16, not in fp16."""
    import llama_oracle as O
    from retrieval_scaling_b200.reader import B200Llama
    cfg1 = dict(LF.CONFIG, num_hidden_layers=1)
    sd = LF.seeded_state_dict(cfg1)
    sd["model.embed_tokens.weight"].fill_(65000.0)
    sd["model.layers.0.self_attn.o_proj.weight"] *= 1e4
    hot16 = B200Llama(cfg1)
    hot16.load_state_dict(sd)
    with pytest.raises(FloatingPointError, match="overflow"):
        hot16.nll([[5, 6, 7]], [[5, 6, 7]])
    del hot16
    hot = B200Llama(cfg1, dtype="bfloat16")
    hot.load_state_dict(sd)
    rng = np.random.default_rng(4)
    windows = [rng.integers(0, cfg1["vocab_size"], S) for S in (3, 64, 300)]
    hf = LF.hf_model(cfg1, dtype=BF, attn_implementation="sdpa")
    hf.load_state_dict(sd, strict=False)
    hf = hf.to(BF).cuda()
    for w, o in zip(windows, hot.nll(windows, windows)):
        o = o.numpy().astype(np.float64)[1:]
        ref = O.token_nll(sd, cfg1, w)[1:]
        b = LF.hf_token_nll(hf, w)[1:]
        assert np.all(np.isfinite(o))
        print(f"overflow fixture, {len(w)} tokens: max |err| ours {np.abs(o - ref).max():.3e} HF bf16 "
              f"{np.abs(b - ref).max():.3e}; window mean ours {abs(o.mean() - ref.mean()):.3e} HF bf16 "
              f"{abs(b.mean() - ref.mean()):.3e}")
        assert abs(o.mean() - ref.mean()) <= max(RATIO * abs(b.mean() - ref.mean()), 0.05 * max(1.0, abs(ref.mean())))
    part16, part = B200Llama(dict(LF.CONFIG, num_hidden_layers=1)), B200Llama(dict(LF.CONFIG, num_hidden_layers=1), dtype=BF)
    big = torch.full((512,), 1e5, dtype=BF)
    with pytest.raises(ValueError, match="finite in float16"):
        part16.load_weight("model.norm.weight", big)
    assert part.load_weight("model.norm.weight", big)


def test_dtype_refusals():
    from retrieval_scaling_b200.reader import B200Llama
    m = B200Llama(dict(LF.CONFIG, num_hidden_layers=1), dtype=BF)
    T, H = 8, 512
    with pytest.raises(ValueError, match="bfloat16"):
        m.attention(torch.zeros(T, H + 2 * 128, dtype=torch.float16, device="cuda"), _i32([0, T]), T,
                    torch.zeros(T, H, dtype=BF, device="cuda"))
    ids = _i32([1, 2, 3])
    m.load_state_dict(LF.seeded_state_dict(dict(LF.CONFIG, num_hidden_layers=1)))
    assert m.hidden_states(ids, _i32([0, 3]), 3).dtype == BF


def _powf(x, y):
    libm = ctypes.CDLL("libm.so.6")
    libm.powf.restype, libm.powf.argtypes = ctypes.c_float, [ctypes.c_float, ctypes.c_float]
    return libm.powf(x, y)


def _angles(pos, theta, rot):
    """fp32 angles fp32(inv_freq[i] * pos) [n, 1, rot / 2] with the handle's host-side inv_freq, and the float64
    cos / sin of them."""
    inv = torch.tensor([np.float32(1) / np.float32(_powf(theta, 2 * i / rot)) for i in range(rot // 2)],
                       dtype=torch.float32, device="cuda")
    f = torch.as_tensor(np.asarray(pos), dtype=torch.float32, device="cuda")[:, None] * inv[None, :]
    return f[:, None]


def _at_boundary(v64):
    """cos / sin values whose bf16 rounding a 2-fp32-ulp change of the fp32 value can flip."""
    d = v64.abs() * 2.0 ** -22
    return (v64 - d).to(BF) != (v64 + d).to(BF)


def _rope_bf16(x, f, rot):
    """HF's bf16 rotate_half RoPE on dims [0, rot) of x [n, h, d] bf16: cos / sin rounded to bf16, then every product
    and the sum rounded to bf16 (torch's bf16 arithmetic).  Also the mask of elements whose cos / sin sits at a bf16
    rounding boundary."""
    h = rot // 2
    c, s = f.cos().to(BF), f.sin().to(BF)
    x1, x2 = x[..., :h], x[..., h:rot]
    y = x.clone()
    y[..., :h] = x1 * c + (-x2) * s
    y[..., h:rot] = x2 * c + x1 * s
    fd = f.double()
    b = (_at_boundary(fd.cos()) | _at_boundary(fd.sin())).expand(x1.shape)
    near = torch.zeros(x.shape, dtype=torch.bool, device=x.device)
    near[..., :h] = b
    near[..., h:rot] = b
    return y, near


def _rope_check(got, want, near, name):
    bad = got.view(torch.int16) != want.view(torch.int16)
    assert not bool((bad & ~near).any()), f"{name}: {int((bad & ~near).sum())} elements differ away from a boundary"
    print(f"{name}: bit-equal except {int(bad.sum())} of {bad.numel()} elements at a cos / sin rounding boundary "
          f"({int(near.sum())} such elements)")


def _attention_ref_bf16(qkv, cu, heads, kv_heads, d):
    """ctx float64 and a per-element bound for rotated bf16 rows qkv [T, (heads + 2 kv_heads) d]: the fp32 terms of
    oracle.attention_oracle.causal_attention, with P rounded to bf16 (relative 2^-8) and the output rounded to bf16."""
    T, hid, kvd = int(cu[-1]), heads * d, kv_heads * d
    out = torch.zeros((T, hid), dtype=torch.float64, device="cuda")
    bnd = torch.zeros_like(out)
    g = heads // kv_heads
    for b in range(len(cu) - 1):
        t0, S = int(cu[b]), int(cu[b + 1] - cu[b])
        if S == 0:
            continue
        x = qkv[t0:t0 + S].double()
        q = x[:, :hid].view(S, heads, d).transpose(0, 1)
        k = x[:, hid:hid + kvd].view(S, kv_heads, d).transpose(0, 1).repeat_interleave(g, 0)
        v = x[:, hid + kvd:].view(S, kv_heads, d).transpose(0, 1).repeat_interleave(g, 0)
        sc = q @ k.transpose(1, 2) / d ** 0.5
        i = torch.arange(S, device="cuda")
        vis = i[None, :] <= i[:, None]
        p = torch.softmax(sc.masked_fill(~vis, -torch.inf), dim=-1)
        ctx = p @ v
        E = p @ v.abs()
        svis = vis.sum(-1).double()[None, :, None]
        qk = (q.abs() @ k.abs().transpose(1, 2)).masked_fill(~vis, 0).amax(-1, keepdim=True) / d ** 0.5
        smax = sc.abs().masked_fill(~vis, 0).amax(-1, keepdim=True)
        a = 2.0 ** -20 + 2.0 ** -22 * smax + svis * 2.0 ** -24 + d * 2.0 ** -23 * qk
        vmax = v.abs().amax(1, keepdim=True)
        bd = (2.0 ** -8 + (svis + 32) * 2.0 ** -24) * E + svis * 2.0 ** -25 * vmax + 2 * a * (E + ctx.abs()) \
            + 0.5 * _ulpb(ctx)
        out[t0:t0 + S] = ctx.transpose(0, 1).reshape(S, hid)
        bnd[t0:t0 + S] = bd.transpose(0, 1).reshape(S, hid)
    return out, bnd


LENS = [1, 15, 16, 17, 0, 63, 64, 65, 129, 300, 1024]


@pytest.mark.parametrize("family, heads, kv_heads, d", [("llama", 8, 8, 128), ("llama", 8, 2, 128),
                                                        ("neox", 8, 8, 64), ("neox", 8, 8, 80), ("neox", 4, 4, 256)])
def test_rope_and_attention(family, heads, kv_heads, d):
    """Llama RoPE (all 128 dims) or GPT-NeoX partial RoPE (d / 4 dims: 16, 20, 64) bit-equal to torch's bf16 sequence,
    then attention per element within the bf16 bound."""
    from retrieval_scaling_b200 import reader
    H = heads * d
    if family == "llama":
        cfg = dict(LF.CONFIG, hidden_size=H, num_attention_heads=heads, num_key_value_heads=kv_heads,
                   num_hidden_layers=1, max_position_embeddings=4096, rope_theta=10000.0)
        m, rot, theta = reader.B200Llama(cfg, dtype=BF), 128, 10000.0
    else:
        cfg = dict(NF.CONFIG, hidden_size=H, num_attention_heads=heads, intermediate_size=512, num_hidden_layers=1,
                   max_position_embeddings=4096, rotary_pct=0.25)
        m = reader.B200NeoX(cfg, dtype=BF)
        rot, theta = m.geom["rotary_ndims"], m.geom["rotary_emb_base"]
    cu = np.concatenate([[0], np.cumsum(LENS)])
    n = int(cu[-1])
    T = n + 3
    g = torch.Generator(device="cuda").manual_seed(d * 10 + kv_heads)
    qkv0 = (torch.randn(T, H + 2 * kv_heads * d, generator=g, device="cuda") * 2.0).to(BF)
    qkv0[::13] *= 8
    qkv = qkv0.clone()
    ctx = torch.zeros((T, H), dtype=BF, device="cuda")
    m.attention(qkv, _i32(cu), max(LENS), ctx)
    torch.cuda.synchronize()
    assert torch.equal(qkv[n:], qkv0[n:]) and torch.equal(qkv[:n, (heads + kv_heads) * d:], qkv0[:n, (heads + kv_heads) * d:])
    pos = np.concatenate([np.arange(L) for L in LENS])
    nh = heads + kv_heads
    want, near = _rope_bf16(qkv0[:n, :nh * d].view(n, nh, d), _angles(pos, theta, rot), rot)
    _rope_check(qkv[:n, :nh * d].view(n, nh, d), want, near, f"{family} d {d} rot {rot}")
    ref, bound = _attention_ref_bf16(qkv, cu, heads, kv_heads, d)
    err = (ctx[:n].double() - ref).abs()
    print(f"{family} {heads}:{kv_heads} d {d}: attention |err| / bound max {float((err / bound).max()):.3f}")
    assert bool((err <= bound).all())


@pytest.mark.parametrize("version", [1, 2])
def test_olmo_prologue(version):
    """OLMo: the clip_qkv clamp is torch's bf16 clamp_ (V bit-equal), then RoPE with fp32 cos / sin and one rounding,
    bit-equal to torch's sequence.  OLMo-2: the whole-projection QK-norm at position 0 within 1 bf16 ulp of torch's
    Olmo2RMSNorm (fp32 statistics summed in another order)."""
    from retrieval_scaling_b200.reader import B200Olmo
    heads, kv = 8, 2
    H, KV = heads * 128, kv * 128
    kind = "olmo" if version == 1 else "olmo2"
    cfg = OF.config(kind, hidden_size=H, num_attention_heads=heads, num_key_value_heads=kv, intermediate_size=128,
                    num_hidden_layers=1, max_position_embeddings=4096, clip_qkv=3.0 if version == 1 else None)
    m = B200Olmo(cfg, dtype=BF)
    lens = [1] * 16 + LENS
    cu = np.concatenate([[0], np.cumsum(lens)])
    n = int(cu[-1])
    g = torch.Generator(device="cuda").manual_seed(version)
    qkv0 = (torch.randn(n, H + 2 * KV, generator=g, device="cuda") * 2.0).to(BF)
    ctx = torch.zeros((n, H), dtype=BF, device="cuda")
    pos = np.concatenate([np.arange(L) for L in lens])
    f = _angles(pos, float(cfg["rope_theta"]), 128)
    qkv = qkv0.clone()
    if version == 1:
        m.attention(qkv, _i32(cu), max(lens), ctx)
        torch.cuda.synchronize()
        cl = qkv0.clone().clamp_(min=-3.0, max=3.0)                  # torch's clamp_ on the bf16 tensor
        assert float((qkv0.abs() > 3).double().mean()) > 0.01
        assert torch.equal(qkv[:, H + KV:], cl[:, H + KV:])
        x = cl[:, :H + KV].view(n, heads + kv, 128)
        c, s = f.cos(), f.sin()
        x1, x2 = x[..., :64].float(), x[..., 64:].float()
        want = torch.cat((x1 * c + (-x2) * s, x2 * c + x1 * s), -1).to(BF)   # OLMo's apply_rotary_pos_emb
        got = qkv[:, :H + KV].view(n, heads + kv, 128)
        bad = got.view(torch.int16) != want.view(torch.int16)
        # torch's fp32 cos / sin and the kernel's cosf / sinf may differ in the last fp32 bit, which can move a result
        # across a bf16 rounding boundary: such an element is one bf16 ulp away, and rare
        off = (got.double() - want.double()).abs()
        print(f"olmo clamp + fp32 RoPE: bit-equal except {int(bad.sum())} of {bad.numel()} elements")
        assert bool((off[bad] <= _ulpb(want.double())[bad]).all()) and int(bad.sum()) <= 1e-4 * bad.numel()
    else:
        qn = (1.0 + 0.3 * torch.randn(H, generator=g, device="cuda")).to(BF)
        kn = (1.0 + 0.3 * torch.randn(KV, generator=g, device="cuda")).to(BF)
        m.load_weight("model.layers.0.self_attn.q_norm.weight", qn)
        m.load_weight("model.layers.0.self_attn.k_norm.weight", kn)
        m.attention(qkv, _i32(cu), max(lens), ctx)
        torch.cuda.synchronize()
        assert torch.equal(qkv[:, H + KV:], qkv0[:, H + KV:])

        def olmo2_norm(x, w):
            xf = x.float()
            return (w.float() * (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + cfg["rms_norm_eps"]))).to(BF)
        want = torch.cat((olmo2_norm(qkv0[:, :H], qn), olmo2_norm(qkv0[:, H:H + KV], kn)), 1)
        first = torch.as_tensor(pos == 0, device="cuda")
        got = qkv[first, :H + KV].double()
        err = (got - want[first].double()).abs()
        print(f"olmo2 QK-norm: max |err| / bf16 ulp {float((err / _ulpb(want[first].double())).max()):.2f}, "
              f"{int((err > 0).sum())} of {err.numel()} elements differ")
        assert bool((err <= _ulpb(want[first].double())).all())


WIDTHS = {
    "llama2-7b": ("B200Llama", LF, dict(LF.CONFIG, hidden_size=4096, num_attention_heads=32, num_key_value_heads=32,
                                         intermediate_size=11008, vocab_size=32000)),
    "llama3-8b": ("B200Llama", LF, dict(LF.CONFIG, hidden_size=4096, num_attention_heads=32, num_key_value_heads=8,
                                         intermediate_size=14336, vocab_size=128256, rope_theta=500000.0)),
    "pythia-1b": ("B200NeoX", NF, dict(NF.CONFIG, hidden_size=2048, num_attention_heads=8, intermediate_size=8192,
                                        vocab_size=50304)),
    "pythia-6.9b": ("B200NeoX", NF, dict(NF.CONFIG, hidden_size=4096, num_attention_heads=32, intermediate_size=16384,
                                          vocab_size=50432)),
    "olmo-1b": ("B200Olmo", OF, OF.config("olmo", hidden_size=2048, num_attention_heads=16, num_key_value_heads=16,
                                          intermediate_size=8192, vocab_size=50304, clip_qkv=None)),
    "olmo2-7b": ("B200Olmo", OF, OF.config("olmo2", hidden_size=4096, num_attention_heads=32, num_key_value_heads=32,
                                           intermediate_size=11008, vocab_size=100352)),
}
# librsb bf16's per-row RMS error against transformers fp32 over transformers bf16's on the same row
ROW_MULTIPLE = 2.0


@pytest.mark.parametrize("name", list(WIDTHS))
@pytest.mark.parametrize("layers", [1, 2])
def test_hidden_rows_at_published_widths(name, layers):
    """Every row of the residual stream before the final norm, against transformers fp32 with the same weights: its
    RMS error at most ROW_MULTIPLE x transformers bf16's on that row."""
    from retrieval_scaling_b200 import reader
    cls, FX, base = WIDTHS[name]
    cfg = dict(base, num_hidden_layers=layers, max_position_embeddings=512)
    sd = FX.seeded_state_dict(cfg, seed=3)
    lens = [1, 63, 200, 65]
    rng = np.random.default_rng(layers)
    windows = [rng.integers(0, cfg["vocab_size"], S) for S in lens]
    cu = np.concatenate([[0], np.cumsum(lens)])
    m = getattr(reader, cls)(cfg, dtype=BF)
    m.load_state_dict(sd)
    ours = m.hidden_states(_i32(np.concatenate(windows)), _i32(cu), max(lens)).double()
    del m
    torch.cuda.empty_cache()

    def hf_rows(dtype):
        hf = FX.hf_model(cfg, dtype=dtype, seed=3, sd=sd) if FX is not LF else FX.hf_model(cfg, dtype=dtype, seed=3)
        hf = hf.cuda()
        base_model = hf.model if hasattr(hf, "model") else hf.gpt_neox
        got = []
        hook = base_model.layers[-1].register_forward_hook(
            lambda mod, inp, out: got.append((out[0] if isinstance(out, tuple) else out)[0].double()))
        with torch.no_grad():
            for w in windows:
                hf(torch.as_tensor(w, device="cuda")[None])
        hook.remove()
        del hf
        torch.cuda.empty_cache()
        return torch.cat(got)
    ref, hb = hf_rows(torch.float32), hf_rows(BF)
    e_o = (ours - ref).pow(2).mean(-1).sqrt()
    e_b = (hb - ref).pow(2).mean(-1).sqrt()
    ratio = e_o / e_b.clamp_min(1e-30)
    print(f"{name} x{layers}: hidden-row RMS error ours / HF bf16: max {float(ratio.max()):.2f}, median "
          f"{float(ratio.median()):.2f}")
    assert bool((e_o <= ROW_MULTIPLE * e_b).all())


def _e2e(tmp_path, FX, cfg, concate_k, build_dir):
    """`ric/main_ric.py --config-name perplexity ... +model.lm_dtype=bfloat16` on a tiny seeded datastore, against the
    reference's loop with transformers bf16 sdpa on the GPU.  Both readers round to bf16 at the same points; each
    window's mean loss is within ~1e-2 nats of float64 on the goldens for either (see test_golden_within_hf_bf16_
    precision), so the perplexities agree within exp(2e-2) - 1 ~ 2e-2 relative."""
    import json
    import re
    import subprocess

    from golden import roberta_fixture as RF
    from retrieval_scaling_b200 import config as C
    from retrieval_scaling_b200 import perplexity as P
    enc = RF.build(str(tmp_path / "enc"))
    reader_dir = build_dir(str(tmp_path / "reader"))
    rng = np.random.default_rng(9)
    texts = [" ".join(f"w{i}" for i in rng.integers(3, 1000, n)) for n in (300, 200)]
    words = " ".join(texts).split()
    psg_dir = tmp_path / "passages" / "dom" / "1-shards"
    psg_dir.mkdir(parents=True)
    with open(psg_dir / "raw_passages-0-of-1.jsonl", "w") as f:
        for i in range(150):
            if i % 5 == 0:
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
          f"evaluation.results_only_log_file={log}", "+model.lm_dtype=bfloat16"]
    cmd = [sys.executable, os.path.join(ROOT, "ric", "main_ric.py"), "--config-name", "perplexity",
           "tasks.datastore.embedding=true", "tasks.eval.search=true", "tasks.eval.inference=true", *ov]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    ppl_gpu = float(re.search(r"perplexity = ([0-9.]+)", open(log).read()).group(1))
    cfg_run = C.load_config("perplexity", os.path.join(ROOT, "ric", "conf"), ov)
    tok = FX.tokenizer()
    if concate_k:
        from retrieval_scaling_b200.search import get_merged_search_output_path
        eval_data = [json.loads(line) for line in open(get_merged_search_output_path(cfg_run))]
    else:
        eval_data = P.prepare_ppl_eval_data([json.loads(line) for line in open(eval_path)], tok, 128, 64, True)
    contexts, answers, _ = P.build_doc_prompts(eval_data, cfg_run.evaluation)
    hf = _hf(FX, cfg, BF, attn_implementation="sdpa")
    pad = P.lm_pad_token_id(tok)
    total, count = 0.0, 0
    for context, answer in zip(contexts, answers):                # src/evaluate_perplexity.py:117-139
        a = tok(answer, return_tensors="pt")["input_ids"]
        c = tok(context, return_tensors="pt")["input_ids"]
        ids = torch.cat((c, a), 1)
        lab = torch.cat((torch.full(c.size(), -100), a), 1)
        lab = torch.where(lab == pad, torch.tensor(-100), lab)
        with torch.no_grad():
            total += hf(ids[:, -4096:].cuda(), labels=lab[:, -4096:].cuda()).loss.item()
        count += 1
    ppl_hf = float(torch.exp(torch.tensor(total / count)))
    print(f"{cfg['model_type']} concate_k {concate_k}: {count} windows, perplexity librsb bf16 {ppl_gpu:.4f} "
          f"HF bf16 sdpa {ppl_hf:.4f} (rel {abs(ppl_gpu / ppl_hf - 1):.2e})")
    assert ppl_gpu == pytest.approx(ppl_hf, rel=2e-2)


@pytest.mark.parametrize("concate_k", [0, 3])
def test_main_ric_bf16_llama(tmp_path, concate_k):
    _e2e(tmp_path, LF, LF.CONFIG, concate_k, LF.build_dir)


@pytest.mark.parametrize("concate_k", [0, 3])
def test_main_ric_bf16_olmo2(tmp_path, concate_k):
    cfg = OF.CONFIGS["olmo2"]
    _e2e(tmp_path, OF, cfg, concate_k, lambda d: OF.build_dir(d, cfg))
