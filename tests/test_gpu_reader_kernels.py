"""Kernel-level parity of the Llama reader (rsb_llm.cu) against fp64 references, at the released readers' head
geometries, the attention kernel's tile edges and the LM head's chunk edges, through the two diagnostic hooks
(`rsb_llm_attention`, `rsb_llm_hidden_states`) and `rsb_llm_nll`:

  RoPE + attention  rope_kernel bit for bit against oracle/attention_oracle.rope_f16 (HF's fp16 order), then
                    attention_causal_kernel per element within the bound of attention_oracle.causal_attention, for
                    heads : kv_heads 4:1, 4:4, 8:2, 32:32, 32:8, 40:40 and 64:8
  NLL head          final RMSNorm, the chunked LM head and nll_rows_kernel against fp64 of the GPU's own hidden rows,
                    within a derived per-token bound, at vocabularies 128 256, 32 001 and 600 001
  production        every token row and every token's NLL of 1- and 2-layer models at Llama-2-7B, Llama-3-8B and
                    Llama-2-13B width against transformers fp32, within twice transformers fp16's own error

Every comparison also runs against deliberately wrong references (`_must_fail`) and has to reject them, so that a
tolerance that would accept a wrong kernel fails the test instead.  Weights and inputs are generated on the device
from seeds; one model handle is alive at a time."""
import ctypes
import gc
import os
import sys
import zlib

import numpy as np
import pytest
import torch

from oracle import attention_oracle as AO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import llama_fixture as LF  # noqa: E402

pytestmark = pytest.mark.gpu

D = 128
PAD = 64                                           # rows past cu_seqlens[B]: never rotated nor written
LENGTHS = [1, 2, 7, 8, 9, 15, 16, 17, 31, 32, 33, 48, 63, 64, 65, 127, 128, 129, 191, 192, 193, 1000, 4095, 4096, 4097,
           8191, 8192]
# heads : kv_heads -> (heads, kv_heads, rope_theta)
GEOMS = {"4:1": (4, 1, 1e4), "4:4": (4, 4, 5e5), "8:2": (8, 2, 1e4), "32:32": (32, 32, 1e4), "32:8": (32, 8, 5e5),
         "40:40": (40, 40, 1e4), "64:8": (64, 8, 5e5)}


def _must_fail(name, ok):
    """A wrong reference has to be rejected by the comparison somewhere in the case."""
    assert not bool(np.all(ok)), f"the comparison also accepts the wrong reference {name!r}: its tolerance is too loose"


def _ulp16(x):
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e.clamp_min(-14) - 10)


def _r16(x):
    return x.half().double()


def _i32(a):
    return torch.as_tensor(np.asarray(a), dtype=torch.int32, device="cuda")


def _cfg(heads, kv_heads, **kw):
    c = dict(LF.CONFIG, num_hidden_layers=1, hidden_size=heads * D, num_attention_heads=heads,
             num_key_value_heads=kv_heads, intermediate_size=128, vocab_size=128, max_position_embeddings=8192)
    c.update(kw)
    return c


_HANDLE = {}


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    """Frees the last handle and torch's cached blocks when the module ends: later tests allocate through librsb's own
    cudaMalloc, which cannot reuse blocks cached by torch."""
    yield
    _HANDLE.clear()
    gc.collect()
    torch.cuda.empty_cache()


def _handle(key, make):
    """One live model handle: the previous one is freed before the next geometry is built."""
    if key not in _HANDLE:
        _HANDLE.clear()
        gc.collect()
        torch.cuda.empty_cache()
        _HANDLE[key] = make()
    return _HANDLE[key]


def _seeded(cfg, seed, dtype=torch.float32):
    """HF LlamaForCausalLM keys on the device, at the scales of tests/golden/llama_fixture.py, each tensor drawn in
    fp32 and stored in `dtype` (so the fp16 weights of a seed are the fp32 weights of that seed rounded)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    H, I, V, KV = cfg["hidden_size"], cfg["intermediate_size"], cfg["vocab_size"], cfg["num_key_value_heads"] * D

    def n(*shape, std, base=0.0):
        return (base + torch.randn(*shape, generator=g, device="cuda") * std).to(dtype)

    sd = {"model.embed_tokens.weight": n(V, H, std=3.0 / H ** 0.5 if cfg["tie_word_embeddings"] else 1.0),
          "model.norm.weight": n(H, std=0.1, base=1.0)}
    for i in range(cfg["num_hidden_layers"]):
        p = f"model.layers.{i}."
        sd[p + "self_attn.q_proj.weight"] = n(H, H, std=1.5 / H ** 0.5)
        sd[p + "self_attn.k_proj.weight"] = n(KV, H, std=1.5 / H ** 0.5)
        sd[p + "self_attn.v_proj.weight"] = n(KV, H, std=1.0 / H ** 0.5)
        sd[p + "self_attn.o_proj.weight"] = n(H, H, std=1.0 / H ** 0.5)
        sd[p + "mlp.gate_proj.weight"] = n(I, H, std=1.0 / H ** 0.5)
        sd[p + "mlp.up_proj.weight"] = n(I, H, std=1.0 / H ** 0.5)
        sd[p + "mlp.down_proj.weight"] = n(H, I, std=1.0 / I ** 0.5)
        sd[p + "input_layernorm.weight"] = n(H, std=0.1, base=1.0)
        sd[p + "post_attention_layernorm.weight"] = n(H, std=0.1, base=1.0)
    if not cfg["tie_word_embeddings"]:
        sd["lm_head.weight"] = n(V, H, std=3.0 / H ** 0.5)
    return sd


def _reader(cfg, sd):
    from retrieval_scaling_b200.reader import B200Llama
    m = B200Llama(cfg)
    assert m.load_state_dict(sd) == []
    return m


# ---------------------------------------------------------------------------------------------------------------
# RoPE and attention
# ---------------------------------------------------------------------------------------------------------------
def _attention_model(geom):
    """Attention reads no weight: a one-layer handle with a tiny vocabulary and intermediate size, nothing loaded."""
    heads, kv, theta = GEOMS[geom]
    from retrieval_scaling_b200.reader import B200Llama
    return _handle(("attention", geom), lambda: B200Llama(_cfg(heads, kv, rope_theta=theta)))


def _composition(name):
    """(window lengths, max_seqlen); max_seqlen None = the longest window."""
    rng = np.random.default_rng(len(name))
    short = [S for S in LENGTHS if S <= 1000]
    rng.shuffle(short)
    h = len(short) // 2
    return {
        # every length; the longest window first, 8191 in the middle and 4097 last
        "every_length": ([8192] + short[:h] + [4095, 8191, 4096] + short[h:] + [4097], None),
        "stress": ([1, 9, 64, 65, 129, 193, 1000, 33, 17], None),
        "b1": ([4097], None),
        "many_short": (list(rng.integers(1, 41, 2000)), None),
        "zero_length_inside": ([5, 0, 64, 0, 0, 17, 129, 0, 3], None),
        "max_seqlen_above_longest": ([40, 20, 97], 8192),
    }[name]


def _qkv(arm, lens, heads, kv, seed):
    """fp16 [T + PAD, (heads + 2 kv) 128] inputs of an arm (see test_rope_and_attention_per_element)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    T = int(np.sum(lens))
    hid, kvd = heads * D, kv * D
    n = lambda *s: torch.randn(*s, generator=g, device="cuda")   # noqa: E731
    x = n(T + PAD, hid + 2 * kvd)
    qk = slice(0, hid + kvd)
    wid = torch.repeat_interleave(torch.arange(len(lens), device="cuda"), torch.as_tensor(lens, device="cuda"))
    if arm == "gauss":                                   # q.k / sqrt(128) with std ~2.5
        x[:, qk] *= 1.6
    elif arm == "exact":                                 # multiples of 1/4 in [-2, 2]: q.k exact in fp32
        x[:, qk] = torch.randint(-8, 9, (T + PAD, hid + kvd), generator=g, device="cuda").float() / 4
    elif arm == "large":                                 # |scores| ~ 12
        x[:, qk] *= 3.5
    elif arm in ("dominant_first", "dominant_diag", "dominant_below"):
        # one key ~14 above the others for every query that sees it: key 0 of the window, the query's own position,
        # or the position just below it
        x[:, qk] *= 0.5
        U = torch.randint(0, 2, (T + PAD, D), generator=g, device="cuda").float() * 2 - 1
        if arm == "dominant_first":
            starts = torch.as_tensor(np.concatenate([[0], np.cumsum(lens)[:-1]]), device="cuda")
            Uq = U[starts[wid]]
            Uk = torch.zeros_like(U[:T])
            Uk[starts[wid]] = Uq
        elif arm == "dominant_diag":
            Uq, Uk = U[:T], U[:T]
        else:
            Uq, Uk = torch.roll(U[:T], 1, 0), U[:T]
        x[:T, :hid] += 0.5 * Uq.repeat(1, heads)
        x[:T, hid:hid + kvd] += 2.5 * Uk.repeat(1, kv)
    elif arm == "equal":                                 # every key of a window identical
        x[:T, hid:hid + kvd] = (n(len(lens), kvd) * 0.5)[wid]
    elif arm == "per_kv_head":                           # distinct content per KV head: the head map is observable
        for j in range(kv):
            x[:, hid + j * D:hid + (j + 1) * D] *= 0.5 + j
            x[:, hid + kvd + j * D:hid + kvd + (j + 1) * D] += 3.0 * (j + 1)
        x[:, :hid] *= 1.3
    else:
        raise ValueError(arm)
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return x.half(), cu


def _run_attention(m, qkv0, cu, max_seqlen, hid):
    qkv = qkv0.clone()
    ctx = torch.full((qkv.shape[0], hid), float("nan"), dtype=torch.float16, device="cuda")
    m.attention(qkv, _i32(cu), max_seqlen, ctx)
    torch.cuda.synchronize()
    return qkv, ctx


CASES = ([("every_length", a) for a in ("gauss", "exact")]
         + [("stress", a) for a in ("dominant_first", "dominant_diag", "dominant_below", "equal", "large", "per_kv_head")]
         + [("b1", "gauss"), ("many_short", "gauss"), ("zero_length_inside", "exact"),
            ("max_seqlen_above_longest", "gauss")])


@pytest.mark.parametrize("comp,arm", CASES)
@pytest.mark.parametrize("geom", list(GEOMS))
def test_rope_and_attention_per_element(geom, comp, arm):
    """rsb_llm_attention on packed windows: the rotated Q / K heads are bit-equal to `rope_f16` (HF's fp16 order), where
    an fp32 cos / sin within 2 fp32 ulp of an fp16 boundary may take either fp16 neighbour; V and every row
    past cu_seqlens[B] are untouched; every ctx element is within `causal_attention`'s bound (fp16 rounding of P, fp32
    accumulation over the visible keys, hardware exp2, fp32 q.k, output rounding); rows past cu_seqlens[B] keep their
    NaN sentinel; a window run alone gives bit-equal rows.  Arms: Gaussian scores (std ~2.5), exact q.k, a dominant key
    at position 0 / on the diagonal / just below it, all scores equal, large scores, distinct content per KV head.

    Rejected wrong references: global positions, GPT-J pair rotation, fp64 angles (at positions >= 4096); the
    interleaved GQA map h % kv_heads, the causal mask shifted by one either way, key 63 (the last of the first 64-key
    block) dropped."""
    heads, kv, theta = GEOMS[geom]
    m = _attention_model(geom)
    torch.cuda.reset_peak_memory_stats()
    lens, max_seqlen = _composition(comp)
    max_seqlen = max(lens) if max_seqlen is None else max_seqlen
    seed = zlib.crc32(f"{geom} {comp} {arm}".encode())
    qkv0, cu = _qkv(arm, lens, heads, kv, seed)
    T, hid, nrot = int(cu[-1]), heads * D, heads + kv
    qkv, ctx = _run_attention(m, qkv0, cu, max_seqlen, hid)

    # RoPE, in row chunks (the full [T, heads + kv_heads, 128] tensors of a 40 000-token pack would take GBs per copy)
    pos = AO.window_positions(cu, T)
    assert torch.equal(qkv[:, nrot * D:].view(torch.int16), qkv0[:, nrot * D:].view(torch.int16)), "V was written"
    assert torch.equal(qkv[T:].view(torch.int16), qkv0[T:].view(torch.int16)), "rows past cu_seqlens[B] were rotated"
    wrong_ok = {"GPT-J adjacent-pair rotation": True, "global positions": True, "fp64 angles": True}
    rc = max(1, (1 << 22) // (nrot * D))
    for r0 in range(0, T, rc):
        r1 = min(T, r0 + rc)
        x0 = qkv0[r0:r1, :nrot * D].view(r1 - r0, nrot, D)
        got = qkv[r0:r1, :nrot * D].view(r1 - r0, nrot, D).view(torch.int16)
        ref, near = AO.rope_f16(x0, pos[r0:r1], theta)
        nearx = near.expand_as(got)
        same = got == ref.view(torch.int16)
        assert (same | nearx).all(), ("rope", r0, int((~same & ~nearx).sum()))
        for i in (-1, 0, 1):                           # flagged elements: the result of either fp16 cos / sin neighbour
            for j in (-1, 0, 1):
                same |= got == AO.rope_f16(x0, pos[r0:r1], theta, cs_shift=(i, j))[0].view(torch.int16)
        assert same.all(), ("rope at an fp16 boundary of cos / sin", r0, int((~same).sum()))
        exact = lambda r: bool(((got == r.view(torch.int16)) | nearx).all())   # noqa: E731
        wrong_ok["GPT-J adjacent-pair rotation"] &= exact(AO.rope_f16(x0, pos[r0:r1], theta, pairing="adjacent")[0])
        wrong_ok["global positions"] &= exact(AO.rope_f16(x0, np.arange(r0, r1), theta)[0])
        far = torch.as_tensor(pos[r0:r1] >= 4096, device="cuda")
        if far.any():
            f64 = AO.rope_f16(x0, pos[r0:r1], theta, angles="fp64")[0]
            wrong_ok["fp64 angles"] &= bool(((got == f64.view(torch.int16)) | nearx)[far].all())
        del x0, got, ref, near, same
    if max(lens) > 1:
        _must_fail("GPT-J adjacent-pair rotation", wrong_ok["GPT-J adjacent-pair rotation"])
    if sum(S > 0 for S in lens) > 1 and max(lens[1:]) > 1:
        _must_fail("global positions", wrong_ok["global positions"])
    if (pos >= 4096).any():
        _must_fail("fp64 angles", wrong_ok["fp64 angles"])

    # attention, per group of consecutive windows of up to 8 192 tokens (one longer window is a group of its own)
    assert torch.isnan(ctx[T:]).all(), "rows past cu_seqlens[B] were written"
    wrong = {"interleaved GQA map": dict(kv_map="interleaved"), "causal mask one key too far": dict(mask_shift=1),
             "causal mask one key short": dict(mask_shift=-1), "key 63 dropped": dict(drop_key=63)}
    wrong_ok = {name: True for name in wrong}
    worst = 0.0
    b0 = 0
    while b0 < len(lens):
        b1 = b0 + 1
        while b1 < len(lens) and cu[b1 + 1] - cu[b0] <= 8192:
            b1 += 1
        t0, t1 = int(cu[b0]), int(cu[b1])
        if t1 > t0:
            sub, gcu = qkv[t0:t1], cu[b0:b1 + 1] - t0
            out = ctx[t0:t1].double()
            assert torch.isfinite(out).all(), ("rows of the windows left unwritten", b0, b1)
            ref, bound = AO.causal_attention(sub, gcu, heads, kv, with_bound=True)
            ratio = (out - ref).abs_().div_(bound)
            w = ratio.max().item()
            assert w <= 1.0, (geom, comp, arm, b0, w, np.unravel_index(int(torch.argmax(ratio)), tuple(ratio.shape)))
            worst = max(worst, w)
            del ref, ratio
            for name, kw in wrong.items():
                wrong_ok[name] &= bool(((out - AO.causal_attention(sub, gcu, heads, kv, **kw)).abs_() <= bound).all())
            del out, bound
        b0 = b1
    print(f"[attention {geom} {comp} {arm}] max |err| / bound = {worst:.3f}; "
          f"peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
    if 1 < kv < heads:
        _must_fail("interleaved GQA map", wrong_ok["interleaved GQA map"])
    if max(lens) >= 2:
        _must_fail("causal mask one key too far", wrong_ok["causal mask one key too far"])
        _must_fail("causal mask one key short", wrong_ok["causal mask one key short"])
    if max(lens) >= 64:
        _must_fail("key 63 dropped", wrong_ok["key 63 dropped"])

    if comp in ("every_length", "zero_length_inside", "stress"):
        for i, S in enumerate(lens):                       # the same window alone: bit-equal rows
            if S == 0 or (i % 4 and S not in (65, 4097, 8192)):
                continue
            q1, c1 = _run_attention(m, qkv0[cu[i]:cu[i + 1]], [0, S], S, hid)
            assert torch.equal(c1.view(torch.int16), ctx[cu[i]:cu[i + 1]].view(torch.int16)), (i, S)
            assert torch.equal(q1.view(torch.int16), qkv[cu[i]:cu[i + 1]].view(torch.int16)), (i, S)


def test_hook_refusals_before_any_launch():
    """rsb_llm_attention / rsb_llm_hidden_states refuse null arguments, sequences past max_position_embeddings and
    malformed offsets before any launch (the output keeps its sentinel); hidden_states refuses a handle without its
    weights."""
    from retrieval_scaling_b200 import _lib
    m = _attention_model("8:2")
    L = m.L
    qkv = torch.zeros((40, 12 * D), dtype=torch.float16, device="cuda")
    ctx = torch.full((40, 8 * D), float("nan"), dtype=torch.float16, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())   # noqa: E731
    for cu, B, T, ms, rc, msg in [
            ([0, 8193], 1, 8193, 8193, _lib.RSB_ERR_UNSUPPORTED, b"max_position_embeddings"),
            ([0, 5, 3], 2, 40, 8, _lib.RSB_ERR_INVALID, b"decreases"),
            ([0, 20, 41], 2, 40, 21, _lib.RSB_ERR_INVALID, b"from 0"),
            ([1, 20], 1, 40, 20, _lib.RSB_ERR_INVALID, b"from 0"),
            ([0, 30], 1, 40, 20, _lib.RSB_ERR_INVALID, b"max_seqlen"),
            ([0, 5], 0, 40, 5, _lib.RSB_ERR_INVALID, b"empty"),
            ([0, 5], 1, 0, 5, _lib.RSB_ERR_INVALID, b"empty")]:
        cut = _i32(cu)
        assert L.rsb_llm_attention(m._h, p(qkv), p(cut), B, T, ms, p(ctx), None) == rc, cu
        assert msg in L.rsb_llm_last_error(), (cu, L.rsb_llm_last_error())
    assert L.rsb_llm_attention(m._h, None, p(_i32([0, 5])), 1, 40, 5, p(ctx), None) == _lib.RSB_ERR_INVALID
    assert L.rsb_llm_attention(m._h, p(qkv), p(_i32([0, 5])), 1, 40, 5, None, None) == _lib.RSB_ERR_INVALID
    torch.cuda.synchronize()
    assert torch.isnan(ctx).all() and (qkv == 0).all()
    ids = torch.zeros(5, dtype=torch.int32, device="cuda")
    with pytest.raises(RuntimeError, match="not loaded"):
        m.hidden_states(ids, _i32([0, 5]), 5)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    out = torch.empty((5, 8 * D), dtype=torch.float16, device="cuda")
    assert L.rsb_llm_hidden_states(m._h, p(ids), p(_i32([0, 5])), 1, 5, 8193, p(out), p(ws), ws.numel(),
                                   None) == _lib.RSB_ERR_UNSUPPORTED
    assert L.rsb_llm_hidden_states(m._h, p(ids), p(_i32([0, 5])), 1, 5, 5, None, p(ws), ws.numel(),
                                   None) == _lib.RSB_ERR_INVALID


# ---------------------------------------------------------------------------------------------------------------
# final norm, chunked LM head, nll_rows_kernel
# ---------------------------------------------------------------------------------------------------------------
def _pack(windows):
    lens = [len(w) for w in windows]
    return (_i32(np.concatenate(windows)), np.concatenate([[0], np.cumsum(lens)]).astype(np.int64), max(lens))


def _head_reference(m, sd, X, windows, labels, eps):
    """Per scored token of the pack, in label-row order: (row, label, out index) and the fp64 reference of
    nll = logsumexp(logits) - logits[label] from the GPU's own hidden rows X, with its bound.  Also the normed fp16 rows
    n16 and the gathered label rows W[label] (for the wrong references), the log-sum-exp over the whole 8-wide vectors
    only (lse8), and each row's largest logit and its column.  No [rows, vocab] tensor is kept."""
    cfg = m.geom
    V, H = cfg["vocab_size"], cfg["hidden_size"]
    rows, labs, outi = [], [], []
    t0 = 0
    for w, lb in zip(windows, labels):
        for t in range(1, len(w)):
            if lb[t] != -100:
                rows.append(t0 + t - 1); labs.append(int(lb[t])); outi.append(t0 + t)
        t0 += len(w)
    g = sd["model.norm.weight"].half().double()
    W = (sd["model.embed_tokens.weight"] if cfg["tie_word_embeddings"] else sd["lm_head.weight"]).half().double()
    Wa = W.abs()
    xs = X[torch.as_tensor(rows, device="cuda")].double()
    # HF LlamaRMSNorm: fp32 statistics, x * rstd rounded to half, times the half weight; an fp32 rstd can round an
    # element to the other fp16 neighbour where x * rstd lies within its relative error of a boundary
    h = xs * torch.rsqrt((xs * xs).mean(-1, keepdim=True) + eps)
    eps_r = H * 2.0 ** -24 + 2.0 ** -21
    amb = _r16(h * (1 - eps_r)) != _r16(h * (1 + eps_r))
    n16 = _r16(_r16(h) * g)
    dn = torch.where(amb, _ulp16(h) * g.abs() + _ulp16(n16), torch.zeros_like(n16))
    y = torch.as_tensor(labs, device="cuda")
    out = dict(rows=rows, labs=labs, outi=outi, n16=n16, Wy=W[y], nll=[], bound=[], lse=[], ly=[], lse8=[], lmax=[],
               argmax=[])
    step = max(1, (1 << 23) // V)
    for r0 in range(0, len(rows), step):
        r1 = min(len(rows), r0 + step)
        lg = n16[r0:r1] @ W.T
        e = 2 * H * 2.0 ** -24 * (n16[r0:r1].abs() @ Wa.T) + dn[r0:r1] @ Wa.T + 2.0 ** -24 * lg.abs()
        b = e.add_(0.5 * _ulp16(lg.abs() + e))                             # |fp16 logit - lg|
        lse = torch.logsumexp(lg, -1)
        ly = lg.gather(1, y[r0:r1, None])[:, 0]
        # fp32 log-sum-exp: V / 256 sequential adds and V / 2048 rescalings per thread, 16 merges, expf to 2 ulp
        a = (V / 128 + 32) * 2.0 ** -24 + 2.0 ** -22 * (lse.abs() + ly.abs())
        out["nll"].append(lse - ly)
        out["bound"].append(b.max(1).values + b.gather(1, y[r0:r1, None])[:, 0] + a)
        out["lse"].append(lse)
        out["ly"].append(ly)
        out["lse8"].append(torch.logsumexp(lg[:, : V // 8 * 8], -1))
        mx = lg.max(1)
        out["lmax"].append(mx.values)
        out["argmax"].append(mx.indices)
        del lg, e, b
    for k in ("nll", "bound", "lse", "ly", "lse8", "lmax", "argmax"):
        out[k] = torch.cat(out[k])
    return out


def _nll_and_hidden(m, windows, labels):
    ids, cu, ms = _pack(windows)
    X = m.hidden_states(ids, _i32(cu), ms)
    nll = torch.cat(m.nll(windows, labels, max_tokens=1 << 30)).cuda().double()
    return X, nll


def _windows_for(nl, rng, V):
    """Windows whose scored positions (all labels kept) add up to nl label rows."""
    lens = {1: [2], 1023: [1024], 1024: [500, 526], 1025: [600, 427], 3073: [1000, 1500, 576]}.get(nl)
    if lens is None:
        lens = [nl + 1]
    return [rng.integers(0, V, S) for S in lens]


HEAD_CASES = [  # (vocab, heads, tied, label-row counts)
    (128256, 4, False, [1, 1023, 1024, 1025, 3073]),
    (32001, 4, True, [3073, 4500]),
    (600001, 1, False, [1, 500]),
]


@pytest.mark.parametrize("V,heads,tied,counts", HEAD_CASES)
def test_nll_head_against_fp64_of_the_gpu_hidden_rows(V, heads, tied, counts):
    """The final norm, the LM head in chunks of chunk_rows() label rows and the fp32 log-sum-exp against fp64 of the
    GPU's own hidden rows (rsb_llm_hidden_states) in HF's order (RMSNorm, head, log-softmax), per token within
        max_j b_j + b_label + (V / 128 + 32) 2^-24 + 2^-22 (|lse| + |logit_label|),
    b_j = 2 H 2^-24 sum|n||W_j| + (fp16 neighbours of ambiguous normed elements) + 1/2 ulp of the fp16 logit.
    Vocabularies 128 256 (chunks of 1 024 rows: 1, 1 023, 1 024, 1 025 and 3 073 label rows, windows straddling a chunk
    boundary), 32 001 tied (chunks of 4 096, a vocabulary tail of 1 inside the last 8-wide vector) and 600 001 at hidden
    128 (chunks at the floor of 128, an odd tail).  Every token's NLL is bit-equal wherever its row falls: windows
    reordered, and labels masked in front of them.  Rejected: the label logit of the neighbouring row, a chunk's rows
    offset by one."""
    cfg = _cfg(heads, max(1, heads // 4), vocab_size=V, tie_word_embeddings=tied, intermediate_size=256,
               max_position_embeddings=8192)
    sd = _seeded(cfg, 7 + V)
    m = _handle(("head", V, tied), lambda: _reader(cfg, sd))
    chunk = max(128, (256 << 20) // (((V + 127) // 128 * 128) * 2) // 128 * 128)
    rng = np.random.default_rng(V)
    worst = 0.0
    torch.cuda.reset_peak_memory_stats()
    for nl in counts:
        windows = _windows_for(nl, rng, V)
        X, nll = _nll_and_hidden(m, windows, windows)
        R = _head_reference(m, sd, X, windows, windows, cfg["rms_norm_eps"])
        assert len(R["rows"]) == nl
        oi = torch.as_tensor(R["outi"], device="cuda")
        got = nll[oi]
        ratio = ((got - R["nll"]).abs() / R["bound"])
        worst = max(worst, ratio.max().item())
        assert ratio.max().item() <= 1.0, (V, nl, ratio.max().item(), int(torch.argmax(ratio)))
        if nl >= 2:
            # the label logit read from the neighbouring row: logits[r + 1, label_r]
            wrong = R["lse"] - (torch.roll(R["n16"], -1, 0) * R["Wy"]).sum(1)
            _must_fail("label logit of the neighbouring row", ((got - wrong).abs() <= R["bound"]).cpu().numpy())
        if nl > chunk:
            # a chunk's rows offset by one: label row i >= chunk scored on the hidden row of label row i - 1
            wrong = torch.roll(R["lse"], 1, 0) - (torch.roll(R["n16"], 1, 0) * R["Wy"]).sum(1)
            okv = (got - wrong).abs() <= R["bound"]
            _must_fail("a chunk's rows offset by one", okv[chunk:].cpu().numpy())
        # bit-equal wherever the row falls: windows reversed, and labels masked in front of them
        rev = m.nll(windows[::-1], windows[::-1], max_tokens=1 << 30)[::-1]
        masked = [np.array(w) for w in windows]
        masked[0] = masked[0].copy()
        masked[0][: min(len(masked[0]) - 1, 37)] = -100
        msk = m.nll(windows, masked, max_tokens=1 << 30)
        full = m.nll(windows, windows, max_tokens=1 << 30)
        for f, r, k, lb in zip(full, rev, msk, masked):
            assert torch.equal(f, r)
            sc = np.zeros(len(lb), bool)
            sc[1:] = lb[1:] != -100
            assert torch.equal(f[sc], k[sc])
        del R
        torch.cuda.empty_cache()
    print(f"[nll head V={V} tied={tied}] max |err| / bound = {worst:.3f}; "
          f"peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")


@pytest.mark.parametrize("arm", ["all_below_zero", "last_id_top"])
def test_nll_head_designed_logits(arm):
    """With o_proj and down_proj zero a layer is the identity, so the final rows are embedding rows and the logits can be
    chosen (vocabulary 32 001, 127 pad columns, a tail of 1 in the last 8-wide vector):
      all_below_zero  every real logit ~ -20: a zero pad column in the sum would dominate it
      last_id_top     the label is the last id, in the partial last vector, with the largest logit (~ +12)
    Within the bound of test_nll_head_against_fp64_of_the_gpu_hidden_rows; rejected: pad columns in the sum (first
    arm), the partial last vector dropped (second arm)."""
    V, H = 32001, 512
    cfg = _cfg(4, 1, vocab_size=V, intermediate_size=256)
    sd = _seeded(cfg, 3)
    g = torch.Generator(device="cuda").manual_seed(5)
    sd["model.layers.0.self_attn.o_proj.weight"].zero_()
    sd["model.layers.0.mlp.down_proj.weight"].zero_()
    sd["model.norm.weight"].fill_(1.0)
    u = torch.randint(0, 2, (H,), generator=g, device="cuda").float() * 2 - 1
    sd["model.embed_tokens.weight"] = u[None].repeat(V, 1) * (1 + 0.05 * torch.rand(V, 1, generator=g, device="cuda"))
    noise = torch.randn(V, H, generator=g, device="cuda") / H ** 0.5
    if arm == "all_below_zero":
        sd["lm_head.weight"] = -20.0 / H * u[None] + 0.5 * noise
    else:
        sd["lm_head.weight"] = noise.clone()
        sd["lm_head.weight"][V - 1] = 12.0 / H * u
    m = _handle(("designed", arm), lambda: _reader(cfg, sd))
    rng = np.random.default_rng(11)
    windows = [rng.integers(0, V, S) for S in (300, 4000)]
    labels = [w.copy() for w in windows]
    if arm == "last_id_top":
        labels = [np.full(len(w), V - 1) for w in windows]
    X, nll = _nll_and_hidden(m, windows, labels)
    R = _head_reference(m, sd, X, windows, labels, cfg["rms_norm_eps"])
    got = nll[torch.as_tensor(R["outi"], device="cuda")]
    ratio = (got - R["nll"]).abs() / R["bound"]
    assert ratio.max().item() <= 1.0, ratio.max().item()
    print(f"[nll head designed {arm}] max |err| / bound = {ratio.max().item():.3f}")
    if arm == "all_below_zero":
        assert R["lmax"].max().item() < -10
        pad = (V + 127) // 128 * 128 - V
        wrong = torch.logaddexp(R["lse"], torch.full_like(R["lse"], float(np.log(pad)))) - R["ly"]
        _must_fail("pad columns in the sum", ((got - wrong).abs() <= R["bound"]).cpu().numpy())
    else:
        assert (R["argmax"] == V - 1).all()
        wrong = R["lse8"] - R["ly"]
        _must_fail("partial last vector dropped", ((got - wrong).abs() <= R["bound"]).cpu().numpy())


# ---------------------------------------------------------------------------------------------------------------
# token rows and NLL at production geometry
# ---------------------------------------------------------------------------------------------------------------
PROD = {  # name -> (heads, kv_heads, intermediate, vocab, rope_theta, window lengths)
    "llama2-7b": (32, 32, 11008, 32000, 1e4, [4096, 1, 65, 300]),
    "llama3-8b": (32, 8, 14336, 128256, 5e5, [8192, 129]),
    "llama2-13b": (40, 40, 13824, 32000, 1e4, [4096, 200]),
}


def _hf(cfg, sd, dtype):
    """transformers LlamaForCausalLM on the device holding `sd` (cast to dtype), built on the meta device."""
    import transformers
    kw = {k: v for k, v in cfg.items() if k != "model_type"}
    c = transformers.LlamaConfig(**kw)
    c._attn_implementation = "sdpa"
    with torch.device("meta"):
        model = transformers.LlamaForCausalLM(c)
    model.load_state_dict({k: v.to(dtype) for k, v in sd.items()}, strict=False, assign=True)
    for mod in model.modules():
        if hasattr(mod, "inv_freq") and hasattr(mod, "compute_default_rope_parameters"):
            inv = mod.compute_default_rope_parameters(mod.config)[0].to("cuda")
            mod.inv_freq, mod.original_inv_freq = inv, inv
    return model.eval()


def _hf_rows_and_nll(model, ids):
    """(pre-norm rows [S, H] fp64, nll [S] fp64 with 0 at t = 0, max |logit| per row) of one window; the logits are
    taken from the normed rows in chunks of 256."""
    cap = []
    hk = model.model.norm.register_forward_hook(lambda mod, a, o: cap.append((a[0][0], o[0])))
    x = torch.as_tensor(ids, device="cuda")[None]
    with torch.no_grad():
        model.model(x)
    hk.remove()
    pre, normed = cap[0]
    nll = torch.zeros(len(ids), dtype=torch.float64, device="cuda")
    lmax = torch.zeros(len(ids), dtype=torch.float64, device="cuda")
    with torch.no_grad():
        for r0 in range(0, len(ids), 256):
            r1 = min(len(ids), r0 + 256)
            lg = model.lm_head(normed[r0:r1]).double()
            lmax[r0:r1] = lg.abs().max(1).values
            lp = torch.log_softmax(lg, -1)
            t = torch.arange(r0 + 1, r1 + 1, device="cuda").clamp_max(len(ids) - 1)
            v = -lp.gather(1, x[0, t][:, None])[:, 0]
            keep = t > torch.arange(r0, r1, device="cuda")
            nll[t[keep]] = v[keep]
    return pre.double(), nll, lmax


@pytest.mark.parametrize("layers", [1, 2])
@pytest.mark.parametrize("name", list(PROD))
def test_token_rows_and_nll_at_production_geometry(name, layers, monkeypatch):
    """Every token row of rsb_llm_hidden_states and every token's NLL of a model at a released reader's width against
    transformers fp32 on the device: per row max |err| <= 2x transformers fp16's own max |err| on that row (floor: 1
    fp16 ulp of the row's largest element); per token |err| <= 2x the larger of fp16's error on that token and 1 fp16
    ulp of the row's largest |logit| (the resolution of fp16 logits, below which fp16's error on one token is chance).
    transformers fp16 rounds where the kernels do (fp32 RMSNorm statistics then fp16, fp16 linears, fp16 residual
    adds) and, like the kernels, runs the fp32 weights rounded to fp16.  Rejected: the fp32 rows shifted by one within
    each window, the NLL of the neighbouring token."""
    import transformers.integrations.sdpa_attention as hf_sdpa
    # transformers hands grouped KV heads to torch's sdpa as enable_gqa when there is no mask, which torch serves in
    # fp32 only with its math kernel: the [heads, S, S] scores of an 8 192-token window would take 9 GB.  repeat_kv,
    # transformers' own path whenever a mask is given, computes the same attention with the memory-efficient kernel.
    monkeypatch.setattr(hf_sdpa, "use_gqa_in_sdpa", lambda *a, **k: False)
    heads, kv, inter, V, theta, lens = PROD[name]
    cfg = dict(LF.CONFIG, num_hidden_layers=layers, hidden_size=heads * D, num_attention_heads=heads,
               num_key_value_heads=kv, intermediate_size=inter, vocab_size=V, rope_theta=theta,
               max_position_embeddings=max(lens), rms_norm_eps=1e-5)
    _HANDLE.clear()
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    # one copy of the weights at a time: fp16 for the kernels and transformers fp16, then fp32 drawn again from the seed
    sd = _seeded(cfg, 100 + layers, torch.float16)
    m = _reader(cfg, sd)
    rng = np.random.default_rng(layers)
    windows = [rng.integers(0, V, S) for S in lens]
    ids, cu, ms = _pack(windows)
    ours = m.hidden_states(ids, _i32(cu), ms).double()
    ours_nll = [o.cuda().double() for o in m.nll(windows, windows)]
    del m
    gc.collect()
    res = {}
    for dt in (torch.float16, torch.float32):
        if dt == torch.float32:
            del sd
            gc.collect()
            sd = _seeded(cfg, 100 + layers, torch.float32)
        hf = _hf(cfg, sd, dt)
        res[dt] = [_hf_rows_and_nll(hf, w) for w in windows]
        del hf
        gc.collect()
        torch.cuda.empty_cache()
    del sd
    worst_r, worst_n = 0.0, 0.0
    shifted_ok, nb_ok = [], []
    for b, w in enumerate(windows):
        h32, n32, l32 = res[torch.float32][b]
        h16, n16, _ = res[torch.float16][b]
        got = ours[cu[b]:cu[b + 1]]
        err = (got - h32).abs().max(1).values
        lim = torch.maximum(2 * (h16 - h32).abs().max(1).values, _ulp16(h32.abs().max(1).values))
        worst_r = max(worst_r, (err / lim).max().item())
        assert (err <= lim).all(), (name, layers, b, (err / lim).max().item(), int(torch.argmax(err / lim)))
        if len(w) > 1:
            sh = torch.roll(h32, 1, 0)
            shifted_ok.append(((got - sh).abs().max(1).values <= lim).cpu().numpy())
            en = (ours_nll[b] - n32).abs()[1:]
            ln = 2 * torch.maximum((n16 - n32).abs(), _ulp16(torch.roll(l32, 1, 0)))[1:]
            worst_n = max(worst_n, (en / ln).max().item())
            assert (en <= ln).all(), (name, layers, b, (en / ln).max().item(), int(torch.argmax(en / ln)))
            nb_ok.append(((ours_nll[b] - torch.roll(n32, 1, 0)).abs()[2:] <= ln[1:]).cpu().numpy())
    _must_fail("rows shifted by one", np.concatenate(shifted_ok))
    _must_fail("NLL of the neighbouring token", np.concatenate(nb_ok))
    print(f"[production {name} L={layers}] max err / (2x fp16 err): rows {worst_r:.3f}, nll {worst_n:.3f}; "
          f"peak {torch.cuda.max_memory_allocated() / 2 ** 30:.1f} GiB")
