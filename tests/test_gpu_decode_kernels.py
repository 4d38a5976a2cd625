"""Kernel-level parity of the decode path of greedy generation (rsb_llm_generate, rsb_llm.cu) against fp64 references,
through its two diagnostic entry points:

  RoPE + KV cache  rsb_llm_decode_attention rotates a row at its explicit position bit-equal to rsb_llm_attention's
                   rotation of the same row at the same position of a prefill window (rope_kernel / olmo_qkv_kernel), and
                   kv_store_kernel writes that row's K and V at (slot, :, pos) of the cache and no other byte: Llama
                   (rope_theta 1e4 and 5e5), GPT-NeoX (rotary_pct 0.25), OLMo (clip_qkv) and OLMo-2 (QK-norm)
  split-KV         decode_attention_kernel and decode_combine_kernel per element within the bound of
                   oracle/attention_oracle.causal_attention (a decode row at position p is the last row of a window of
                   p + 1 positions), for 1, 4, 8, 16, 20 and 32 query heads per KV head at head_dim 128 and head_dim 64,
                   80 and 256, in fp16 and bf16, with Gaussian, flat, peaked and late-maximum scores
  greedy           greedy_rows_kernel (rsb_llm_greedy) against oracle/greedy_oracle.greedy: the id bit-equal, the
                   log-probability within a derived bound, at vocabularies 1 001 to 600 001, with ties at every
                   reduction level of the kernel, maxima at the ends of the vocabulary, -inf entries and poisoned pad
                   columns

Every attention and RoPE comparison also runs against deliberately wrong references (`_must_fail`) and has to reject
them.  Rows sit in shuffled, non-contiguous cache slots; every cache position past a row's own, every unused slot and
every split-KV partial starts as NaN, so a read of any of them shows up as a non-finite output.  Every refusal of the
two entry points returns before any launch and leaves the outputs as they were."""
import ctypes
import gc
import os
import sys
import zlib

import numpy as np
import pytest
import torch

from oracle import attention_oracle as AO
from oracle import greedy_oracle as GO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import llama_fixture as LF  # noqa: E402
import neox_fixture as NF  # noqa: E402
import olmo_fixture as OF  # noqa: E402

pytestmark = pytest.mark.gpu

DT = {"fp16": torch.float16, "bf16": torch.bfloat16}
MAX_POS = 2048
DCH = 64                                           # positions per split-KV chunk (rsb_llm.cu)
# the 16-key steps and 64-position chunks on both sides, a long row and the last position of the model
POSITIONS = [0, 1, 15, 16, 17, 63, 64, 65, 127, 128, 255, 256, 257, 1000, MAX_POS - 1]
SLOTS = 24
NAN16 = 0x7FFF                                     # a NaN in fp16 and in bf16


def _must_fail(name, ok):
    """A wrong reference has to be rejected by the comparison somewhere in the case."""
    assert not bool(np.all(ok)), f"the comparison also accepts the wrong reference {name!r}: its tolerance is too loose"


def _i32(a):
    return torch.as_tensor(np.asarray(a), dtype=torch.int32, device="cuda")


def _bits(t):
    return t.view(torch.int16)


def _nan_like(shape, dtype):
    return torch.full(shape, NAN16, dtype=torch.int16, device="cuda").view(dtype)


_HANDLE = {}


@pytest.fixture(scope="module", autouse=True)
def _release_device_memory():
    yield
    _HANDLE.clear()
    gc.collect()
    torch.cuda.empty_cache()


def _model(family, dtype, heads, kv, d=128, theta=1e4):
    """One live reader handle with one layer and nothing loaded (attention reads no weight; OLMo-2 gets layer 0's
    q_norm / k_norm).  family: llama, neox, olmo, olmo2."""
    key = (family, dtype, heads, kv, d, theta)
    if key not in _HANDLE:
        _HANDLE.clear()
        gc.collect()
        torch.cuda.empty_cache()
        from retrieval_scaling_b200 import reader
        small = dict(num_hidden_layers=1, intermediate_size=128, vocab_size=128, max_position_embeddings=MAX_POS)
        if family == "llama":
            m = reader.B200Llama(dict(LF.CONFIG, hidden_size=heads * 128, num_attention_heads=heads,
                                      num_key_value_heads=kv, rope_theta=theta, **small), dtype=DT[dtype])
        elif family == "neox":
            m = reader.B200NeoX(dict(NF.CONFIG, hidden_size=heads * d, num_attention_heads=heads, rotary_pct=0.25,
                                     **small), dtype=DT[dtype])
        else:
            m = reader.B200Olmo(OF.config(family, hidden_size=heads * 128, num_attention_heads=heads,
                                          num_key_value_heads=kv, clip_qkv=3.0 if family == "olmo" else None, **small),
                                dtype=DT[dtype])
            if family == "olmo2":
                g = torch.Generator(device="cuda").manual_seed(heads)
                m.load_weight("model.layers.0.self_attn.q_norm.weight", 1 + 0.3 * torch.randn(heads * 128, generator=g,
                                                                                             device="cuda"))
                m.load_weight("model.layers.0.self_attn.k_norm.weight", 1 + 0.3 * torch.randn(kv * 128, generator=g,
                                                                                             device="cuda"))
        _HANDLE[key] = m
    return _HANDLE[key]


def _slots(n, seed):
    """n distinct slots out of SLOTS, shuffled: rows never sit in slot order, and some slots stay unused."""
    return np.random.default_rng(seed).permutation(SLOTS)[:n]


def _decode(m, qkv0, slot, pos, kc0, vc0):
    """rsb_llm_decode_attention on copies: (qkv after, k_cache after, v_cache after, ctx)."""
    qkv, kc, vc = qkv0.clone(), kc0.clone(), vc0.clone()
    ctx = _nan_like((qkv.shape[0], m.geom["hidden_size"]), qkv.dtype)
    m.decode_attention(qkv, _i32(slot), _i32(pos), kc, vc, ctx)
    torch.cuda.synchronize()
    return qkv, kc, vc, ctx


def _check_cache(kc, vc, kc0, vc0, qkv, slot, pos, heads, kv, d):
    """The caches equal their inputs except (slot, :, pos) of every row, which holds that row's K and V after the
    call, bit for bit."""
    n = qkv.shape[0]
    s, p = torch.as_tensor(slot, device="cuda"), torch.as_tensor(pos, device="cuda")
    want_k, want_v = kc0.clone(), vc0.clone()
    want_k[s, :, p] = qkv[:, heads * d:(heads + kv) * d].reshape(n, kv, d)
    want_v[s, :, p] = qkv[:, (heads + kv) * d:].reshape(n, kv, d)
    assert torch.equal(_bits(kc), _bits(want_k)), "K cache: a wrong element written, or the row's K not stored"
    assert torch.equal(_bits(vc), _bits(want_v)), "V cache: a wrong element written, or the row's V not stored"


# ---------------------------------------------------------------------------------------------------------------
# RoPE / prologue and the cache store
# ---------------------------------------------------------------------------------------------------------------
ROPE_FAMILIES = {  # name -> (family, heads, kv_heads, head_dim, rope_theta)
    "llama-theta1e4": ("llama", 8, 2, 128, 1e4),
    "llama-theta5e5": ("llama", 8, 2, 128, 5e5),
    "neox-rot16": ("neox", 4, 4, 64, 1e4),
    "olmo-clip": ("olmo", 8, 2, 128, 1e4),
    "olmo2-qknorm": ("olmo2", 8, 2, 128, 1e4),
}


@pytest.mark.parametrize("dtype", list(DT))
@pytest.mark.parametrize("name", list(ROPE_FAMILIES))
def test_rope_and_cache_bit_for_bit(name, dtype):
    """Each decode row after the call (Q and K rotated, OLMo's clamp of Q, K and V, OLMo-2's QK-norm) is bit-equal to the
    same row at the same position of a prefill window run through rsb_llm_attention; the cache holds that row's K and V
    at (slot, :, pos) and every other byte keeps its NaN pattern.  Rejected: the prefill's rotation one position
    further on."""
    family, heads, kv, d, theta = ROPE_FAMILIES[name]
    m = _model(family, dtype, heads, kv, d, theta)
    W = (heads + 2 * kv) * d
    n = len(POSITIONS)
    seed = zlib.crc32(f"rope {name} {dtype}".encode())
    g = torch.Generator(device="cuda").manual_seed(seed)
    qkv0 = (torch.randn(n, W, generator=g, device="cuda") * 2).to(DT[dtype])
    slot = _slots(n, seed)
    kc0 = _nan_like((SLOTS, kv, MAX_POS, d), DT[dtype])
    vc0 = kc0.clone()
    qkv, kc, vc, _ = _decode(m, qkv0, slot, POSITIONS, kc0, vc0)   # ctx: attention over a NaN cache
    _check_cache(kc, vc, kc0, vc0, qkv, slot, POSITIONS, heads, kv, d)

    # prefill: window b holds row b at position p and again at p + 1 (where the model has room for it)
    lens = [min(p + 2, MAX_POS) for p in POSITIONS]
    cu = np.concatenate([[0], np.cumsum(lens)])
    pre0 = (torch.randn(int(cu[-1]), W, generator=g, device="cuda") * 2).to(DT[dtype])
    at_p = torch.as_tensor(cu[:-1] + np.asarray(POSITIONS), device="cuda")
    nxt = torch.as_tensor([c + p + 1 for c, p, L in zip(cu[:-1], POSITIONS, lens) if p + 1 < L], device="cuda")
    pre0[at_p] = qkv0
    pre0[nxt] = qkv0[[i for i, (p, L) in enumerate(zip(POSITIONS, lens)) if p + 1 < L]]
    pre = pre0.clone()
    m.attention(pre, _i32(cu), max(lens), torch.empty((int(cu[-1]), heads * d), dtype=DT[dtype], device="cuda"))
    torch.cuda.synchronize()
    same = _bits(qkv) == _bits(pre[at_p])
    assert same.all(), (name, dtype, [POSITIONS[i] for i in torch.nonzero(~same.all(1))[:, 0].tolist()])
    one_on = [i for i, (p, L) in enumerate(zip(POSITIONS, lens)) if p + 1 < L]
    _must_fail("rotation one position further on", (_bits(qkv[one_on]) == _bits(pre[nxt])).cpu().numpy())
    print(f"[rope {name} {dtype}] {n} rows bit-equal to the prefill rotation; cache writes exact")


# ---------------------------------------------------------------------------------------------------------------
# split-KV attention per element
# ---------------------------------------------------------------------------------------------------------------
ATT_GEOMS = {  # name -> (family, heads, kv_heads, head_dim); G = heads / kv_heads query heads per KV head
    "G1-d128": ("llama", 2, 2, 128),
    "G4-d128": ("llama", 8, 2, 128),
    "G8-d128": ("llama", 16, 2, 128),
    "G16-d128": ("llama", 32, 2, 128),
    "G20-d128": ("llama", 40, 2, 128),             # a partial second 16-row tile
    "G32-d128": ("llama", 64, 2, 128),             # two full tiles
    "G1-d64": ("neox", 2, 2, 64),
    "G1-d80": ("neox", 8, 8, 80),                  # hidden 640: the readers take multiples of 128
    "G1-d256": ("neox", 2, 2, 256),
}
ARMS = ["gauss", "flat", "peaked", "late_max"]


def _rotate64(x, pos, theta, rot, sign=1.0):
    """Approximate RoPE in fp64 of x [n, h, d] at positions pos [n] (sign -1: the inverse rotation), on dims [0, rot):
    only used to aim designed keys at the rotated queries."""
    half = rot // 2
    inv = 1.0 / theta ** (torch.arange(0, rot, 2, dtype=torch.float64, device="cuda") / rot)
    f = sign * torch.as_tensor(pos, dtype=torch.float64, device="cuda")[:, None, None] * inv
    c, s = f.cos(), f.sin()
    y = x.clone()
    x1, x2 = x[..., :half], x[..., half:rot]
    y[..., :half] = x1 * c - x2 * s
    y[..., half:rot] = x2 * c + x1 * s
    return y


def _arm_data(arm, m, dtype, heads, kv, d, slot, pos, seed):
    """(qkv0 [n, W], k_cache, v_cache [SLOTS, kv, MAX_POS, d]) in the dtype.  Positions 0 .. pos - 1 of each row's slot
    hold the arm's keys and values, everything else NaN; position pos comes from the row itself.  Scores in nats:
      gauss     q and k Gaussian, scores with std ~2.5
      flat      q = 0: every score 0, ctx = mean of v over 0 .. pos
      peaked    one key at +60 in chunk pos // 64 - 1 (the only chunk for pos < 64), the rest of its chunk 0.5 .. 8 below
                it, every other key at -55 or lower: the other chunks are more than 150 log2 units below and their
                combine weights underflow to 0
      late_max  every key of the earlier chunks at 20 .. 21, one key of the last chunk at 25, the rest of it near 0
    The designed arms give the G query heads of a KV head one q, and aim each key (the row's own key through the inverse
    rotation) along that head's rotated q."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    n, G, rot = len(pos), heads // kv, m.geom.get("rotary_ndims", 128)
    theta = m.geom.get("rope_theta", m.geom.get("rotary_emb_base"))
    rnd = lambda *s: torch.randn(*s, generator=g, device="cuda", dtype=torch.float64)   # noqa: E731
    uni = lambda *s: torch.rand(*s, generator=g, device="cuda", dtype=torch.float64)    # noqa: E731
    K = torch.full((SLOTS, kv, MAX_POS, d), float("nan"), dtype=torch.float64, device="cuda")
    V = K.clone()
    off = 2.0 * torch.arange(kv, device="cuda", dtype=torch.float64)[:, None, None]       # distinct V per KV head
    q = rnd(n, heads, d) * 1.6
    k_new = rnd(n, kv, d) * 1.6
    if arm == "flat":
        q.zero_()
    elif arm in ("peaked", "late_max"):
        q = rnd(n, kv, 1, d).expand(n, kv, G, d).reshape(n, heads, d).clone()
        qr = _rotate64(q, pos, theta, rot)[:, ::G]                                           # [n, kv, d]
        aim = qr * d ** 0.5 / (qr * qr).sum(-1, keepdim=True)                               # score of t * aim = t
    for i, (s, p) in enumerate(zip(slot, pos)):
        V[s, :, :p + 1] = rnd(kv, p + 1, d) + off
        if arm in ("gauss", "flat"):
            K[s, :, :p] = rnd(kv, p, d) * 1.6
            continue
        c_last = p // DCH
        t = torch.empty(kv, p + 1, dtype=torch.float64, device="cuda")
        if arm == "peaked":
            c = max(c_last - 1, 0)
            lo, hi = c * DCH, min((c + 1) * DCH, p + 1)
            t[:] = -55.0 - 5 * uni(kv, p + 1)
            t[:, lo:hi] = 60.0 - 0.5 - 7.5 * uni(kv, hi - lo)
            t[torch.arange(kv), lo + torch.randint(0, hi - lo, (kv,), generator=g, device="cuda")] = 60.0
        else:
            t[:, :c_last * DCH] = 20.0 + uni(kv, c_last * DCH)
            t[:, c_last * DCH:] = 2 * uni(kv, p + 1 - c_last * DCH) - 1
            t[torch.arange(kv), c_last * DCH + torch.randint(0, p + 1 - c_last * DCH, (kv,), generator=g,
                                                             device="cuda")] = 25.0
        keys = t[..., None] * aim[i][:, None, :]                                            # [kv, p + 1, d]
        K[s, :, :p] = keys[:, :p]
        k_new[i] = _rotate64(keys[None, :, p], [p], theta, rot, sign=-1.0)[0]
    W = (heads + 2 * kv) * d
    qkv0 = torch.empty(n, W, dtype=torch.float64, device="cuda")
    qkv0[:, :heads * d] = q.reshape(n, -1)
    qkv0[:, heads * d:(heads + kv) * d] = k_new.reshape(n, -1)
    qkv0[:, (heads + kv) * d:] = V[torch.as_tensor(slot, device="cuda"), :, torch.as_tensor(pos, device="cuda")].reshape(n, -1)
    V[torch.as_tensor(slot, device="cuda"), :, torch.as_tensor(pos, device="cuda")] = float("nan")
    return qkv0.to(DT[dtype]), K.to(DT[dtype]), V.to(DT[dtype])


@pytest.mark.parametrize("dtype", list(DT))
@pytest.mark.parametrize("geom", list(ATT_GEOMS))
def test_split_kv_attention_per_element(geom, dtype):
    """One rsb_llm_decode_attention call per arm with a row at every position of POSITIONS in shuffled slots; ctx of
    every row and query head is within causal_attention's bound of fp64 attention of its rotated q (read back from qkv)
    over its cache as read back after the call (K and V of positions 0 .. pos).  The cache is written only at each
    row's (slot, :, pos).  Rejected, per arm: the last key dropped, the chunk before the row's last one dropped, the
    neighbouring KV head, and the scales 1 / sqrt(head_dim +- 8) (not in the flat arm, whose scores are all 0)."""
    family, heads, kv, d = ATT_GEOMS[geom]
    m = _model(family, dtype, heads, kv, d)
    n = len(POSITIONS)
    slot_of = _slots(n, zlib.crc32(geom.encode()))
    report = []
    for arm in ARMS:
        seed = zlib.crc32(f"{geom} {dtype} {arm}".encode())
        qkv0, kc0, vc0 = _arm_data(arm, m, dtype, heads, kv, d, slot_of, POSITIONS, seed)
        qkv, kc, vc, ctx = _decode(m, qkv0, slot_of, POSITIONS, kc0, vc0)
        _check_cache(kc, vc, kc0, vc0, qkv, slot_of, POSITIONS, heads, kv, d)
        assert torch.isfinite(ctx).all(), (geom, dtype, arm, "a NaN cache position or partial was read")
        wrong = {"last key dropped": lambda p: dict(mask_shift=-1),
                 "one chunk dropped": lambda p: dict(drop_key=np.arange((p // DCH - 1) * DCH, p // DCH * DCH)),
                 "neighbouring KV head": lambda p: dict(kv_map="next"),
                 "scale 1/sqrt(d+8)": lambda p: dict(scale=(d + 8) ** -0.5),
                 "scale 1/sqrt(d-8)": lambda p: dict(scale=(d - 8) ** -0.5)}
        applies = {"last key dropped": lambda p: p >= 1, "one chunk dropped": lambda p: p >= DCH,
                   "neighbouring KV head": lambda p: True, "scale 1/sqrt(d+8)": lambda p: arm != "flat",
                   "scale 1/sqrt(d-8)": lambda p: arm != "flat"}
        ok = {w: [] for w in wrong}
        worst = 0.0
        for i, (s, p) in enumerate(zip(slot_of, POSITIONS)):
            win = torch.zeros((p + 1, (heads + 2 * kv) * d), dtype=DT[dtype], device="cuda")
            win[p, :heads * d] = qkv[i, :heads * d]
            win[:, heads * d:(heads + kv) * d] = kc[s, :, :p + 1].permute(1, 0, 2).reshape(p + 1, kv * d)
            win[:, (heads + kv) * d:] = vc[s, :, :p + 1].permute(1, 0, 2).reshape(p + 1, kv * d)
            cu = [0, p + 1]
            ref, bound = AO.causal_attention(win, cu, heads, kv, last_row_only=True, with_bound=True)
            ref, bound = ref[p], bound[p]
            got = ctx[i].double()
            ratio = ((got - ref).abs() / bound).max().item()
            assert ratio <= 1.0, (geom, dtype, arm, p, ratio, int(((got - ref).abs() / bound).argmax()))
            worst = max(worst, ratio)
            for w, kw in wrong.items():
                if applies[w](p):
                    r = AO.causal_attention(win, cu, heads, kv, last_row_only=True, **kw(p))[p]
                    ok[w].append(bool(((got - r).abs() <= bound).all()))
        for w in wrong:
            if ok[w]:
                _must_fail(f"{w} ({arm})", ok[w])
        report.append(f"{arm} {worst:.3f}")
    print(f"[decode attention {geom} {dtype}] max |err| / bound: " + ", ".join(report))


# ---------------------------------------------------------------------------------------------------------------
# greedy choice
# ---------------------------------------------------------------------------------------------------------------
VOCABS = [1001, 32000, 50280, 128256, 600001]
TIE = 10.0                                          # above every Gaussian logit of the designed rows


def _greedy_rows(vocab, ld, dtype, seed):
    """(names, logits [n, ld] in the dtype).  Gaussian rows (std 3) with their pad columns [vocab, ld) at 0, then the
    designed rows:
      tie+1, tie+8, tie+256, tie+2048   ids 298 and 298 + k at the row's maximum: one 8-wide load, neighbouring
                                        threads, another warp, the same thread's next iteration
      tie-lane                          ids 255 (lane 31 of warp 0) and 2048 (lane 0's next iteration): the lower id
                                        in the higher lane
      tie-wrap                          ids 2047 (last thread, warp 7) and 2048 (thread 0's next iteration): the lower
                                        id in the higher warp
      max-first, max-last               the maximum at id 0, and at vocab - 1
      all-equal                         every logit 0.75: id 0 and log-probability -log(vocab)
      neg-inf, one-finite               half the logits -inf (id 0 among them), and every logit but one -inf
      pad-nan, pad-inf, pad-max         the pad columns NaN, +inf and the largest finite value, the maximum at vocab - 1
                                        (rows that exist only where ld > vocab)"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    dt = DT[dtype]
    base = lambda: torch.randn(ld, generator=g, device="cuda") * 3   # noqa: E731
    rows, names = [], []

    def add(name, r):
        r = r.to(dt)
        names.append(name)
        rows.append(r)
        return r
    for i in range(4):
        r = base()
        r[vocab:] = 0
        add(f"gauss{i}", r)
    for k, (a, b) in {"tie+1": (298, 299), "tie+8": (298, 306), "tie+256": (298, 554), "tie+2048": (298, 2346),
                      "tie-lane": (255, 2048), "tie-wrap": (2047, 2048)}.items():
        if b < vocab:
            r = base().clamp_(-9, 9)
            r[a] = r[b] = TIE
            r[vocab:] = 0
            add(k, r)
    for k, at in (("max-first", 0), ("max-last", vocab - 1)):
        r = base().clamp_(-9, 9)
        r[at] = TIE
        r[vocab:] = 0
        add(k, r)
    r = torch.full((ld,), 0.75, device="cuda")
    r[vocab:] = 0
    add("all-equal", r)
    r = base()
    r[torch.rand(ld, generator=g, device="cuda") < 0.5] = -float("inf")
    r[0] = -float("inf")
    r[vocab:] = 0
    add("neg-inf", r)
    r = torch.full((ld,), -float("inf"), device="cuda")
    r[vocab // 2] = 1.0
    r[vocab:] = 0
    add("one-finite", r)
    if ld > vocab:
        for k, fill in (("pad-nan", float("nan")), ("pad-inf", float("inf")), ("pad-max", torch.finfo(dt).max)):
            r = base().clamp_(-9, 9)
            r[vocab - 1] = TIE
            r = r.to(dt)
            r[vocab:] = fill
            add(k, r)
    return names, torch.stack(rows)


def _greedy(logits, vocab, dtype):
    from retrieval_scaling_b200 import _lib
    L = _lib.lib()
    n, ld = logits.shape
    ids = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    lp = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
    code = _lib.RSB_DTYPE_BF16 if dtype == "bf16" else _lib.RSB_DTYPE_F16
    rc = L.rsb_llm_greedy(code, ctypes.c_void_p(logits.data_ptr()), vocab, ld, n, ctypes.c_void_p(ids.data_ptr()),
                          ctypes.c_void_p(lp.data_ptr()), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == _lib.RSB_OK, L.rsb_llm_last_error()
    torch.cuda.synchronize()
    return ids.cpu().numpy(), lp.cpu().numpy().astype(np.float64)


@pytest.mark.parametrize("dtype", list(DT))
@pytest.mark.parametrize("vocab", VOCABS)
def test_greedy_choice(vocab, dtype):
    """rsb_llm_greedy at ld = vocab rounded up to 128 (the LM head's vocab_pad): every id equals numpy's argmax of the
    fp32 values of the logits over [0, vocab) (the lowest id on ties), and every log-probability is within
    greedy_oracle.greedy's bound of fp64 x[id] - logsumexp(x[:vocab]).  The logits are not written."""
    ld = (vocab + 127) // 128 * 128
    names, logits = _greedy_rows(vocab, ld, dtype, zlib.crc32(f"greedy {vocab} {dtype}".encode()))
    before = logits.clone()
    ids, lp = _greedy(logits, vocab, dtype)
    assert torch.equal(_bits(logits), _bits(before))
    want, ref, bound = GO.greedy(logits.float().cpu().numpy(), vocab)
    for name, i, w in zip(names, ids, want):
        assert i == w, (vocab, dtype, name, int(i), int(w))
    err = np.abs(lp - ref)
    ratio = err / bound
    assert np.all(ratio <= 1.0), (vocab, dtype, names[int(np.argmax(ratio))], float(ratio.max()))
    at = {name: k for k, name in enumerate(names)}
    assert ids[at["all-equal"]] == 0 and abs(lp[at["all-equal"]] + np.log(vocab)) <= bound[at["all-equal"]]
    assert ids[at["one-finite"]] == vocab // 2 and lp[at["one-finite"]] == 0.0
    for k in ("tie+1", "tie+8", "tie+256", "tie+2048", "tie-lane", "tie-wrap"):
        if k in at:
            assert ids[at[k]] == {"tie-lane": 255, "tie-wrap": 2047}.get(k, 298), k
    print(f"[greedy V={vocab} {dtype}] {len(names)} rows: ids exact, max |err| / bound {ratio.max():.3f} "
          f"(bound {bound.min():.1e} .. {bound.max():.1e})")


# ---------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------
def test_refusals_before_any_launch():
    """Each refusal of rsb_llm_decode_attention and rsb_llm_greedy returns its error before any launch: qkv, both caches
    and ctx (ids and logprob) keep their sentinels.  A call with the same buffers and valid arguments then runs."""
    from retrieval_scaling_b200 import _lib
    heads, kv, d, n = 8, 2, 128, 3
    m = _model("llama", "fp16", heads, kv, d)
    L = m.L
    p = lambda t: ctypes.c_void_p(t.data_ptr())   # noqa: E731
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    cap = MAX_POS + 64                                  # room past max_pos, so that position refusal is reachable
    qkv = torch.zeros((n, (heads + 2 * kv) * d), dtype=torch.float16, device="cuda")
    kc = _nan_like((4, kv, cap, d), torch.float16)
    vc = kc.clone()
    ctx = _nan_like((n, heads * d), torch.float16)

    def untouched():
        torch.cuda.synchronize()
        return bool((qkv == 0).all()) and bool((_bits(kc) == NAN16).all()) and bool((_bits(vc) == NAN16).all()) \
            and bool((_bits(ctx) == NAN16).all())

    good_s, good_p = _i32([2, 0, 3]), _i32([5, 0, 70])
    for slot, pos, rows, slots, cp, rc, msg in [
            ([2, 0, 4], [5, 0, 70], n, 4, cap, _lib.RSB_ERR_INVALID, b"outside [0, slots"),
            ([2, -1, 3], [5, 0, 70], n, 4, cap, _lib.RSB_ERR_INVALID, b"outside [0, slots"),
            ([2, 0, 2], [5, 0, 70], n, 4, cap, _lib.RSB_ERR_INVALID, b"two rows"),
            ([2, 0, 3], [5, cap, 70], n, 4, cap, _lib.RSB_ERR_INVALID, b"cap"),
            ([2, 0, 3], [5, -1, 70], n, 4, cap, _lib.RSB_ERR_INVALID, b"cap"),
            ([2, 0, 3], [5, MAX_POS, 70], n, 4, cap, _lib.RSB_ERR_UNSUPPORTED, b"max_position_embeddings"),
            ([2, 0, 3], [5, 0, 70], 0, 4, cap, _lib.RSB_ERR_INVALID, b"positive"),
            ([2, 0, 3], [5, 0, 70], -1, 4, cap, _lib.RSB_ERR_INVALID, b"positive"),
            ([2, 0, 3], [5, 0, 70], n, 0, cap, _lib.RSB_ERR_INVALID, b"positive"),
            ([2, 0, 3], [5, 0, 70], n, 4, 0, _lib.RSB_ERR_INVALID, b"positive")]:
        ds, dp = _i32(slot), _i32(pos)                  # alive across the call
        got = L.rsb_llm_decode_attention(m._h, p(qkv), p(ds), p(dp), rows, p(kc), p(vc), slots, cp, p(ctx), st)
        assert got == rc and msg in L.rsb_llm_last_error(), (slot, pos, rows, slots, cp, got, L.rsb_llm_last_error())
    args = [m._h, p(qkv), p(good_s), p(good_p), n, p(kc), p(vc), 4, cap, p(ctx), st]
    for k in (0, 1, 2, 3, 5, 6, 9):                   # each pointer null in turn
        a = list(args)
        a[k] = None
        assert L.rsb_llm_decode_attention(*a) == _lib.RSB_ERR_INVALID, k
    a = list(args)
    a[1] = ctypes.c_void_p(qkv.data_ptr() + 2)
    assert L.rsb_llm_decode_attention(*a) == _lib.RSB_ERR_INVALID and b"aligned" in L.rsb_llm_last_error()
    assert untouched()
    kc.zero_()                                          # finite keys and values for the call that runs
    vc.zero_()
    assert L.rsb_llm_decode_attention(*args) == _lib.RSB_OK
    torch.cuda.synchronize()
    assert torch.isfinite(ctx).all()

    qkv.zero_()                                         # sentinels again, for the OLMo-2 refusal
    ctx.copy_(_nan_like(ctx.shape, torch.float16))
    kc.copy_(_nan_like(kc.shape, torch.float16))
    vc.copy_(kc)
    from retrieval_scaling_b200.reader import B200Olmo
    bare = B200Olmo(OF.config("olmo2", hidden_size=heads * 128, num_attention_heads=heads, num_key_value_heads=kv,
                              num_hidden_layers=1, intermediate_size=128, vocab_size=128,
                              max_position_embeddings=MAX_POS), dtype=torch.float16)   # no q_norm / k_norm loaded
    assert L.rsb_llm_decode_attention(bare._h, *args[1:]) == _lib.RSB_ERR_STATE
    assert b"q_norm" in L.rsb_llm_last_error() and untouched()
    del bare

    logits = torch.zeros((2, 1024), dtype=torch.float16, device="cuda")
    ids = torch.full((2,), -7, dtype=torch.int32, device="cuda")
    lp = torch.full((2,), 5.0, dtype=torch.float32, device="cuda")
    g = [_lib.RSB_DTYPE_F16, p(logits), 1001, 1024, 2, p(ids), p(lp), st]
    for k, v in [(0, _lib.RSB_DTYPE_F32), (0, _lib.RSB_DTYPE_SQ8), (1, None), (5, None), (6, None), (2, 0), (2, -3),
                 (3, 1000), (3, 1020), (4, -1), (1, ctypes.c_void_p(logits.data_ptr() + 8))]:
        a = list(g)
        a[k] = v
        assert L.rsb_llm_greedy(*a) == _lib.RSB_ERR_INVALID, (k, v)
    torch.cuda.synchronize()
    assert bool((ids == -7).all()) and bool((lp == 5.0).all())
    assert L.rsb_llm_greedy(*g) == _lib.RSB_OK
    torch.cuda.synchronize()
    assert ids.tolist() == [0, 0] and float(lp[0]) == pytest.approx(-np.log(1001), abs=1e-5)
