"""Kernel-level parity of the encoder (rsb_bert.cu) against fp64 references, at the sequence-length, batch and tile
edges, through the two diagnostic hooks (`rsb_bert_attention`, `RSB_POOL_TOKENS`) and `rsb_gemm_f16`:

  attention   both kernels (<= 32 tokens: attention_mma32_kernel, 33..512: attention_flash_kernel on the side stream)
              in the BERT and the T5 form, per element against oracle/attention_oracle.py
  GEMM        gemm_tn_kernel, every epilogue rsb_gemm_f16 reaches, both row-tile orders, per element
  forward     every token row of the BERT and T5 forwards against the fp16 and fp32 torch oracles
  head        pool_kernel, the Dense GEMM and l2normalize_rows_kernel, each against fp64 of the GPU's own previous step

Every comparison is also run against deliberately wrong references (`_must_fail`) and has to reject them, so that a
tolerance that would accept a wrong kernel fails the test instead."""
import ctypes
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import attention_oracle as AO
from oracle import bert_oracle as BO
from oracle import t5_oracle as T5O

pytestmark = pytest.mark.gpu

LENGTHS = [1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 96, 97, 127, 128, 129, 160, 255, 256, 257, 384, 385, 511, 512]
BERT_CFG = dict(hidden_size=768, num_hidden_layers=1, num_attention_heads=12, intermediate_size=3072, vocab_size=3000,
                max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12)
T5_CFG = dict(T5O.T5_CONFIG, num_layers=1, vocab_size=2048)


def _L():
    from retrieval_scaling_b200 import _lib
    return _lib.lib()


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ulp16(x):
    """attention_oracle.ulp16 on a device tensor."""
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e.clamp_min(-14) - 10)


def _must_fail(name, ok):
    """A wrong reference has to be rejected by the comparison somewhere in the case."""
    assert not bool(np.all(ok)), f"the comparison also accepts the wrong reference {name!r}: its tolerance is too loose"


# ---------------------------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------------------------
_HANDLES = {}


def _attention_model(form):
    """A one-layer handle per form; attention reads no weight except the T5 relative-attention bias, which is random
    per bucket and head, in multiples of 1/8 (so that the exact-score arm stays exact)."""
    if form not in _HANDLES:
        from retrieval_scaling_b200.encoder import B200Contriever, B200T5Encoder
        if form == "bert":
            _HANDLES[form] = (B200Contriever(BERT_CFG), None)
        else:
            m = B200T5Encoder(T5_CFG)
            nb, md = T5_CFG["relative_attention_num_buckets"], T5_CFG["relative_attention_max_distance"]
            w = torch.from_numpy(np.random.default_rng(77).integers(-24, 25, (nb, 12)) / 8).half()
            m.load_state_dict({"encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight": w})
            _HANDLES[form] = (m, AO.t5_bias_table(w.numpy(), AO.t5_buckets(nb, md)))
    return _HANDLES[form]


def _attention(form, qkv, cu, max_seqlen, pad=64):
    """ctx [T + pad, 768] from rsb_bert_attention, every row pre-filled with a NaN sentinel."""
    m, _ = _attention_model(form)
    T = qkv.shape[0]
    ctx = torch.full((T + pad, 768), float("nan"), dtype=torch.float16, device="cuda")
    qd = torch.from_numpy(qkv).cuda()
    cd = torch.from_numpy(np.asarray(cu, np.int32)).cuda()
    rc = _L().rsb_bert_attention(m._h, ctypes.c_void_p(qd.data_ptr()), ctypes.c_void_p(cd.data_ptr()), len(cu) - 1, T,
                                 int(max_seqlen), ctypes.c_void_p(ctx.data_ptr()), _stream())
    assert rc == 0, _L().rsb_bert_last_error()
    torch.cuda.synchronize()
    return ctx.cpu().numpy()


def _composition(name):
    """(lengths, max_seqlen) of a batch; max_seqlen None = the longest length."""
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    comp = {
        "every_length": (list(rng.permutation(LENGTHS)), None),                 # mixed, long sequences in the middle
        "short_only": ([1, 2, 15, 16, 17, 31, 32, 7, 32, 1], None),
        "long_only": ([33, 63, 64, 65, 96, 97, 127, 128, 129, 160, 255, 256, 257, 384, 385, 511, 512], None),
        "long_first": ([512, 1, 2, 17, 32, 31], None),
        "long_last": ([3, 31, 32, 5, 16, 385], None),
        "long_middle": ([7, 32, 300, 12, 1], None),
        "b1_short": ([17], None),
        "b1_long": ([511], None),
        "b3_odd": ([33, 1, 129], None),
        "queries_3000": (list(rng.integers(1, 33, 3000)), None),
        "zero_length_inside": ([5, 0, 40, 0, 0, 17, 129, 0, 3], None),
        "max_seqlen_above_longest": ([40, 20, 97], 512),
        "max_seqlen_gt32_no_long": ([1, 32, 17, 8, 31], 100),
    }[name]
    return comp


def _qkv(arm, form, lens, rng):
    """fp16 [T, 2304] inputs of an arm (see test_attention_matches_fp64_reference)."""
    T = int(np.sum(lens))
    cu = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    x = np.empty((T, 2304))
    x[:, 1536:] = rng.standard_normal((T, 768))                                    # V
    if arm == "gauss":
        x[:, :1536] = rng.standard_normal((T, 1536)) * (1.5 if form == "bert" else 0.6)
    elif arm == "exact":                                                           # q.k exact in fp32; T5: fp16 too
        hi = 8 if form == "bert" else 3
        x[:, :1536] = rng.integers(-hi, hi + 1, (T, 1536)) / 4
    elif arm == "large":
        x[:, :1536] = rng.standard_normal((T, 1536)) * (4.0 if form == "bert" else 2.0)
    elif arm in ("dominant_first", "dominant_last"):
        # one key per sequence with a score ~10 above the others for every query; in the first 32-key block the running
        # maximum is set at once, in the last one it moves at the end and every earlier block is rescaled
        x[:, :1536] = rng.standard_normal((T, 1536)) * 0.5
        u = rng.choice([-1.0, 1.0], 768)
        a, b = (0.5, 2.5) if form == "bert" else (0.25, 0.6)
        x[:, :768] += a * u
        for i, S in enumerate(lens):
            if S == 0:
                continue
            nblk = (S + 31) // 32
            j = int(rng.integers(0, min(S, 32))) if arm == "dominant_first" else int(rng.integers((nblk - 1) * 32, S))
            x[cu[i] + j, 768:1536] = b * u
    elif arm == "equal":                                                           # every key of a sequence identical
        x[:, :768] = rng.standard_normal((T, 768))
        for i, S in enumerate(lens):
            x[cu[i]:cu[i + 1], 768:1536] = rng.standard_normal(768) * 0.5
    else:
        raise ValueError(arm)
    return x.astype(np.float16), cu


CASES = ([(c, a) for c in ("every_length", "short_only", "long_only", "long_first", "long_last", "long_middle", "b1_short",
                           "b1_long", "b3_odd", "queries_3000", "zero_length_inside", "max_seqlen_above_longest",
                           "max_seqlen_gt32_no_long") for a in ("gauss", "exact")]
         + [("stress", a) for a in ("dominant_first", "dominant_last", "equal", "large")])


@pytest.mark.parametrize("form", ["bert", "t5"])
@pytest.mark.parametrize("comp,arm", CASES)
def test_attention_matches_fp64_reference(form, comp, arm):
    """Every element of ctx within the bound of `attention_oracle.attention` (its docstring derives the terms: the fp16
    rounding of each probability, fp32 accumulation of q.k and P.V, hardware exp2, T5's fp16 score roundings where
    fp32 and fp64 may round differently, and the output rounding).  Arms: Gaussian Q/K/V at realistic score scale
    (BERT: q.k / 8 with std ~2; T5: q.k with std ~5 plus the bias); exact scores (Q, K small multiples of 1/4: the
    bound reduces to 2^-11 sum p|v| + fp32 P.V + 1/2 ulp); a dominant key in the first / last 32-key block; all scores
    equal; large |scores| (std ~16 after scaling).

    Also: every row in [0, T) is written and no row at or past T changes (NaN sentinel); a sequence run alone gives
    bit-equal rows; and the comparison rejects a reference without the last key, and BERT without the 1/8 scale or T5
    with the relative position negated or the neighbouring head's bias."""
    rng = np.random.default_rng([len(comp), len(arm), 1 if form == "bert" else 2])
    if comp == "stress":
        lens, max_seqlen = [33, 64, 65, 129, 257, 512, 31, 17, 1], None
    else:
        lens, max_seqlen = _composition(comp)
    max_seqlen = max(lens) if max_seqlen is None else max_seqlen
    qkv, cu = _qkv(arm, form, lens, rng)
    T = int(cu[-1])
    _, table = _attention_model(form)
    got = _attention(form, qkv, cu, max_seqlen).astype(np.float64)
    assert np.isfinite(got[:T]).all(), "rows in [0, T) left unwritten"
    assert np.isnan(got[T:]).all(), "rows past T were written"
    ref, bound = AO.attention(qkv, cu, form, table, with_bound=True)
    err = np.abs(got[:T] - ref)
    ratio = err / bound
    worst = np.unravel_index(np.argmax(ratio), ratio.shape)
    assert ratio.max() <= 1.0, (form, comp, arm, "row", worst[0], "col", worst[1], err[worst], bound[worst], ratio.max())
    print(f"[attention {form} {comp} {arm}] max |err| / bound = {ratio.max():.3f}")

    if max(lens) >= 2:
        _must_fail("last key dropped", np.abs(got[:T] - AO.attention(qkv, cu, form, table, drop_last_key=True)) <= bound)
        if form == "t5":
            _must_fail("relative position negated",
                       np.abs(got[:T] - AO.attention(qkv, cu, form, table, rel_sign=-1)) <= bound)
    if form == "bert" and arm != "equal":                  # equal scores make the scale invisible
        _must_fail("no 1/8 scale", np.abs(got[:T] - AO.attention(qkv, cu, form, table, scale=1.0)) <= bound)
    if form == "t5":
        _must_fail("neighbouring head's bias", np.abs(got[:T] - AO.attention(qkv, cu, form, table, head_shift=1)) <= bound)

    if comp in ("every_length", "zero_length_inside", "stress") and arm in ("gauss", "dominant_last"):
        for i, S in enumerate(lens):                       # the same sequence alone: bit-equal rows
            if S == 0 or (i % 3 and S not in (32, 33, 512)):
                continue
            alone = _attention(form, qkv[cu[i]:cu[i + 1]], [0, S], S)
            assert np.array_equal(alone[:S].view(np.uint16), got[cu[i]:cu[i + 1]].astype(np.float16).view(np.uint16)), (i, S)


def test_attention_refusals_that_need_a_handle():
    from retrieval_scaling_b200 import _lib
    from retrieval_scaling_b200.encoder import B200T5Encoder
    m, _ = _attention_model("bert")
    qkv = torch.zeros((600, 2304), dtype=torch.float16, device="cuda")
    ctx = torch.zeros((600, 768), dtype=torch.float16, device="cuda")
    cu = torch.tensor([0, 513], dtype=torch.int32, device="cuda")
    args = (ctypes.c_void_p(qkv.data_ptr()), ctypes.c_void_p(cu.data_ptr()), 1, 513, 513, ctypes.c_void_p(ctx.data_ptr()),
            _stream())
    assert _L().rsb_bert_attention(m._h, *args) == _lib.RSB_ERR_UNSUPPORTED
    t5 = B200T5Encoder(T5_CFG)                              # bucket table uploaded, relative_attention_bias not loaded
    a2 = list(args)
    a2[2:5] = [1, 20, 20]
    assert _L().rsb_bert_attention(t5._h, *a2) == _lib.RSB_ERR_STATE
    assert b"relative_attention_bias" in _L().rsb_bert_last_error()


# ---------------------------------------------------------------------------------------------------------------
# GEMM
# ---------------------------------------------------------------------------------------------------------------
GEMM_M = [1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257, 4097, 41000, 262144]
GEMM_NK = [(2304, 768), (768, 768), (3072, 768), (768, 3072), (128, 64), (128, 128), (2304, 3072), (3072, 64)]
# the reader's (N, K) at Llama-2-7B / Llama-3-8B / Llama-2-13B width, each at a small or partial M: q|k|v (MHA, GQA
# 32:8), gate|up, down, LM head (Llama-2, Llama-3)
READER_NK = [(12288, 4096), (6144, 4096), (22016, 4096), (28672, 4096), (27648, 5120), (4096, 11008), (4096, 14336),
             (5120, 13824), (32000, 4096), (128256, 4096)]
READER_M = [1, 65, 129, 7, 200, 255, 1, 63, 129, 130]


def _gemm_nk(i, M):
    if i >= len(GEMM_M):
        return READER_NK[i - len(GEMM_M)]
    if M == 262144:
        return 768, 3072                                    # FFN2 of 512 passages x 512 tokens
    if M == 41000:
        return 3072, 768                                    # FFN1 of 10k NQ-length queries
    return GEMM_NK[i % len(GEMM_NK)]


@pytest.mark.parametrize("i,M", list(enumerate(GEMM_M)) + [(len(GEMM_M) + j, M) for j, M in enumerate(READER_M)])
def test_gemm_per_element_bound(i, M):
    """rsb_gemm_f16 for epilogues bias / GELU / residual / ReLU, each in both row-tile orders (RSB_GEMM_REVERSED is the
    order FFN2 runs in), and the residual epilogue in place (C == residual, as the reader's o_proj and down_proj run it)
    in both orders, against fp64 of the same fp16 operands, per element:
        pre = A W^T + bias (fp64); e = 2 K 2^-24 (|A| |W|^T) + 2^-24 |pre|   (fp32 accumulation with truncation, the
                                                                          fp32 bias add)
        bias / ReLU:  |out - f(pre)| <= e + 1/2 ulp(f(pre) + e)
        GELU:         |out - gelu(pre)| <= 1.13 e + 1.5 ulp(gelu(pre) + 1.13 e)   (|gelu'| <= 1.13; the kernel's
                                                                          restated GELU is within 1 ulp of erf's)
        residual:     |out - (pre + r)| <= e + 1/2 ulp(pre + e) + 1/2 ulp(pre + r + 2e)   (rounded, then added in half)
    The encoder's shapes and the reader's (N, K) at small and partial M.  Large M is compared in row chunks, the fp64
    product once per chunk for every epilogue.  The comparison must reject the reference shifted by one row."""
    from retrieval_scaling_b200 import _lib
    N, K = _gemm_nk(i, M)
    g = torch.Generator(device="cuda").manual_seed(1000 + i)
    A = (torch.randn(M, K, generator=g, device="cuda") * 0.5).half()
    W = (torch.randn(N, K, generator=g, device="cuda") * (1.0 / K ** 0.5)).half()
    b = (torch.randn(N, generator=g, device="cuda") * 0.1).half()
    R = (torch.randn(M, N, generator=g, device="cuda") * 0.5).half()
    outs = {}
    for epi in (0, 1, 2, 3, "in_place"):
        for rev in (0, _lib.GEMM_REVERSED):
            if epi == "in_place":
                C = R.clone()
                res = C
            else:
                C = torch.full((M, N), float("nan"), dtype=torch.float16, device="cuda")
                res = R
            rc = _L().rsb_gemm_f16(ctypes.c_void_p(A.data_ptr()), ctypes.c_void_p(W.data_ptr()), ctypes.c_void_p(b.data_ptr()),
                                   ctypes.c_void_p(res.data_ptr()), ctypes.c_void_p(C.data_ptr()), M, N, K,
                                   (2 if epi == "in_place" else epi) | rev, _stream())
            assert rc == 0, _L().rsb_bert_last_error()
            outs[(epi, rev)] = C
    torch.cuda.synchronize()
    chunk = max(1, (1 << 26) // max(N, K))
    Wd, bd = W.double(), b.double()
    Wa = Wd.abs()
    worst = {}
    shifted_ok = {key: True for key in outs}
    for r0 in range(0, M, chunk):
        r1 = min(M, r0 + chunk)
        Ad = A[r0:r1].double()
        pre = Ad @ Wd.T + bd
        e = 2 * K * 2.0 ** -24 * (Ad.abs() @ Wa.T) + 2.0 ** -24 * pre.abs()
        for epi in (0, 1, 2, 3):
            if epi == 0:
                ref, bnd = pre, e + 0.5 * _ulp16(pre.abs() + e)
            elif epi == 3:
                ref = pre.clamp_min(0)
                bnd = e + 0.5 * _ulp16(ref + e)
            elif epi == 1:
                ref = F.gelu(pre)
                bnd = 1.13 * e + 1.5 * _ulp16(ref.abs() + 1.13 * e)
            else:
                ref = pre + R[r0:r1].double()
                bnd = e + 0.5 * _ulp16(pre.abs() + e) + 0.5 * _ulp16(ref.abs() + 2 * e)
            for key, C in outs.items():
                if (2 if key[0] == "in_place" else key[0]) != epi:
                    continue
                out = C[r0:r1].double()
                assert torch.isfinite(out).all(), (key, r0)
                ratio = ((out - ref).abs() / bnd).max().item()
                worst[key[0]] = max(worst.get(key[0], 0.0), ratio)
                assert ratio <= 1.0, (M, N, K, key, r0, ratio)
                if r1 - r0 >= 2:
                    shifted_ok[key] &= bool(((out[1:] - ref[:-1]).abs() <= bnd[1:]).all().item())
    if M >= 2:
        for key, ok in shifted_ok.items():
            _must_fail(f"reference shifted by one row {key}", ok)
    worst = max(worst.values())
    print(f"[gemm M={M} N={N} K={K}] max |err| / bound = {worst:.3f}")


# ---------------------------------------------------------------------------------------------------------------
# the forward, token by token
# ---------------------------------------------------------------------------------------------------------------
TOKEN_LENS = [1, 2, 15, 16, 17, 31, 32, 33, 63, 64, 65, 97, 128, 129, 257, 385, 512]


def _padded_batch(rng, lens, vocab):
    S = int(max(lens))
    ids = torch.from_numpy(rng.integers(3, vocab, (len(lens), S)))
    mask = (torch.arange(S)[None, :] < torch.as_tensor(lens)[:, None]).long()
    return (ids * mask).cuda(), mask.cuda()


def _unpad_rows(x, mask):
    return x[mask.bool()]


@pytest.mark.parametrize("arch", ["bert", "t5"])
@pytest.mark.parametrize("layers", [1, 2])
def test_forward_token_rows_against_fp16_and_fp32_oracles(arch, layers):
    """Every token row of the final hidden states (RSB_POOL_TOKENS) against the torch oracles: cosine >= 0.9999 per
    token against both (the existing encoder bar, per token instead of per pooled vector), and per row max |err|
    against fp32 <= 2x the fp16 oracle's own max |err| against fp32 for that row, with a floor of 1 fp16 ulp of the
    row's largest element (the output is fp16).  The comparison rejects the fp32 rows shifted by one within each
    sequence."""
    from retrieval_scaling_b200.encoder import B200Contriever, B200T5Encoder
    rng = np.random.default_rng(layers * 10 + (arch == "t5"))
    if arch == "bert":
        cfg = dict(BERT_CFG, num_hidden_layers=layers)
        sd = BO.seeded_state_dict(cfg, 20 + layers)
        m = B200Contriever(cfg)
    else:
        cfg = dict(T5_CFG, num_layers=layers)
        sd = T5O.seeded_state_dict(cfg, 20 + layers, head=False)
        m = B200T5Encoder(cfg)
    assert m.load_state_dict(sd) == []
    ids, mask = _padded_batch(rng, TOKEN_LENS, cfg["vocab_size"])
    tok, cu = m.hidden_states(input_ids=ids, attention_mask=mask)
    assert tok.shape == (int(mask.sum()), 768)
    with torch.no_grad():
        if arch == "bert":
            def hidden(dtype):
                return BO.bert_hidden(sd, cfg, ids, mask, None, dtype)
        else:
            def hidden(dtype):
                return T5O.t5_hidden(sd, cfg, ids, mask, dtype)
        h16 = _unpad_rows(hidden(torch.float16), mask).double()
        h32 = _unpad_rows(hidden(torch.float32), mask).double()
    got = tok.double()
    cos16 = F.cosine_similarity(got, h16, dim=1)
    cos32 = F.cosine_similarity(got, h32, dim=1)
    assert cos16.min().item() >= 0.9999 and cos32.min().item() >= 0.9999, (cos16.min().item(), cos32.min().item())
    err = (got - h32).abs().max(1).values
    cost = (h16 - h32).abs().max(1).values
    floor = _ulp16(h32.abs().max(1).values)
    lim = torch.maximum(2 * cost, floor)
    assert (err <= lim).all(), ((err / lim).max().item(), int(torch.argmax(err / lim)))
    print(f"[tokens {arch} L={layers}] min cos fp16 {cos16.min().item():.6f} fp32 {cos32.min().item():.6f}, "
          f"max err/(2x fp16 cost) {(err / lim).max().item():.3f}")
    cuh = cu.cpu().numpy()
    shifted = torch.cat([torch.roll(h32[cuh[b]:cuh[b + 1]], 1, 0) for b in range(len(cuh) - 1)])
    _must_fail("token rows shifted by one", (F.cosine_similarity(got, shifted, dim=1) >= 0.9999).cpu().numpy())


# ---------------------------------------------------------------------------------------------------------------
# the head: pooling -> Dense -> Normalize, each against fp64 of the GPU's previous step
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch", ["bert", "t5"])
def test_head_chain_against_fp64_of_the_previous_gpu_step(arch):
    """Mean pooling within 1/2 ulp of the fp64 mean of the GPU's token rows plus the fp32 accumulation
    (S 2^-24 mean|x|) and the rounding of the fp32 division (1/2 ulp); the CLS row bit-equal to token row 0; a
    zero-length sequence pools to zeros; Dense within the GEMM bound (K = 768) of fp64 Dense of the GPU's pooled rows;
    Normalize within 1/2 ulp + 2^-23 relative of x / fp16(||x||) for one of the two fp16 neighbours of the fp64 norm
    (the kernel's fp32 norm may round to either when the exact one is near a midpoint), norms within 2^-10 of 1.
    The mean comparison rejects a mean over the padded length."""
    from retrieval_scaling_b200 import _lib
    from retrieval_scaling_b200.encoder import B200Contriever, B200T5Encoder
    rng = np.random.default_rng(5 if arch == "bert" else 6)
    if arch == "bert":
        sd = BO.seeded_state_dict(BERT_CFG, 31)
        g = torch.Generator().manual_seed(31)
        sd["dense.weight"], sd["dense.bias"] = torch.randn(768, 768, generator=g) * 0.04, torch.randn(768, generator=g) * 0.02
        m, vocab = B200Contriever(BERT_CFG, dense=True, normalize=True), BERT_CFG["vocab_size"]
    else:
        sd = T5O.seeded_state_dict(T5_CFG, 31)
        m, vocab = B200T5Encoder(T5_CFG, dense=True, normalize=True), T5_CFG["vocab_size"]
    assert m.load_state_dict(sd) == []
    lens = [5, 0, 1, 32, 33, 0, 200, 512, 17, 0]
    cu = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)).cuda()
    T = int(sum(lens))
    ids = torch.from_numpy(rng.integers(3, vocab, T).astype(np.int32)).cuda()
    run = lambda flags: m.forward_varlen(ids, cu, max(lens), pool_flags=flags).double()   # noqa: E731
    tok = run(_lib.POOL_TOKENS)
    mean = run(_lib.POOL_MEAN)
    cls = run(_lib.POOL_CLS)
    dense = run(_lib.POOL_MEAN | _lib.POOL_DENSE)
    norm = run(_lib.POOL_MEAN | _lib.POOL_DENSE | _lib.POOL_NORMALIZE)
    cuh = cu.cpu().numpy()
    worst = {}
    mean_ok_padded = []
    for b, S in enumerate(lens):
        rows = tok[cuh[b]:cuh[b + 1]]
        if S == 0:
            assert (mean[b] == 0).all() and (cls[b] == 0).all(), b
            continue
        ref = rows.mean(0)
        bnd = _ulp16(ref) + S * 2.0 ** -24 * rows.abs().mean(0)       # 1/2 ulp output + 1/2 ulp division + fp32 sum
        worst["mean"] = max(worst.get("mean", 0), ((mean[b] - ref).abs() / bnd).max().item())
        assert ((mean[b] - ref).abs() <= bnd).all(), (b, S)
        mean_ok_padded.append(((mean[b] - rows.sum(0) / max(lens)).abs() <= bnd).cpu().numpy())
        assert torch.equal(cls[b], rows[0]), b
    _must_fail("mean over the padded length", np.concatenate(mean_ok_padded))
    Wd = sd["dense.weight"].cuda().half().double()
    bd = sd["dense.bias"].cuda().half().double()
    pre = mean @ Wd.T + bd
    e = 2 * 768 * 2.0 ** -24 * (mean.abs() @ Wd.abs().T) + 2.0 ** -24 * pre.abs()
    bnd = e + 0.5 * _ulp16(pre.abs() + e)
    worst["dense"] = ((dense - pre).abs() / bnd).max().item()
    assert ((dense - pre).abs() <= bnd).all()
    nrm = dense.norm(dim=1, keepdim=True)
    errs = []
    for d in (AO.round16(nrm.cpu().numpy() * (1 - 2.0 ** -20)), AO.round16(nrm.cpu().numpy() * (1 + 2.0 ** -20))):
        ref = dense / torch.from_numpy(np.maximum(d, 1e-12)).cuda()
        errs.append((norm - ref).abs() / (0.5 * _ulp16(ref) + 2.0 ** -23 * ref.abs()))
    ratio = torch.minimum(errs[0].max(1).values, errs[1].max(1).values)
    worst["normalize"] = ratio.max().item()
    assert (ratio <= 1.0).all(), ratio.max().item()
    assert ((norm.norm(dim=1) - 1).abs() <= 2.0 ** -10).all()
    print(f"[head {arch}] max |err| / bound: {worst}")


def test_tokens_bit_refuses_every_combination():
    from retrieval_scaling_b200 import _lib
    m, _ = _attention_model("bert")
    cu = torch.tensor([0, 3], dtype=torch.int32, device="cuda")
    ids = torch.ones(3, dtype=torch.int32, device="cuda")
    for extra in (_lib.POOL_CLS, _lib.POOL_DENSE, _lib.POOL_NORMALIZE, _lib.POOL_DENSE | _lib.POOL_NORMALIZE):
        with pytest.raises(ValueError, match="RSB_POOL_TOKENS"):
            m.forward_varlen(ids, cu, 3, pool_flags=_lib.POOL_TOKENS | extra)
