"""GPU parity of the sentence-transformers retrievers: the T5 encoder (`B200T5Encoder`, GTR-T5) and the BERT-base + head
stack (e5) on librsb against (a) the fp32 goldens of `transformers.T5EncoderModel` and (b) the torch oracle run in fp16
on the GPU (the like-for-like of `SentenceTransformer(name).half()`, reference src/search.py:257-258).  Bar: cosine
>= 0.9999 per row, the existing encoder bar."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import bert_oracle as BO
from oracle import t5_oracle as T

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CFG2 = dict(T.T5_CONFIG, num_layers=2, vocab_size=2048)


def _case(name):
    z = np.load(os.path.join(GOLD, name + ".npz"))
    return z, {k[4:]: z[k].item() for k in z.files if k.startswith("cfg_")}


def _model(cfg, sd, pooling="average", dense=True, normalize=True):
    from retrieval_scaling_b200.encoder import B200T5Encoder
    m = B200T5Encoder(cfg, pooling, dense=dense, normalize=normalize)
    assert m.load_state_dict(sd) == []
    m.require_all_weights()
    return m


def _cos(a, b):
    return F.cosine_similarity(a.float().cpu(), b.float().cpu(), dim=1).min().item()


def _batch(rng, lens, vocab):
    S = int(max(lens))
    ids = torch.from_numpy(rng.integers(3, vocab, (len(lens), S)))
    mask = (torch.arange(S)[None, :] < torch.as_tensor(lens)[:, None]).long()
    return (ids * mask).cuda(), mask.cuda()


@pytest.mark.parametrize("name", ["encoder_t5_l2", "encoder_t5_l12"])
def test_t5_matches_transformers_golden_and_fp16_oracle(name):
    z, cfg = _case(name)
    sd = T.seeded_state_dict(cfg, int(z["seed"]))
    ids, mask = torch.from_numpy(z["input_ids"]).cuda(), torch.from_numpy(z["attention_mask"]).cuda()
    with torch.no_grad():
        tok16 = T.t5_hidden(sd, cfg, ids, mask, dtype=torch.float16)
    for key, pooling, head in (("out_mean", "average", False), ("out_cls", "cls", False), ("out_head", "average", True)):
        out = _model(cfg, sd, pooling, dense=head, normalize=head)(input_ids=ids, attention_mask=mask)
        assert out.dtype == torch.float16 and tuple(out.shape) == (ids.shape[0], 768)
        half = T.st_head(tok16, mask, pooling, sd["dense.weight"].cuda() if head else None,
                         sd["dense.bias"].cuda() if head else None, head)
        gold = torch.from_numpy(z[key])
        assert torch.isfinite(out).all()
        # against fp32, the bar is 0.9999 or what fp16 itself costs (the first-token row of 12 layers: ~2e-4)
        fp16_cost = _cos(half, gold)
        assert _cos(out, half) >= 0.9999, (key, _cos(out, half))
        assert _cos(out, gold) >= min(0.9999, fp16_cost - 1e-4), (key, _cos(out, gold), fp16_cost)


@pytest.mark.parametrize("kind", ["queries", "passages", "mixed"])
def test_t5_lengths_against_fp16_and_fp32_oracle(kind):
    """<= 32 tokens: the warp-per-(sequence, head) kernel; 33..512: the flash kernel; mixed batches take both."""
    rng = np.random.default_rng({"queries": 1, "passages": 2, "mixed": 3}[kind])
    if kind == "queries":
        lens = rng.integers(1, 33, 70)
        lens[:3] = (1, 32, 2)
    elif kind == "passages":
        lens = rng.integers(33, 513, 6)
        lens[:2] = (512, 33)
    else:
        lens = np.concatenate([rng.integers(1, 33, 20), rng.integers(33, 300, 5), [512]])
    sd = T.seeded_state_dict(CFG2, 5)
    ids, mask = _batch(rng, lens, CFG2["vocab_size"])
    out = _model(CFG2, sd)(input_ids=ids, attention_mask=mask)
    with torch.no_grad():
        half = T.t5_st_forward(sd, CFG2, ids, mask, dtype=torch.float16)
        full = T.t5_st_forward(sd, CFG2, ids, mask, dtype=torch.float32)
    assert _cos(out, half) >= 0.9999 and _cos(out, full) >= 0.9999, (_cos(out, half), _cos(out, full))


def test_t5_batch_invariance():
    """The un-padded token stream: a sequence's embedding does not depend on the rest of its batch."""
    rng = np.random.default_rng(11)
    lens = np.concatenate([rng.integers(1, 33, 30), [40, 200, 512, 7]])
    sd = T.seeded_state_dict(CFG2, 6)
    ids, mask = _batch(rng, lens, CFG2["vocab_size"])
    m = _model(CFG2, sd)
    full = m(input_ids=ids, attention_mask=mask)
    for i in (0, 5, 30, 31, 32, 33):
        n = int(lens[i])
        alone = m(input_ids=ids[i:i + 1, :n], attention_mask=mask[i:i + 1, :n])
        assert torch.equal(alone[0], full[i]), i


def _gemm(A, W, bias, epi):
    from retrieval_scaling_b200 import _lib
    L = _lib.lib()
    C = torch.empty((A.shape[0], W.shape[0]), dtype=torch.float16, device="cuda")
    rc = L.rsb_gemm_f16(ctypes.c_void_p(A.data_ptr()), ctypes.c_void_p(W.data_ptr()), ctypes.c_void_p(bias.data_ptr()),
                        None, ctypes.c_void_p(C.data_ptr()), A.shape[0], W.shape[0], A.shape[1], epi,
                        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, L.rsb_bert_last_error()
    torch.cuda.synchronize()
    return C


@pytest.mark.parametrize("M,N,K", [(1, 3072, 768), (300, 3072, 768), (1000, 768, 768)])
def test_relu_epilogue_matches_torch(M, N, K):
    g = torch.Generator(device="cuda").manual_seed(M + N)
    A = (torch.randn(M, K, generator=g, device="cuda") * 0.5).half()
    W = (torch.randn(N, K, generator=g, device="cuda") * 0.05).half()
    b = (torch.randn(N, generator=g, device="cuda") * 0.1).half()
    ref = torch.relu(A.float() @ W.float().T + b.float())
    out = _gemm(A, W, b, 3).float()
    assert (out - ref).abs().max().item() < 2e-3 * max(1.0, ref.abs().max().item())
    assert ((out == 0) == (ref.half().float() == 0)).float().mean().item() > 0.999


def test_t5_fp16_clamp_rule():
    """Residual adds that overflow fp16 (one feed-forward site, one attention site): HF clamps the whole batch to
    +-(65504 - 1000) and continues; without the clamp the RMS norm would turn the inf into NaN.  Equal-length
    sequences, so HF's condition over the padded tensor and this one over the real tokens agree."""
    sd = T.seeded_state_dict(CFG2, 8)
    sd["encoder.block.0.layer.1.DenseReluDense.wo.weight"] *= 3e4
    sd["encoder.block.1.layer.0.SelfAttention.o.weight"] *= 3e4
    rng = np.random.default_rng(9)
    for lens in ([20] * 16, [200] * 4):
        ids, mask = _batch(rng, lens, CFG2["vocab_size"])
        for head in (False, True):
            out = _model(CFG2, sd, dense=head, normalize=head)(input_ids=ids, attention_mask=mask)
            with torch.no_grad():
                tok = T.t5_hidden(sd, CFG2, ids, mask, dtype=torch.float16)
                assert not torch.isinf(tok).any() and torch.isfinite(tok).all()
                half = T.st_head(tok, mask, "average", sd["dense.weight"].cuda() if head else None,
                                 sd["dense.bias"].cuda() if head else None, head)
            assert torch.isfinite(out).all()
            assert _cos(out, half) >= 0.9999, (lens[0], head, _cos(out, half))
    # the overflow really happens: the first feed-forward's output alone is past the fp16 range
    with torch.no_grad():
        x = torch.randn(4, 768, device="cuda").half()
        wi = sd["encoder.block.0.layer.1.DenseReluDense.wi.weight"].cuda().half()
        wo = sd["encoder.block.0.layer.1.DenseReluDense.wo.weight"].cuda().half()
        assert torch.isinf(F.linear(F.relu(F.linear(x, wi)), wo)).any()


def test_bert_with_sentence_transformers_head():
    """The e5 stack: BERT-base, mean pooling, Dense, Normalize (and each head piece alone) against the oracle."""
    from retrieval_scaling_b200 import _lib
    from retrieval_scaling_b200.encoder import B200Contriever
    cfg = dict(hidden_size=768, num_hidden_layers=2, num_attention_heads=12, intermediate_size=3072, vocab_size=3000,
               max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12)
    sd = BO.seeded_state_dict(cfg, 4)
    g = torch.Generator().manual_seed(4)
    dw, db = torch.randn(768, 768, generator=g) * 0.04, torch.randn(768, generator=g) * 0.02
    rng = np.random.default_rng(4)
    ids, mask = _batch(rng, np.concatenate([rng.integers(1, 33, 12), [100, 512]]), 3000)
    with torch.no_grad():
        pooled = {p: BO.bert_forward(sd, cfg, ids, mask, None, p, dtype=torch.float16) for p in ("average", "cls")}
    for pooling in ("average", "cls"):
        for dense, normalize in ((True, True), (True, False), (False, True)):
            m = B200Contriever(cfg, pooling, dense=dense, normalize=normalize)
            m.load_state_dict(dict(sd, **({"dense.weight": dw, "dense.bias": db} if dense else {})))
            m.require_all_weights()
            out = m(input_ids=ids, attention_mask=mask)
            ref = pooled[pooling]
            if dense:
                ref = F.linear(ref, dw.cuda().half(), db.cuda().half())
            if normalize:
                ref = F.normalize(ref, p=2, dim=1)
                assert torch.allclose(out.float().norm(dim=1), torch.ones(len(out), device="cuda"), atol=2e-3)
            assert _cos(out, ref) >= 0.9999, (pooling, dense, normalize, _cos(out, ref))
    # a head flag without its weights is a state error, not uninitialised memory
    m = B200Contriever(cfg, "average", dense=True)
    m.load_state_dict(sd)
    with pytest.raises(KeyError, match="dense.weight"):
        m.require_all_weights()
    with pytest.raises(_lib.RsbError, match="dense.weight"):
        m(input_ids=ids, attention_mask=mask)


def test_t5_forward_before_bias_table_is_refused():
    from retrieval_scaling_b200 import _lib
    from retrieval_scaling_b200.encoder import B200T5Encoder
    sd = T.seeded_state_dict(CFG2, 3)
    m = B200T5Encoder(CFG2, "average")
    m.load_state_dict({k: v for k, v in sd.items() if "relative_attention_bias" not in k and not k.startswith("dense.")})
    ids, mask = _batch(np.random.default_rng(0), [5, 9], CFG2["vocab_size"])
    with pytest.raises(_lib.RsbError, match="relative_attention_bias"):
        m(input_ids=ids, attention_mask=mask)
    bad = torch.full((1023,), 40, dtype=torch.int32, device="cuda")           # bucket >= num_buckets
    rc = m.L.rsb_bert_load(m._h, b"relative_position_bucket", ctypes.c_void_p(bad.data_ptr()), 1023,
                           ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == _lib.RSB_ERR_INVALID


@pytest.fixture(scope="module")
def fx(tmp_path_factory):
    from golden import st_fixture
    return st_fixture.build(str(tmp_path_factory.mktemp("st")))


def test_embed_queries_and_passage_task_on_fixture_directories(fx, tmp_path):
    """search.load_query_encoder / embed_queries and the passage-embedding task end to end on the two fixture
    directories: loaded from disk, tokenised by their own tokenizers, against the fp32 oracle."""
    import pickle

    import transformers

    from retrieval_scaling_b200 import config as C
    from retrieval_scaling_b200 import embed as E
    from retrieval_scaling_b200 import search as S
    queries = ["who wrote the origin of species", "What is the capital of Australia?", "  b200 hbm3e bandwidth ",
               "a", "largest moon of saturn " * 40]
    passages = [{"id": i, "title": f"title {i}", "text": "the tallest mountain in south america " * (1 + i % 60)}
                for i in range(130)]
    for k in ("t5", "bert"):
        d, sd, cfg = fx[k]["dir"], fx[k]["state_dict"], fx[k]["config"]
        tok = transformers.AutoTokenizer.from_pretrained(d, local_files_only=True)

        def oracle(texts):
            enc = tok([t.strip() for t in texts], return_tensors="pt", padding=True, truncation=True, max_length=256)
            ids, mask = enc["input_ids"].cuda(), enc["attention_mask"].cuda()
            with torch.no_grad():
                if k == "t5":
                    return T.t5_st_forward(sd, cfg, ids, mask)
                tt = enc["token_type_ids"].cuda()
                return F.normalize(BO.bert_forward(sd, cfg, ids, mask, tt, "average"), p=2, dim=1)

        qcfg = C.DictConfig({"model": {"query_encoder": d}, "datastore": {"index": {}}})
        model, tokenizer = S.load_query_encoder(qcfg)
        assert tokenizer is None
        args = C.DictConfig({"per_gpu_batch_size": 2, "question_maxlength": 32, "lowercase": False, "normalize_text": False})
        q = S.embed_queries(args, queries, model, tokenizer, d)
        assert q.shape == (5, 768) and q.dtype == np.float16
        assert _cos(torch.from_numpy(q), oracle(queries)) >= 0.9999
        root = tmp_path / k
        os.makedirs(root / "passages")
        with open(root / "passages" / "raw_passages-0-of-1.jsonl", "w") as f:
            for p in passages:
                f.write(__import__("json").dumps(p) + "\n")
        ecfg = C.DictConfig({"model": {}, "datastore": {"embedding": {
            "model_name_or_path": d, "per_gpu_batch_size": 64, "passage_maxlength": 512, "no_title": False,
            "lowercase": False, "normalize_text": False, "shard_ids": [0], "num_shards": 1,
            "passages_dir": str(root / "passages"), "embedding_dir": str(root / "emb"), "prefix": "passages"}}})
        paths = E.generate_passage_embeddings(ecfg)
        ids, emb = pickle.load(open(paths[0], "rb"))
        assert ids == list(range(130)) and emb.shape == (130, 768)
        sel = [0, 1, 59, 63, 64, 129]
        ref = oracle([passages[i]["title"] + " " + passages[i]["text"] for i in sel])
        assert _cos(torch.from_numpy(emb[sel]), ref) >= 0.9999
