"""GPU parity of the query encoder: the tensor-core (wgmma/TMA) GEMM against torch.matmul (the test keeps the name of
the tcgen05 kernel it was written for), and the full BERT forward against
(a) golden outputs of the reference's own Contriever class and (b) the torch oracle run in fp16 on the GPU
(the like-for-like of `query_encoder.half()`, src/search.py:257-258).  Tolerances: cosine >= 0.9999 and
max |err| within fp16 noise (SURVEY.md App. C.4)."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import bert_oracle as BO

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _gemm(A, W, bias, res, epi):
    from retrieval_scaling_b200 import _lib
    L = _lib.lib()
    M, K = A.shape
    N = W.shape[0]
    C = torch.empty((M, N), dtype=torch.float16, device="cuda")
    rc = L.rsb_gemm_f16(ctypes.c_void_p(A.data_ptr()), ctypes.c_void_p(W.data_ptr()), ctypes.c_void_p(bias.data_ptr()),
                        ctypes.c_void_p(res.data_ptr() if res is not None else 0), ctypes.c_void_p(C.data_ptr()),
                        M, N, K, epi, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0, L.rsb_bert_last_error()
    torch.cuda.synchronize()
    return C


@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (128, 128, 768), (300, 768, 768), (1, 2304, 768), (1000, 3072, 768),
                                   (257, 768, 3072)])
def test_tcgen05_gemm_matches_torch(M, N, K):
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    A = (torch.randn(M, K, generator=g, device="cuda") * 0.5).half()
    W = (torch.randn(N, K, generator=g, device="cuda") * 0.05).half()
    b = (torch.randn(N, generator=g, device="cuda") * 0.1).half()
    R = (torch.randn(M, N, generator=g, device="cuda") * 0.5).half()
    ref = A.float() @ W.float().T + b.float()
    scale = ref.abs().max().item()
    out = _gemm(A, W, b, None, 0).float()
    assert (out - ref).abs().max().item() < 2e-3 * max(1.0, scale), (out - ref).abs().max().item()
    out = _gemm(A, W, b, None, 1).float()
    assert (out - torch.nn.functional.gelu(ref)).abs().max().item() < 2e-3 * max(1.0, scale)
    out = _gemm(A, W, b, R, 2).float()
    assert (out - (ref + R.float())).abs().max().item() < 2e-3 * max(1.0, scale)


def _case(name):
    z = np.load(os.path.join(GOLD, name + ".npz"))
    cfg = {k[4:]: (float(z[k]) if k == "cfg_layer_norm_eps" else int(z[k])) for k in z.files if k.startswith("cfg_")}
    return z, cfg


@pytest.mark.parametrize("name", ["encoder_l2", "encoder_l12"])
def test_encoder_matches_reference_golden_and_fp16_oracle(name):
    from retrieval_scaling_b200.encoder import B200Contriever
    z, cfg = _case(name)
    sd = BO.seeded_state_dict(cfg, int(z["seed"]))
    ids, mask, tt = (torch.from_numpy(z[k]).cuda() for k in ("input_ids", "attention_mask", "token_type_ids"))
    for pooling in ("average", "cls"):
        model = B200Contriever(cfg, pooling)
        assert model.load_state_dict(sd) == []
        model = model.eval().half()
        out = model(input_ids=ids, attention_mask=mask, token_type_ids=tt)
        assert out.dtype == torch.float16 and tuple(out.shape) == (ids.shape[0], 768)
        out = out.float().cpu()
        gold = torch.from_numpy(z["out_" + pooling])                      # reference class, fp32
        with torch.no_grad():
            half = BO.bert_forward(sd, cfg, ids, mask, tt, pooling, dtype=torch.float16).float().cpu()  # `.half()` like-for-like
        cos_gold = torch.nn.functional.cosine_similarity(out, gold, dim=1).min().item()
        cos_half = torch.nn.functional.cosine_similarity(out, half, dim=1).min().item()
        err_gold = (out - gold).abs().max().item()
        err_half_ref = (half - gold).abs().max().item()                   # what fp16 itself costs
        assert cos_gold >= 0.9999 and cos_half >= 0.9999, (cos_gold, cos_half)
        assert err_gold <= max(2.0 * err_half_ref, 2e-2), (err_gold, err_half_ref)


def test_encoder_varlen_and_launch_count():
    from retrieval_scaling_b200.encoder import B200Contriever, random_state_dict
    cfg = dict(hidden_size=768, num_hidden_layers=2, num_attention_heads=12, intermediate_size=3072, vocab_size=3000,
               max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12)
    sd = random_state_dict(cfg, 3)
    model = B200Contriever(cfg, "average")
    model.load_state_dict(sd)
    rng = np.random.default_rng(5)
    B, S = 70, 64
    lens = rng.integers(1, S + 1, B); lens[3] = 1; lens[4] = S
    ids = torch.from_numpy(rng.integers(1, 3000, (B, S))).cuda()
    mask = (torch.arange(S)[None, :] < torch.from_numpy(lens)[:, None]).long().cuda()
    out = model(input_ids=ids * mask, attention_mask=mask).float().cpu()
    with torch.no_grad():
        ref = BO.bert_forward(sd, cfg, ids * mask, mask, None, "average", dtype=torch.float32).float().cpu()
    cos = torch.nn.functional.cosine_similarity(out, ref, dim=1)
    assert cos.min().item() >= 0.9999, cos.min().item()
    # embed + pool + the list of sequences > 32 tokens (once per forward), and per layer 4 GEMMs + 2 LayerNorms +
    # attention (tensor-core kernel for sequences <= 32 tokens plus the long-sequence kernel because this batch also
    # holds sequences up to 64 tokens)
    assert model.launches == 3 + (6 + 2) * 2
    with pytest.raises(NotImplementedError):
        B200Contriever(dict(cfg, hidden_size=1024))


@pytest.mark.parametrize("B,S,min_len", [(6, 512, 300), (24, 200, 33), (9, 129, 100)])
def test_encoder_passage_length_sequences_tensor_core_attention(B, S, min_len):
    """Passage side (reference src/embed.py:24-94, passage_maxlength up to 512): sequences of 33..512 tokens run through
    the flash-style tensor-core attention kernel; output vs the fp32 torch oracle of the reference encoder."""
    from retrieval_scaling_b200.encoder import B200Contriever, random_state_dict
    cfg = dict(hidden_size=768, num_hidden_layers=2, num_attention_heads=12, intermediate_size=3072, vocab_size=3000,
               max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12)
    sd = random_state_dict(cfg, 7)
    rng = np.random.default_rng(B + S)
    lens = rng.integers(min_len, S + 1, B)
    lens[0], lens[-1] = S, min_len
    if B > 8:
        lens[1], lens[2] = 5, 32                      # short sequences in the same batch take the other kernel
    ids = torch.from_numpy(rng.integers(1, 3000, (B, S))).cuda()
    mask = (torch.arange(S)[None, :] < torch.from_numpy(lens)[:, None]).long().cuda()
    with torch.no_grad():
        ref = {p: BO.bert_forward(sd, cfg, ids * mask, mask, None, p, dtype=torch.float32).float().cpu() for p in ("average", "cls")}
    for pooling in ("average", "cls"):
        model = B200Contriever(cfg, pooling)
        model.load_state_dict(sd)
        out = model(input_ids=ids * mask, attention_mask=mask).float().cpu()
        cos = torch.nn.functional.cosine_similarity(out, ref[pooling], dim=1)
        assert cos.min().item() >= 0.9999, (pooling, cos.min().item())
        assert (out - ref[pooling]).abs().max().item() <= 3e-2 * ref[pooling].abs().max().item()


def test_embed_passages_on_gpu_matches_oracle_and_keeps_order(tmp_path):
    """`embed_passages` (reference src/embed.py:24-94) at the reference's passage settings (batch 512, title + text,
    truncation to passage_maxlength) on the GPU: ids in order, embeddings equal to the torch oracle's, host copies
    made batch by batch."""
    from retrieval_scaling_b200 import config as C
    from retrieval_scaling_b200.embed import embed_passages
    from retrieval_scaling_b200.encoder import B200Contriever, random_state_dict

    class Tok:                                            # whitespace tokens hashed into the vocabulary, right padding
        def __call__(self, texts, return_tensors="pt", max_length=512, padding=True, truncation=True):
            rows = [[101] + [1000 + (sum(map(ord, w)) * 31 + len(w)) % 1500 for w in t.split()][: max_length - 2] + [102] for t in texts]
            S = max(len(r) for r in rows)
            ids = torch.zeros((len(rows), S), dtype=torch.long)
            mask = torch.zeros((len(rows), S), dtype=torch.long)
            for i, r in enumerate(rows):
                ids[i, : len(r)] = torch.tensor(r)
                mask[i, : len(r)] = 1
            return {"input_ids": ids, "attention_mask": mask, "token_type_ids": torch.zeros_like(ids)}

    cfg = dict(hidden_size=768, num_hidden_layers=2, num_attention_heads=12, intermediate_size=3072, vocab_size=3000,
               max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12)
    sd = random_state_dict(cfg, 9)
    model = B200Contriever(cfg, "average")
    model.load_state_dict(sd)
    rng = np.random.default_rng(1)
    passages = [{"id": 1000 + i, "title": f"title {i}", "text": " ".join(f"w{rng.integers(0, 500)}" for _ in range(int(rng.integers(20, 300))))}
                for i in range(700)]
    args = C.DictConfig({"model_name_or_path": "contriever-test", "per_gpu_batch_size": 512, "passage_maxlength": 256,
                     "no_title": False, "lowercase": False, "normalize_text": False})
    ids, emb = embed_passages(args, passages, model, Tok())
    assert ids == [p["id"] for p in passages] and emb.shape == (700, 768) and emb.dtype == np.float16
    tok = Tok()
    sel = [0, 1, 511, 512, 699]
    enc = tok([passages[i]["title"] + " " + passages[i]["text"] for i in sel], max_length=256)
    with torch.no_grad():
        ref = BO.bert_forward(sd, cfg, enc["input_ids"], enc["attention_mask"], None, "average", dtype=torch.float32).numpy()
    got = emb[sel].astype(np.float32)
    cos = (got * ref).sum(1) / (np.linalg.norm(got, axis=1) * np.linalg.norm(ref, axis=1))
    assert cos.min() >= 0.9999, cos
