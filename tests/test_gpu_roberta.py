"""GPU parity of the RoBERTa retrievers (`B200Roberta`, DRAGON-RoBERTa's query and context encoders) on the fixture of
tests/golden/roberta_fixture.py: 2 layers of roberta-base geometry with seeded weights, not the released checkpoints.

  token rows     every row of the final hidden states against the fp16 / fp32 torch oracle (tests/roberta_oracle.py),
                 with the bounds of test_gpu_encoder_kernels.py, across both attention kernels, with pad ids inside
  CLS rows       against HF RobertaModel's fp32 golden (tests/golden/roberta_golden.npz), the <pad> queries included
  edges          ids 0, 1, 2 and 50264 on the full vocabulary; batch composition; refusals before any launch
  end to end     ric/main_ric.py: passage embedding with the context encoder -> Flat index -> search with the query
                 encoder, against the same pipeline on the CPU from HF RobertaModel embeddings"""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import roberta_oracle as RO
from golden import roberta_fixture as RF

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "roberta_golden.npz")
LENGTHS = [1, 2, 31, 32, 33, 255, 256, 257, 511, 512]


@pytest.fixture(scope="module")
def fx(tmp_path_factory):
    return RF.build(str(tmp_path_factory.mktemp("roberta")))


def _ulp16(x):
    e = torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -14)))
    return torch.exp2(e.clamp_min(-14) - 10)


def _model(sd, pooling="cls", config=RF.CONFIG):
    from retrieval_scaling_b200.encoder import B200Roberta
    m = B200Roberta(config, pooling)
    assert m.load_state_dict(sd) == []                      # pooler.* is not read
    m.require_all_weights()
    return m


def _batch(rng, lens, vocab, pad_share=0.03):
    """Right-padded [B, S] ids (pad positions hold id 1, as the tokenizer writes them) with a share of pad ids inside
    the sequences, and the attention mask."""
    S = int(max(lens))
    ids = rng.integers(3, vocab, (len(lens), S))
    ids[rng.random(ids.shape) < pad_share] = 1
    mask = np.arange(S)[None, :] < np.asarray(lens)[:, None]
    ids[~mask] = 1
    return torch.from_numpy(ids).cuda(), torch.from_numpy(mask.astype(np.int64)).cuda()


def _check_token_rows(got, sd, ids, mask, tag):
    """test_gpu_encoder_kernels.py's bar: cosine >= 0.9999 per token against the fp16 and fp32 oracles, and per row
    max |err| against fp32 <= 2x the fp16 oracle's own, floored at 1 fp16 ulp of the row's largest element."""
    sdc = {k: v.cuda() for k, v in sd.items()}
    with torch.no_grad():
        h16 = RO.roberta_token_rows(sdc, RF.CONFIG, ids, mask, torch.float16).double()
        h32 = RO.roberta_token_rows(sdc, RF.CONFIG, ids, mask, torch.float32).double()
    got = got.double()
    cos16, cos32 = F.cosine_similarity(got, h16, dim=1), F.cosine_similarity(got, h32, dim=1)
    assert cos16.min().item() >= 0.9999 and cos32.min().item() >= 0.9999, (tag, cos16.min().item(), cos32.min().item())
    err = (got - h32).abs().max(1).values
    lim = torch.maximum(2 * (h16 - h32).abs().max(1).values, _ulp16(h32.abs().max(1).values))
    assert (err <= lim).all(), (tag, (err / lim).max().item(), int(torch.argmax(err / lim)))
    print(f"[roberta {tag}] min cos fp16 {cos16.min().item():.6f} fp32 {cos32.min().item():.6f}, "
          f"max err/(2x fp16 cost) {(err / lim).max().item():.3f}")
    return h32


def test_token_rows_against_the_oracle_at_every_length(fx):
    """Lengths 1 ... 512 (both attention kernels and the <= 32 / longer split), 3% pad ids inside the sequences.  The
    comparison rejects the oracle with BERT's positions (every token counted)."""
    sd = fx["query"]["state_dict"]
    m = _model(sd)
    rng = np.random.default_rng(7)
    ids, mask = _batch(rng, LENGTHS, RF.CONFIG["vocab_size"])
    assert int((ids[mask.bool()] == 1).sum()) > 20
    tok, cu = m.hidden_states(input_ids=ids, attention_mask=mask)
    assert tok.shape == (int(mask.sum()), 768) and torch.isfinite(tok).all()
    _check_token_rows(tok, sd, ids, mask, "lengths")
    naive = dict(sd)
    naive["embeddings.position_embeddings.weight"] = sd["embeddings.position_embeddings.weight"][2:]
    from oracle import bert_oracle as BO
    with torch.no_grad():
        wrong = torch.cat([BO.bert_hidden({k: v.cuda() for k, v in naive.items()}, RF.CONFIG, ids[b:b + 1, :L],
                                          mask[b:b + 1, :L])[0] for b, L in enumerate(LENGTHS)]).double()
    assert (F.cosine_similarity(tok.double(), wrong, dim=1) < 0.9999).any(), "BERT positions were accepted"


def test_special_and_last_ids_on_the_full_vocabulary(fx):
    """Ids 0 (<s>), 1 (<pad>: position padding_idx, not counted), 2 (</s>) and 50264 (the last row)."""
    sd = fx["context"]["state_dict"]
    m = _model(sd)
    seqs = [[0, 50264, 1, 5, 2], [1], [50264], [0, 2], [0, 1, 1, 1, 50264, 2], [1, 0, 2, 50264] * 10]
    S = max(len(s) for s in seqs)
    ids = torch.ones((len(seqs), S), dtype=torch.long)
    mask = torch.zeros((len(seqs), S), dtype=torch.long)
    for i, s in enumerate(seqs):
        ids[i, :len(s)] = torch.tensor(s)
        mask[i, :len(s)] = 1
    ids, mask = ids.cuda(), mask.cuda()
    tok, _ = m.hidden_states(input_ids=ids, attention_mask=mask)
    _check_token_rows(tok, sd, ids, mask, "special ids")


def test_cls_rows_against_the_transformers_golden(fx):
    """Through `load_retriever` on the fixture directories (the loader `search.load_query_encoder` and
    `embed.load_passage_encoder` call for dragon* names): the fixture tokenizer's ids equal the golden's, and every
    CLS row has cosine >= 0.9999 with HF RobertaModel's fp32 row -- the empty, 512-token and <pad> queries included."""
    from retrieval_scaling_b200.encoder import B200Roberta, load_retriever
    z = np.load(GOLD)
    texts = [str(t) for t in z["texts"]]
    for which in ("query", "context"):
        model, tok, _ = load_retriever(fx[which]["dir"], pooling="cls")
        assert isinstance(model, B200Roberta)
        enc = tok(texts, return_tensors="pt", padding=True, truncation=True, max_length=512)
        assert np.array_equal(enc["input_ids"].numpy(), z["input_ids"])
        out = model(**{k: v.cuda() for k, v in enc.items()})
        assert out.dtype == torch.float16 and tuple(out.shape) == (len(texts), 768)
        cos = F.cosine_similarity(out.double().cpu(), torch.from_numpy(z[f"cls_{which}"]).double(), dim=1)
        print(f"[roberta golden {which}] min cos {cos.min().item():.6f}")
        assert (cos >= 0.9999).all(), [(texts[i][:30], cos[i].item()) for i in range(len(texts)) if cos[i] < 0.9999]


def test_batch_composition_is_bit_identical(fx):
    """A query alone and at several places inside a group of 2048 NQ-length sequences (with and without pad ids): the
    same bits, for CLS and mean pooling."""
    sd = fx["query"]["state_dict"]
    rng = np.random.default_rng(11)
    nq = np.load(os.path.join(ROOT, "tests", "golden", "nq_open_token_lengths.npy")).astype(np.int64)
    lens = rng.choice(nq, 2048)
    lens[[0, 700, 2047]] = (17, 33, 9)
    ids, mask = _batch(rng, lens, RF.CONFIG["vocab_size"])
    for pooling in ("cls", "average"):
        m = _model(sd, pooling)
        full = m(input_ids=ids, attention_mask=mask)
        for b in (0, 5, 700, 2047):
            L = int(lens[b])
            alone = m(input_ids=ids[b:b + 1, :L], attention_mask=mask[b:b + 1, :L])
            assert torch.equal(alone[0].view(torch.int16), full[b].view(torch.int16)), (pooling, b, L)


def test_refusals_before_any_launch(fx):
    """A sequence whose positions would pass max_position_embeddings and a nonzero token type are refused with nothing
    written; a checkpoint without one of its weights is refused by require_all_weights."""
    from retrieval_scaling_b200 import _lib
    from retrieval_scaling_b200.encoder import B200Roberta
    small = dict(RF.CONFIG, num_hidden_layers=1, max_position_embeddings=40, vocab_size=1000)
    from oracle.bert_oracle import seeded_state_dict
    m = _model(seeded_state_dict(small, 3), config=small)
    L = _lib.lib()

    def call(S, types=None):
        ids = torch.full((S,), 7, dtype=torch.int32, device="cuda")
        cu = torch.tensor([0, S], dtype=torch.int32, device="cuda")
        out = torch.full((1, 768), float("nan"), dtype=torch.float16, device="cuda")
        ws = torch.empty(L.rsb_bert_workspace_bytes(m._h, S), dtype=torch.uint8, device="cuda")
        tt = ctypes.c_void_p(types.data_ptr()) if types is not None else ctypes.c_void_p(0)
        rc = L.rsb_bert_forward(m._h, ctypes.c_void_p(ids.data_ptr()), tt, ctypes.c_void_p(cu.data_ptr()), 1, S, S,
                                _lib.POOL_CLS, ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(ws.data_ptr()), ws.numel(),
                                ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        return rc, out

    rc, out = call(38)                                     # last position 1 + 38 = 39: the table's last row
    assert rc == _lib.RSB_OK and torch.isfinite(out).all()
    rc, out = call(39)                                     # position 40 would pass the 40-row table
    assert rc == _lib.RSB_ERR_UNSUPPORTED and torch.isnan(out).all()
    assert b"max_position_embeddings" in L.rsb_bert_last_error()
    zeros = torch.zeros(10, dtype=torch.int32, device="cuda")
    assert call(10, zeros)[0] == _lib.RSB_OK
    ones = zeros.clone()
    ones[4] = 1
    rc, out = call(10, ones)
    assert rc == _lib.RSB_ERR_INVALID and torch.isnan(out).all()
    with pytest.raises(ValueError, match="token type"):
        m(input_ids=torch.full((1, 10), 7, device="cuda"), token_type_ids=ones[None].long())
    with pytest.raises(NotImplementedError, match="max_position_embeddings"):
        m(input_ids=torch.full((1, 39), 7, device="cuda"))

    sd = dict(fx["query"]["state_dict"])
    del sd["encoder.layer.1.attention.self.value.bias"]
    mm = B200Roberta(RF.CONFIG, "cls")
    mm.load_state_dict(sd, strict=False)
    with pytest.raises(KeyError, match="attention.self.value.bias"):
        mm.require_all_weights("fixture without one weight")


# ---------------------------------------------------------------------------------------------------------------
# end to end through ric/main_ric.py
# ---------------------------------------------------------------------------------------------------------------
def _texts(rng, n, lo, hi):
    out = []
    for i in range(n):
        words = list(rng.choice(RF.WORDS, int(rng.integers(lo, hi))))
        if i % 9 == 4:
            words.insert(len(words) // 2, "<pad>")
        out.append(" ".join(words))
    return out


def test_main_ric_embedding_flat_search_matches_a_cpu_pipeline(fx, tmp_path):
    """`tasks.datastore.embedding` with the context encoder -> Flat index -> `tasks.eval.search` with the query encoder
    (the asymmetric pair: model.query_encoder vs datastore.embedding.model_name_or_path), against the same pipeline on
    the CPU: HF RobertaModel CLS embeddings in fp32 and the oracle's exact Flat search.  Ids must agree rank by rank
    except inside groups of scores closer than the bound the embeddings' fp16 differences put on a score."""
    import transformers

    from oracle import ann_oracle as O
    rng = np.random.default_rng(3)
    passages = _texts(rng, 600, 3, 60)
    passages[7] = " ".join(RF.WORDS * 20)                   # past passage_maxlength: truncated at 512 tokens
    queries = _texts(rng, 24, 2, 12)
    psg_dir = tmp_path / "passages" / "dom" / "1-shards"
    psg_dir.mkdir(parents=True)
    with open(psg_dir / "raw_passages-0-of-1.jsonl", "w") as f:
        for i, t in enumerate(passages):
            f.write(json.dumps({"id": i, "title": f"t{i % 5}", "text": t}) + "\n")
    eval_path = tmp_path / "nq.jsonl"
    qcache = tmp_path / "query_embeddings.pkl"              # written by the run: the GPU query embeddings
    with open(eval_path, "w") as f:
        for q in queries:
            f.write(json.dumps({"query": q}) + "\n")
    cmd = [sys.executable, os.path.join(ROOT, "ric", "main_ric.py"), "--config-name", "default",
           f"datastore.datastore_root_dir={tmp_path}", "datastore.domain=dom", "evaluation.domain=dom",
           "model.datastore_encoder=dragon-roberta", f"model.query_encoder={fx['query']['dir']}",
           f"datastore.embedding.model_name_or_path={fx['context']['dir']}", "datastore.embedding.per_gpu_batch_size=128",
           "datastore.index.index_type=Flat", "evaluation.search.n_docs=10", f"evaluation.data.eval_data={eval_path}",
           "tasks.datastore.embedding=true", "tasks.eval.search=true", "tasks.eval.task_name=lm-eval",
           "+evaluation.search.cache_query_embedding=true", f"+evaluation.search.query_embedding_save_path={qcache}"]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    out = os.path.join(str(tmp_path), "retrieved_results", "dragon-roberta", "dom", "top_10", "0", "nq_retrieved_results.jsonl")
    res = [json.loads(line) for line in open(out)]
    assert len(res) == len(queries)
    pid = lambda c: int(c["id"][-1] if isinstance(c["id"], list) else c["id"])   # noqa: E731
    I = np.array([[pid(c) for c in ex["ctxs"]] for ex in res])
    D = np.array([[float(c["retrieval score"]) for c in ex["ctxs"]] for ex in res], np.float32)

    def hf_cls(which, texts, max_len):
        tok = transformers.AutoTokenizer.from_pretrained(fx[which]["dir"], local_files_only=True)
        model = transformers.AutoModel.from_pretrained(fx[which]["dir"], local_files_only=True).eval().float()
        rows = []
        with torch.no_grad():
            for i in range(0, len(texts), 64):
                enc = tok(texts[i:i + 64], return_tensors="pt", padding=True, truncation=True, max_length=max_len)
                rows.append(model(**enc).last_hidden_state[:, 0, :])
        return torch.cat(rows).numpy().astype(np.float32)

    xb = hf_cls("context", [f"t{i % 5} {t}" for i, t in enumerate(passages)], 512).astype(np.float64)
    xq = hf_cls("query", queries, 512).astype(np.float64)
    import pickle
    emb = os.path.join(str(tmp_path), "embeddings", "dragon-roberta", "dom", "1-shards", "passages_00.pkl")
    ids, gb = pickle.load(open(emb, "rb"))
    assert list(ids) == list(range(len(passages)))
    gq = pickle.load(open(qcache, "rb"))
    gb, gq = gb.astype(np.float64), gq.astype(np.float64)
    # each side ran its own encoder: the context encoder for passages, the query encoder for queries
    for name, got, ref in (("passages", gb, xb), ("queries", gq, xq)):
        cos = F.cosine_similarity(torch.from_numpy(got), torch.from_numpy(ref), dim=1)
        assert cos.min().item() >= 0.9999, (name, cos.min().item())
    # the index: exact search over the pipeline's own fp16 embeddings (fp32 accumulation over d = 768 terms)
    Dg, Ig = O.flat_search(gq.astype(np.float32), gb.astype(np.float32), 10)
    fp32 = 768 * 2.0 ** -24 * float(np.max(np.abs(gq) @ np.abs(gb).T))
    O.assert_topk_equivalent(D, I, Dg, Ig, score_of=lambda q, j: float(gq[q] @ gb[j]), rtol=1e-5, atol=fp32)
    # end to end against HF RobertaModel's fp32 embeddings: a score moves by at most
    # |dq| |p| + |q| |dp| + |dq| |dp| (Cauchy-Schwarz) when the embeddings move by dq, dp
    dq, dp = np.linalg.norm(gq - xq, axis=1), np.linalg.norm(gb - xb, axis=1)
    nq_, np_ = np.linalg.norm(xq, axis=1), np.linalg.norm(xb, axis=1)
    moved = float(np.max(dq[:, None] * np_[None] + nq_[:, None] * dp[None] + dq[:, None] * dp[None]))
    Dr, Ir = O.flat_search(xq.astype(np.float32), xb.astype(np.float32), 10)
    same = float(np.mean(I == Ir))
    print(f"[roberta main_ric] score bound from the embeddings {moved:.3g} (scores up to {np.abs(Dr).max():.3g}), "
          f"ids equal rank by rank: {same:.3f}")
    O.assert_topk_equivalent(D, I, Dr, Ir, score_of=lambda q, j: float(xq[q] @ xb[j]), rtol=1e-5, atol=moved + fp32)
