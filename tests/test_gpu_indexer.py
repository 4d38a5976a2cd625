"""End-to-end through the drop-in boundary on the GPU: `Indexer(cfg).search(query_embs, k)` for the three index
types built from `passages_XX.pkl` embedding shards (reference artefact layout), reload from disk, passage
fetch, and the `ric/main_ric.py tasks.eval.search=true` flow with multi-index merge (query embeddings come from
the reference's `cache_query_embedding` mechanism because no tokenizer / checkpoint exists offline)."""
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

from oracle import ann_oracle as O
from retrieval_scaling_b200 import config as C

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONF = os.path.join(ROOT, "ric", "conf")
D = 64


def _make_datastore(root, nshards=2, n=3000):
    rng = np.random.default_rng(0)
    centres = rng.standard_normal((8, D)).astype(np.float32)
    emb_dir = os.path.join(root, "embeddings", "enc", "dom", f"{nshards}-shards")
    psg_dir = os.path.join(root, "passages", "dom", f"{nshards}-shards")
    os.makedirs(emb_dir); os.makedirs(psg_dir)
    embs = []
    for s in range(nshards):
        e = ((centres[rng.integers(0, 8, n)] + 0.3 * rng.standard_normal((n, D))) / 8.0).astype(np.float16)  # fp16 like the reference; unit-scale norms
        embs.append(e)
        with open(os.path.join(emb_dir, f"passages_{s:02d}.pkl"), "wb") as f:
            pickle.dump((list(range(n)), e), f)
        with open(os.path.join(psg_dir, f"raw_passages-{s}-of-{nshards}.jsonl"), "w") as f:
            for c in range(n):
                f.write(json.dumps({"text": f"passage s{s} c{c}", "id": c, "shard_id": s}) + "\n")
    q = ((centres[rng.integers(0, 8, 12)] + 0.3 * rng.standard_normal((12, D))) / 8.0).astype(np.float16)
    return embs, q


def _cfg(root, index_type, shard_ids, extra=()):
    ov = [f"datastore.datastore_root_dir={root}", "datastore.domain=dom", "model.datastore_encoder=enc",
          "datastore.embedding.num_shards=2", f"datastore.index.index_type={index_type}",
          f"datastore.index.index_shard_ids={shard_ids}", f"datastore.index.projection_size={D}",
          "datastore.index.ncentroids=16", "datastore.index.probe=16", "datastore.index.n_subquantizers=16",
          "datastore.index.sample_train_size=4000", "evaluation.search.n_docs=5"] + list(extra)
    return C.load_config("default", CONF, ov)


@pytest.mark.parametrize("index_type", ["Flat", "IVFFlat", "IVFPQ"])
def test_indexer_build_search_reload(tmp_path, index_type):
    from retrieval_scaling_b200.indicies.base import Indexer
    embs, q = _make_datastore(str(tmp_path))
    cfg = _cfg(str(tmp_path), index_type, "[0,1]")
    index = Indexer(cfg)
    scores, passages, db_ids = index.search(q, 5)
    assert len(scores) == len(passages) == len(db_ids) == 12 and all(len(s) == 5 for s in scores)
    allx = np.concatenate(embs).astype(np.float32)
    Df, If = O.flat_search(q.astype(np.float32), allx, 5)
    if index_type == "IVFPQ":   # lossy by design: the bar is equality with the oracle on the very same trained index
        from oracle import c_oracle as CO
        ix = index.datastore.index
        off, codes, ids = (t.cpu().numpy() for t in ix.export_lists())
        Dr, Ir = CO.ivfpq_search(q.astype(np.float32), ix.get_centroids().cpu().numpy(), ix.get_codebook().cpu().numpy(),
                                 off, codes, ids, 16, 5)
        O.assert_topk_equivalent(np.asarray(scores, np.float32), np.asarray([[s * 3000 + c for s, c in row] for row in db_ids]),
                                 Dr, Ir, rtol=1e-5, atol=1e-5)
    for i in range(12):
        assert scores[i] == sorted(scores[i], reverse=True)
        for (s, c), txt in zip(db_ids[i], passages[i]):
            assert txt == f"passage s{s} c{c}"                        # id map + byte-offset passage fetch agree
        got = [s * 3000 + c for s, c in db_ids[i]]
        if index_type != "IVFPQ":                                      # probe = ncentroids -> exact
            assert got == If[i].tolist()
            assert np.allclose(scores[i], Df[i], rtol=1e-5, atol=1e-5)
    idx_dir = os.path.join(cfg.datastore.embedding.embedding_dir, f"index_{index_type}", "0_1")
    names = os.listdir(idx_dir)
    assert any(n.endswith(".faiss") for n in names) and any(n.endswith(".faiss.meta") for n in names)
    if index_type != "Flat":
        assert any(n.endswith(f".4000.{D}.16.faiss") for n in names)   # reference naming scheme (base.py:24)
    index2 = Indexer(cfg)                                              # second construction loads from disk
    scores2, passages2, db_ids2 = index2.search(q, 5)
    assert db_ids2 == db_ids and passages2 == passages
    ids, sc = index2.search_ids(q.astype(np.float32), 5)               # tensor fast path
    assert tuple(ids.shape) == (12, 5) and ids.is_cuda and sc.is_cuda
    with pytest.raises(NotImplementedError):
        Indexer(_cfg(str(tmp_path), "PQ", "[0,1]"))                    # stale configs say "PQ": rejected like base.py:71-72


def test_main_ric_search_and_multi_index_merge(tmp_path):
    embs, q = _make_datastore(str(tmp_path))
    eval_path = tmp_path / "nq.jsonl"
    with open(eval_path, "w") as f:
        for i in range(12):
            f.write(json.dumps({"query": f"question {i}"}) + "\n")
    qcache = tmp_path / "q.pkl"
    with open(qcache, "wb") as f:
        pickle.dump(q, f)
    cmd = [sys.executable, os.path.join(ROOT, "ric", "main_ric.py"), "--config-name", "default",
           f"datastore.datastore_root_dir={tmp_path}", "datastore.domain=dom", "model.datastore_encoder=enc",
           "datastore.embedding.num_shards=2", "datastore.index.index_type=Flat", "datastore.index.index_shard_ids=[[0],[1]]",
           f"datastore.index.projection_size={D}", "evaluation.search.n_docs=5", "evaluation.domain=dom",
           f"evaluation.data.eval_data={eval_path}", "tasks.eval.search=true", "tasks.eval.task_name=lm-eval",
           "+evaluation.search.cache_query_embedding=true", f"+evaluation.search.query_embedding_save_path={qcache}"]
    r = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    out_root = os.path.join(str(tmp_path), "retrieved_results", "enc", "dom", "top_5")
    merged = [json.loads(l) for l in open(os.path.join(out_root, "0-1", "nq_retrieved_results.jsonl"))]
    allx = np.concatenate(embs).astype(np.float32)
    Df, If = O.flat_search(q.astype(np.float32), allx, 5)
    for i, ex in enumerate(merged):
        got = [c["id"][0] * 3000 + c["id"][1] for c in ex["ctxs"]]
        assert got == If[i].tolist()                                   # per-shard search + merge == one index
        assert [float(c["retrieval score"]) for c in ex["ctxs"]] == sorted((float(c["retrieval score"]) for c in ex["ctxs"]), reverse=True)
        assert ex["ctxs"][0]["retrieval text"].startswith("passage s")


class _HashTokenizer:
    """Stand-in for the HF tokenizer (no vocab file exists offline): whitespace split, hashed ids, right padding."""

    def __call__(self, texts, return_tensors="pt", max_length=512, padding=True, truncation=True):
        import torch
        rows = [[101] + [1000 + (hash(w) % 20000) for w in t.split()][: max_length - 2] + [102] for t in texts]
        S = max(len(r) for r in rows)
        ids = torch.zeros((len(rows), S), dtype=torch.long)
        mask = torch.zeros((len(rows), S), dtype=torch.long)
        for i, r in enumerate(rows):
            ids[i, : len(r)] = torch.tensor(r)
            mask[i, : len(r)] = 1
        return {"input_ids": ids, "attention_mask": mask, "token_type_ids": torch.zeros_like(ids)}


def test_datastore_api_encode_and_search(tmp_path):
    """text -> GPU encoder -> Indexer.search through the reference's DatastoreAPI surface (api/api_index.py:21-67)."""
    import torch
    from oracle import bert_oracle as BO
    from retrieval_scaling_b200.api_index import DatastoreAPI
    from retrieval_scaling_b200.encoder import B200Contriever, random_state_dict
    cfg_enc = dict(hidden_size=768, num_hidden_layers=2, num_attention_heads=12, intermediate_size=3072, vocab_size=30522,
                   max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12)
    sd = random_state_dict(cfg_enc, 1)
    model = B200Contriever(cfg_enc, "average"); model.load_state_dict(sd)
    tok = _HashTokenizer()
    docs = [f"document number {i} about topic {i % 7} and subject {i % 13}" for i in range(400)]
    enc = tok(docs)
    with torch.no_grad():
        emb = model(**{k: v.cuda() for k, v in enc.items()}).float().cpu().numpy()
    emb_dir = os.path.join(str(tmp_path), "embeddings", "enc", "dom", "1-shards")
    psg_dir = os.path.join(str(tmp_path), "passages", "dom", "1-shards")
    os.makedirs(emb_dir); os.makedirs(psg_dir)
    with open(os.path.join(emb_dir, "passages_00.pkl"), "wb") as f:
        pickle.dump((list(range(400)), emb.astype(np.float16)), f)
    with open(os.path.join(psg_dir, "raw_passages-0-of-1.jsonl"), "w") as f:
        for i, t in enumerate(docs):
            f.write(json.dumps({"text": t, "id": i}) + "\n")
    cfg = C.load_config("default", CONF, [f"datastore.datastore_root_dir={tmp_path}", "datastore.domain=dom",
                                          "model.datastore_encoder=enc", "model.query_encoder=contriever-test",
                                          "datastore.index.index_type=Flat", "evaluation.search.per_gpu_batch_size=3"])
    api = DatastoreAPI(cfg, shard_id=0, query_encoder=model, query_tokenizer=tok)
    res = api.search([docs[5], docs[123]], n_docs=3)
    assert res["IDs"][0][0] == [0, 5] and res["IDs"][1][0] == [0, 123]      # a document retrieves itself first
    assert res["passages"][0][0] == docs[5]
    one = api.search(docs[77], n_docs=1)
    assert one["IDs"] == [[[0, 77]]]
    # the embedding the API used matches the torch oracle of the reference encoder
    q = api.embed_query(docs[5])
    with torch.no_grad():
        ref = BO.bert_forward(sd, cfg_enc, enc["input_ids"][5:6, : int(enc["attention_mask"][5].sum())],
                              enc["attention_mask"][5:6, : int(enc["attention_mask"][5].sum())]).numpy()
    cos = float((q[0].astype(np.float32) @ ref[0]) / (np.linalg.norm(q[0].astype(np.float32)) * np.linalg.norm(ref[0])))
    assert cos > 0.9999
