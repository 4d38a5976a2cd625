"""Sentence-transformers retrievers (GTR-T5, e5-base) without a GPU: the T5 oracle against the goldens of
`transformers.T5EncoderModel`, the host-side relative-position bucket table, the model-directory reader and its
refusals, the name dispatch and host logic of the query / passage paths, and the C-ABI refusals that need no device."""
import ctypes
import json
import os
import shutil

import numpy as np
import pytest
import torch

from oracle import t5_oracle as T

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def fx(tmp_path_factory):
    from golden import st_fixture
    return st_fixture.build(str(tmp_path_factory.mktemp("st")))


def _case(name):
    z = np.load(os.path.join(GOLD, name + ".npz"))
    cfg = {k[4:]: z[k].item() for k in z.files if k.startswith("cfg_")}
    return z, cfg


@pytest.mark.parametrize("name", ["encoder_t5_l2", "encoder_t5_l12"])
def test_t5_oracle_matches_transformers_golden(name):
    z, cfg = _case(name)
    sd = T.seeded_state_dict(cfg, int(z["seed"]))
    ids, mask = torch.from_numpy(z["input_ids"]), torch.from_numpy(z["attention_mask"])
    with torch.no_grad():
        tok = T.t5_hidden(sd, cfg, ids, mask)
        got = {"out_mean": T.st_head(tok, mask, "average"), "out_cls": T.st_head(tok, mask, "cls"),
               "out_head": T.t5_st_forward(sd, cfg, ids, mask)}
    for k, v in got.items():
        np.testing.assert_allclose(v.numpy(), z[k], rtol=1e-4, atol=1e-4, err_msg=k)
    assert np.allclose(np.linalg.norm(z["out_head"], axis=1), 1.0, atol=1e-5)


@pytest.mark.parametrize("num_buckets,max_distance", [(32, 128), (64, 256), (16, 64), (32, 32), (8, 16)])
def test_bucket_table_matches_hf(num_buckets, max_distance):
    from transformers.models.t5.modeling_t5 import T5Attention

    from retrieval_scaling_b200.encoder import t5_bucket_table
    r = torch.arange(-511, 512)
    ref = T5Attention._relative_position_bucket(r, bidirectional=True, num_buckets=num_buckets, max_distance=max_distance)
    table = t5_bucket_table(num_buckets, max_distance)
    assert table.dtype == torch.int32 and table.shape == (1023,)
    assert torch.equal(table.long(), ref)
    assert torch.equal(T.relative_position_bucket(r, num_buckets, max_distance), ref)
    assert int(table.min()) >= 0 and int(table.max()) < num_buckets


def test_reader_on_fixtures(fx):
    from retrieval_scaling_b200.encoder import is_sentence_transformers_name, read_sentence_transformer
    t5 = read_sentence_transformer(fx["t5"]["dir"])
    assert (t5["arch"], t5["pooling"], t5["normalize"], t5["max_seq_length"], t5["do_lower_case"]) == ("t5", "average", True, 256, False)
    assert t5["dense"]["bias"] and t5["dense"]["out_features"] == 768
    bert = read_sentence_transformer(fx["bert"]["dir"])
    assert (bert["arch"], bert["pooling"], bert["normalize"], bert["dense"]) == ("bert", "average", True, None)
    for name, want in [("sentence-transformers/gtr-t5-base", True), ("intfloat/e5-base-v2", True),
                       ("facebook/contriever-msmarco", False), ("Qwen/Qwen3-Embedding-0.6B", False),
                       ("sentence-transformers/Qwen3-x", False), ("GritLM/GRIT-7B", False), ("drama-base", False)]:
        assert is_sentence_transformers_name(name) == want, name


def _edit(src, dst, rel, **changes):
    shutil.copytree(src, dst)
    p = os.path.join(dst, rel)
    with open(p) as f:
        obj = json.load(f)
    for k, v in changes.items():
        if v is None:
            obj.pop(k, None)
        else:
            obj[k] = v
    with open(p, "w") as f:
        json.dump(obj, f)
    return dst


@pytest.mark.parametrize("rel,changes,match", [
    ("config.json", dict(d_model=384), "geometry"),                     # all-MiniLM-sized
    ("config.json", dict(d_model=1024, num_heads=16), "geometry"),      # gtr-t5-large
    ("config.json", dict(feed_forward_proj="gated-gelu"), "geometry"),  # T5 v1.1 / Flan
    ("config.json", dict(model_type="roberta"), "model_type"),
    ("sentence_bert_config.json", dict(max_seq_length=1024), "max_seq_length"),
    ("1_Pooling/config.json", dict(pooling_mode_mean_tokens=False, pooling_mode_max_tokens=True), "pooling"),
    ("1_Pooling/config.json", dict(pooling_mode_mean_tokens=False, pooling_mode_lasttoken=True), "pooling"),
    ("1_Pooling/config.json", dict(pooling_mode_mean_tokens=False, pooling_mode_weightedmean_tokens=True), "pooling"),
    ("1_Pooling/config.json", dict(pooling_mode_cls_token=True), "pooling"),
    ("2_Dense/config.json", dict(activation_function="torch.nn.modules.activation.Tanh"), "activation"),
    ("2_Dense/config.json", dict(out_features=256), "Dense"),
])
def test_reader_refusals_t5(fx, tmp_path, rel, changes, match):
    from retrieval_scaling_b200.encoder import read_sentence_transformer
    d = _edit(fx["t5"]["dir"], str(tmp_path / "sentence-transformers-x"), rel, **changes)
    with pytest.raises(AttributeError, match=match):
        read_sentence_transformer(d)


@pytest.mark.parametrize("changes", [dict(hidden_size=384, num_attention_heads=12), dict(hidden_size=1024, num_attention_heads=16),
                                     dict(hidden_act="relu")])
def test_reader_refusals_bert(fx, tmp_path, changes):
    from retrieval_scaling_b200.encoder import read_sentence_transformer
    d = _edit(fx["bert"]["dir"], str(tmp_path / "e5-x"), "config.json", **changes)
    with pytest.raises(AttributeError, match="BERT geometry"):
        read_sentence_transformer(d)


def test_reader_refuses_module_stacks(fx, tmp_path):
    from retrieval_scaling_b200.encoder import read_sentence_transformer
    d = str(tmp_path / "sentence-transformers-y")
    shutil.copytree(fx["t5"]["dir"], d)
    mods = json.load(open(os.path.join(d, "modules.json")))
    json.dump(mods[:1] + mods[2:], open(os.path.join(d, "modules.json"), "w"))          # no Pooling
    with pytest.raises(AttributeError, match="module stack"):
        read_sentence_transformer(d)
    swapped = mods[:2] + [dict(mods[3], idx=2), dict(mods[2], idx=3)]                   # Normalize before Dense
    json.dump(swapped, open(os.path.join(d, "modules.json"), "w"))
    with pytest.raises(AttributeError, match="module stack"):
        read_sentence_transformer(d)
    os.remove(os.path.join(d, "modules.json"))
    with pytest.raises(AttributeError, match="modules.json"):
        read_sentence_transformer(d)
    with pytest.raises(FileNotFoundError):
        read_sentence_transformer(str(tmp_path / "sentence-transformers-not-downloaded"))


def test_query_and_passage_host_logic_with_the_sentence_transformers_encoder(fx, monkeypatch):
    """embed_queries / embed_passages hand a SentenceTransformerEncoder the preprocessed texts in groups and keep
    their order; the encoder strips, truncates to max_seq_length and keeps the fixture's casing rule."""
    import transformers

    from retrieval_scaling_b200 import config as C
    from retrieval_scaling_b200 import embed as E
    from retrieval_scaling_b200 import search as S
    from retrieval_scaling_b200.encoder import SentenceTransformerEncoder
    monkeypatch.setattr(S, "device", "cpu")

    class Model:                                        # per-sequence function of the un-padded tokens
        encode_group = 8
        calls = []

        def __call__(self, input_ids, attention_mask, token_type_ids=None):
            Model.calls.append(tuple(input_ids.shape))
            s = (input_ids * attention_mask).sum(1, keepdim=True).float()
            return torch.cat([s, attention_mask.sum(1, keepdim=True).float()], 1).half()

    tok = transformers.AutoTokenizer.from_pretrained(fx["t5"]["dir"], local_files_only=True)
    st = SentenceTransformerEncoder(Model(), tok, max_seq_length=12, do_lower_case=True)
    args = C.DictConfig({"per_gpu_batch_size": 4, "question_maxlength": 512, "lowercase": False, "normalize_text": False})
    qs = [f"  Who wrote the Origin of species {i} " + "a " * (i % 7) for i in range(19)]
    a = S.embed_queries(args, qs, st, None, "sentence-transformers/gtr-t5-base")
    assert a.shape == (19, 2) and a.dtype == np.float16
    assert [c[0] for c in Model.calls] == [8, 8, 3] and max(c[1] for c in Model.calls) == 12   # max_seq_length
    one = S.embed_queries(args, [qs[5]], st, None, "sentence-transformers/gtr-t5-base")
    assert np.array_equal(one[0], a[5])
    ref = tok([qs[5].strip().lower()], return_tensors="pt", max_length=12, truncation=True)["input_ids"]
    assert a[5, 0] == np.float16(ref.sum().item()) and a[5, 1] == ref.shape[1]
    with pytest.raises(AttributeError):                 # a sentence-transformers name with any other model object
        S.embed_queries(args, qs, Model(), tok, "sentence-transformers/gtr-t5-base")
    with pytest.raises(AttributeError):                 # decoder-LLM embedders stay out of scope
        S.embed_queries(args, qs, st, None, "Qwen/Qwen3-Embedding-0.6B")
    pargs = C.DictConfig({"model_name_or_path": "intfloat/e5-base-v2", "per_gpu_batch_size": 3, "passage_maxlength": 512,
                          "no_title": False, "lowercase": False, "normalize_text": False})
    Model.calls.clear()
    ids, emb = E.embed_passages(pargs, [{"id": i, "title": "T", "text": f"body {i}"} for i in range(7)], st, None)
    assert ids == list(range(7)) and emb.shape == (7, 2) and [c[0] for c in Model.calls] == [3, 3, 1]


def test_loaders_dispatch_by_name(monkeypatch):
    from retrieval_scaling_b200 import config as C
    from retrieval_scaling_b200 import embed as E
    from retrieval_scaling_b200 import encoder as enc
    from retrieval_scaling_b200 import search as S
    seen = []
    monkeypatch.setattr(enc, "load_sentence_transformer", lambda name: seen.append(name) or "ST")
    for name in ("sentence-transformers/gtr-t5-base", "intfloat/e5-base-v2"):
        cfg = C.DictConfig({"model": {"query_encoder": name}, "datastore": {"index": {}}})
        assert S.load_query_encoder(cfg) == ("ST", None)
        assert E.load_passage_encoder(C.DictConfig({"model_name_or_path": name})) == ("ST", None)
    assert seen == ["sentence-transformers/gtr-t5-base"] * 2 + ["intfloat/e5-base-v2"] * 2
    for name in ("Qwen/Qwen3-Embedding-0.6B", "GritLM/GRIT-7B", "drama-1b", "ReasonIR-8B"):
        with pytest.raises(AttributeError):
            S.load_query_encoder(C.DictConfig({"model": {"query_encoder": name}, "datastore": {"index": {}}}))
        with pytest.raises(AttributeError):
            E.load_passage_encoder(C.DictConfig({"model_name_or_path": name}))


def test_t5_create_refusals_need_no_device():
    from retrieval_scaling_b200 import _lib
    L = _lib.lib()
    h = ctypes.c_void_p(0)
    for args in ((2, 3000, 2048, 32, 128), (0, 3072, 2048, 32, 128), (2, 3072, 2048, 1, 128), (2, 3072, 0, 32, 128)):
        assert L.rsb_t5_create(*args, ctypes.c_float(1e-6), ctypes.byref(h)) == _lib.RSB_ERR_UNSUPPORTED, args
        assert h.value is None
    assert L.rsb_t5_create(2, 3072, 2048, 32, 128, ctypes.c_float(1e-6), None) == _lib.RSB_ERR_INVALID
    assert L.rsb_bert_forward(None, None, None, None, 1, 1, 1, 0, None, None, 0, None) == _lib.RSB_ERR_INVALID
    assert (_lib.POOL_MEAN, _lib.POOL_CLS, _lib.POOL_DENSE, _lib.POOL_NORMALIZE) == (0, 1, 2, 4)


def test_fixture_matches_sentence_transformers(fx):
    """The restated head and the fixture directories against the real library, where it is installed."""
    st = pytest.importorskip("sentence_transformers")
    for k in ("t5", "bert"):
        model = st.SentenceTransformer(fx[k]["dir"], device="cpu")
        texts = ["who wrote the origin of species", "What is the capital of Australia?"]
        got = torch.from_numpy(model.encode(texts))
        from retrieval_scaling_b200.encoder import read_sentence_transformer
        d = read_sentence_transformer(fx[k]["dir"])
        enc = model.tokenize(texts)
        sd = fx[k]["state_dict"]
        with torch.no_grad():
            if k == "t5":
                ref = T.t5_st_forward(sd, fx[k]["config"], enc["input_ids"], enc["attention_mask"])
            else:
                from oracle import bert_oracle as BO
                pooled = BO.bert_forward(sd, fx[k]["config"], enc["input_ids"], enc["attention_mask"],
                                         enc.get("token_type_ids"), "average")
                ref = torch.nn.functional.normalize(pooled, p=2, dim=1)
        assert d["normalize"]
        torch.testing.assert_close(got, ref, rtol=1e-4, atol=1e-4)
