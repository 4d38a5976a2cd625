"""CPU-side checks of the RoBERTa retrievers (DRAGON-RoBERTa's query and context encoders): the fixture, its tokenizer and
the committed HF golden, the torch oracle's position rule, the HF directory reader, and the C-ABI entry
`rsb_roberta_create` (argument refusals return before any CUDA call)."""
import ctypes
import filecmp
import os
import re

import numpy as np
import pytest
import torch

import roberta_oracle as RO
from golden import roberta_fixture as RF

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "roberta_golden.npz")


@pytest.fixture(scope="module")
def fx(tmp_path_factory):
    return RF.build(str(tmp_path_factory.mktemp("roberta")))


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def test_fixture_rebuilds_byte_identically(fx, tmp_path):
    again = RF.build(str(tmp_path))
    for which in ("query", "context"):
        a, b = fx[which]["dir"], again[which]["dir"]
        names = sorted(os.listdir(a))
        assert names == sorted(os.listdir(b))
        assert {"config.json", "model.safetensors", "tokenizer.json", "tokenizer_config.json"} <= set(names)
        _, mismatch, errors = filecmp.cmpfiles(a, b, names, shallow=False)
        assert not mismatch and not errors, (which, mismatch, errors)
    qa = open(os.path.join(fx["query"]["dir"], "model.safetensors"), "rb").read()
    ca = open(os.path.join(fx["context"]["dir"], "model.safetensors"), "rb").read()
    assert qa != ca                                         # two encoders, two seeds


def test_fixture_tokenizer_reproduces_the_committed_ids(fx, gold):
    import transformers
    tok = transformers.AutoTokenizer.from_pretrained(fx["query"]["dir"], local_files_only=True)
    assert type(tok).__name__ == "RobertaTokenizer"
    texts = [str(t) for t in gold["texts"]]
    enc = tok(texts, return_tensors="np", padding=True, truncation=True, max_length=512)
    assert "token_type_ids" not in enc
    assert np.array_equal(enc["input_ids"], gold["input_ids"])
    assert np.array_equal(enc["attention_mask"], gold["attention_mask"])
    lens = gold["attention_mask"].sum(1)
    # the query set's edges: empty (<s></s>), one word, 31 / 32 / 33 tokens, truncation at 512, the literal <pad>
    assert {2, 31, 32, 33, 512} <= set(lens.tolist()) and texts[0] == "" and len(texts[1].split()) == 1
    pad_rows = [i for i, t in enumerate(texts) if "<pad>" in t]
    assert pad_rows
    for i in pad_rows:                                      # id 1 inside the sequence, kept by the attention mask
        inside = gold["input_ids"][i, 1:lens[i] - 1]
        assert (inside == 1).any() and gold["attention_mask"][i, :lens[i]].all()
    assert any(any(ord(c) > 127 for c in t) for t in texts)


@pytest.mark.parametrize("which", ["query", "context"])
def test_oracle_matches_the_transformers_golden(fx, gold, which):
    """The oracle's CLS rows within 1e-5 of HF RobertaModel's (max |err| over the row's max |x|), every query -- the
    <pad> ones included; positions taken as BERT's (t + padding_idx + 1, no pad rule) must miss the <pad> queries."""
    ids = torch.from_numpy(gold["input_ids"]).long()
    mask = torch.from_numpy(gold["attention_mask"]).long()
    ref = torch.from_numpy(gold[f"cls_{which}"]).double()
    sd = fx[which]["state_dict"]
    with torch.no_grad():
        got = RO.roberta_cls(sd, RF.CONFIG, ids, mask).double()
    rel = (got - ref).abs().max(1).values / ref.abs().max(1).values
    assert rel.max().item() <= 1e-5, rel.tolist()
    # the rule matters: the same oracle with every token counted misses exactly the rows that hold a pad id
    naive = dict(sd)
    naive["embeddings.position_embeddings.weight"] = sd["embeddings.position_embeddings.weight"][2:]
    from oracle import bert_oracle as BO
    texts = [str(t) for t in gold["texts"]]
    for i, t in enumerate(texts):
        L = int(mask[i].sum())
        with torch.no_grad():
            row = BO.bert_hidden(naive, RF.CONFIG, ids[i:i + 1, :L], mask[i:i + 1, :L])[0, 0].double()
        off = ((row - ref[i]).abs().max() / ref[i].abs().max()).item()
        if "<pad>" in t:
            assert off > 1e-3, (t, off)
        else:
            assert off <= 1e-5, (t, off)


def test_positions_follow_create_position_ids_from_input_ids():
    from transformers.models.roberta.modeling_roberta import RobertaEmbeddings
    ids = torch.tensor([[0, 5, 1, 7, 1, 1, 9, 2, 1, 1], [1, 4, 4, 2, 1, 1, 1, 1, 1, 1]])
    want = RobertaEmbeddings.create_position_ids_from_input_ids(ids, padding_idx=1)
    assert torch.equal(RO.roberta_positions(ids, 1), want)
    assert RO.roberta_positions(ids, 1)[0].tolist() == [2, 3, 1, 4, 1, 1, 5, 6, 1, 1]


def test_read_retriever_files_accepts_the_fixture(fx):
    from retrieval_scaling_b200 import encoder as E
    for which in ("query", "context"):
        sd, cfg, tok, model_id = E.read_retriever_files(fx[which]["dir"])
        assert cfg.model_type == "roberta" and model_id == fx[which]["dir"]
        assert type(tok).__name__ == "RobertaTokenizer"
        keys = {k for k in sd if not k.startswith("pooler.")}
        assert set(E.expected_keys(2)) <= keys
        assert tuple(sd["embeddings.token_type_embeddings.weight"].shape) == (1, 768)
        assert tuple(sd["embeddings.position_embeddings.weight"].shape) == (514, 768)
        assert torch.equal(sd["encoder.layer.1.output.dense.weight"],
                           fx[which]["state_dict"]["encoder.layer.1.output.dense.weight"])
        c = E._roberta_config(cfg)
        assert (c["vocab_size"], c["max_position_embeddings"], c["type_vocab_size"], c["layer_norm_eps"],
                c["pad_token_id"], c["num_hidden_layers"]) == (50265, 514, 1, 1e-5, 1, 2)


def test_roberta_prefix_is_stripped_to_robertamodel_names(fx):
    from retrieval_scaling_b200 import encoder as E
    sd = fx["query"]["state_dict"]
    wrapped = {f"roberta.{k}": v for k, v in sd.items()}
    wrapped["lm_head.dense.weight"] = torch.zeros(2, 2)      # RobertaForMaskedLM's head is dropped with the wrapper
    out = E.strip_wrapper_prefix(wrapped)
    assert set(out) == set(sd) and all(out[k] is sd[k] for k in sd)
    bert = {f"bert.{k}": v for k, v in sd.items()}
    assert set(E.strip_wrapper_prefix(bert)) == set(sd)      # BERT's prefix unchanged


def test_read_retriever_files_refuses_other_model_types_and_geometries(fx, tmp_path):
    import json
    import shutil

    from retrieval_scaling_b200 import encoder as E
    d = str(tmp_path / "xlmr")
    shutil.copytree(fx["query"]["dir"], d)
    cfg = json.load(open(os.path.join(d, "config.json")))
    cfg.update(model_type="xlm-roberta", architectures=["XLMRobertaModel"])
    json.dump(cfg, open(os.path.join(d, "config.json"), "w"))
    with pytest.raises(AttributeError, match="BERT-architecture"):
        E.read_retriever_files(d)
    for bad in (dict(hidden_size=1024, num_attention_heads=16), dict(hidden_act="gelu_new"), dict(num_attention_heads=8)):
        with pytest.raises(AttributeError, match="RoBERTa-base"):
            E._roberta_config(dict(RF.CONFIG, **bad))
    with pytest.raises(AttributeError, match="pad_token_id"):
        E._roberta_config(dict(RF.CONFIG, pad_token_id=None))


def test_c_abi_entry_matches_the_header_and_refuses_before_cuda():
    from retrieval_scaling_b200 import _lib
    header = open(os.path.join(ROOT, "include", "rsb.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    decl = re.search(r"int\s+rsb_roberta_create\s*\(([^)]*)\)", header).group(1)
    params = [p.strip() for p in decl.split(",")]
    ctype = {"int": ctypes.c_int, "float": ctypes.c_float}
    want = [ctype[p.split()[0]] for p in params[:-1]]
    sig = {n: (r, a) for n, r, a in _lib.SIGNATURES}["rsb_roberta_create"]
    assert sig[0] is ctypes.c_int and list(sig[1][:-1]) == want and params[-1].startswith("rsb_bert_t**")
    assert [p.split()[-1] for p in params[:-1]] == ["layers", "intermediate", "vocab", "max_pos", "type_vocab", "ln_eps",
                                                    "padding_idx"]
    L = _lib.lib()
    h = ctypes.c_void_p(0)
    eps = ctypes.c_float(1e-5)
    assert L.rsb_roberta_create(2, 3072, 50265, 514, 1, eps, 1, None) == _lib.RSB_ERR_INVALID
    for pad, max_pos in ((-1, 514), (513, 514), (1, 2)):                 # no position left for a token
        assert L.rsb_roberta_create(2, 3072, 50265, max_pos, 1, eps, pad, ctypes.byref(h)) == _lib.RSB_ERR_INVALID
        assert b"padding_idx" in L.rsb_bert_last_error()
    assert L.rsb_roberta_create(2, 3072, 50265, 514, 3, eps, 1, ctypes.byref(h)) == _lib.RSB_ERR_UNSUPPORTED
    assert L.rsb_roberta_create(2, 3000, 50265, 514, 1, eps, 1, ctypes.byref(h)) == _lib.RSB_ERR_UNSUPPORTED
    assert L.rsb_roberta_create(0, 3072, 50265, 514, 1, eps, 1, ctypes.byref(h)) == _lib.RSB_ERR_UNSUPPORTED
    assert h.value is None
