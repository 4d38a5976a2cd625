"""CPU-side checks of the Llama reader: the fp64 oracle against transformers, the committed golden, the geometry and
config refusals (all before any weight is read or device memory allocated) and the C-ABI refusals of rsb_llm_create /
rsb_llm_nll, which need no device."""
import ctypes
import json
import os
import re
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import llama_fixture as F  # noqa: E402
import llama_oracle as O  # noqa: E402

from retrieval_scaling_b200 import reader  # noqa: E402


@pytest.mark.parametrize("kv_heads", [4, 1])
@pytest.mark.parametrize("theta", [10000.0, 500000.0])
def test_oracle_matches_transformers_fp32(kv_heads, theta):
    cfg = dict(F.CONFIG, num_key_value_heads=kv_heads, rope_theta=theta, max_position_embeddings=256)
    model = F.hf_model(cfg, dtype=torch.float32, seed=7)
    sd = F.seeded_state_dict(cfg, seed=7)
    ids = np.random.default_rng(1).integers(0, cfg["vocab_size"], 150)
    ours = O.token_nll(sd, cfg, ids)
    hf = F.hf_token_nll(model, ids)
    np.testing.assert_allclose(ours, hf, atol=1e-4, rtol=0)


def test_oracle_tied_embeddings():
    cfg = dict(F.CONFIG, tie_word_embeddings=True, num_hidden_layers=1, max_position_embeddings=128)
    model = F.hf_model(cfg, dtype=torch.float32, seed=3)
    sd = F.seeded_state_dict(cfg, seed=3)
    assert "lm_head.weight" not in sd
    ids = np.random.default_rng(2).integers(0, cfg["vocab_size"], 40)
    np.testing.assert_allclose(O.token_nll(sd, cfg, ids), F.hf_token_nll(model, ids), atol=1e-4, rtol=0)


def test_golden_matches_the_oracle():
    g = np.load(F.GOLDEN)
    assert json.loads(str(g["config"])) == F.CONFIG
    cu, ids, nll = g["cu_seqlens"], g["ids"], g["nll"]
    windows = F.window_ids()
    assert [len(w) for w in windows] == list(np.diff(cu)) == list(F.LENGTHS)
    assert F.CONFIG["vocab_size"] % 128 and max(F.LENGTHS) == F.CONFIG["max_position_embeddings"]
    assert np.array_equal(ids, np.concatenate(windows))
    sd = F.seeded_state_dict()
    for b in range(len(windows)):
        if len(windows[b]) > 200:
            continue
        # HF's LlamaRMSNorm takes its statistics in fp32 even in a float64 model: agreement to ~1e-7, not 1e-15
        np.testing.assert_allclose(O.token_nll(sd, F.CONFIG, windows[b]), nll[cu[b]:cu[b + 1]], atol=1e-5, rtol=0)
    assert np.all(nll[cu[:-1]] == 0)


def test_mean_loss_is_hf_loss_with_masks():
    nll = np.array([0.0, 1.0, 2.0, 4.0])
    assert O.mean_loss(nll, [5, 6, 7, 8]) == pytest.approx(7 / 3)
    assert O.mean_loss(nll, [-100, -100, 7, -100]) == pytest.approx(2.0)
    assert np.isnan(O.mean_loss(nll, [5, -100, -100, -100]))          # only the first position: nothing is scored
    assert reader.scored_positions([5, -100, 7, 8]) == [2, 3]
    assert reader.scored_positions([3]) == []


LLAMA2 = dict(model_type="llama", hidden_size=4096, num_attention_heads=32, num_key_value_heads=32,
              intermediate_size=11008, num_hidden_layers=32, vocab_size=32000, max_position_embeddings=4096,
              rms_norm_eps=1e-5, rope_theta=10000.0, hidden_act="silu", rope_scaling=None, tie_word_embeddings=False)


def test_geometry_of_released_readers():
    g = reader.llama_geometry(LLAMA2)
    assert (g["num_key_value_heads"], g["rope_theta"], g["tie_word_embeddings"]) == (32, 10000.0, False)
    g3 = reader.llama_geometry(dict(LLAMA2, num_key_value_heads=8, intermediate_size=14336, vocab_size=128256,
                                    rope_theta=500000.0, max_position_embeddings=8192))
    assert g3["num_key_value_heads"] == 8 and g3["rope_theta"] == 500000.0
    # transformers >= 5 writes rope_theta inside rope_parameters
    g5 = reader.llama_geometry(dict(LLAMA2, rope_scaling=None, rope_parameters={"rope_type": "default", "rope_theta": 5e5}))
    assert g5["rope_theta"] == 5e5


@pytest.mark.parametrize("change, field", [
    (dict(model_type="gpt_neox"), "model_type"),
    (dict(model_type="mistral"), "model_type"),
    (dict(hidden_size=2048, num_attention_heads=32), "head_dim"),
    (dict(head_dim=64), "head_dim"),
    (dict(num_key_value_heads=5), "num_key_value_heads"),
    (dict(hidden_act="gelu"), "hidden_act"),
    (dict(intermediate_size=11000), "intermediate_size"),
    (dict(attention_bias=True), "attention_bias"),
    (dict(mlp_bias=True), "mlp_bias"),
    (dict(rope_scaling={"rope_type": "llama3", "factor": 8.0}), "rope_scaling"),
    (dict(rope_parameters={"rope_type": "linear", "rope_theta": 1e4, "factor": 2.0}), "rope_parameters"),
    (dict(vocab_size=0), "vocab_size"),
])
def test_geometry_refusals_name_the_field(change, field):
    with pytest.raises(AttributeError, match=field):
        reader.llama_geometry(dict(LLAMA2, **change))


def test_gpt_neox_refusal_says_why():
    with pytest.raises(AttributeError, match="head_dim-256 attention, partial rotary and a parallel residual"):
        reader.llama_geometry(dict(model_type="gpt_neox", hidden_size=2048, num_attention_heads=8))


def test_load_reader_refuses_before_reading_weights(tmp_path, monkeypatch):
    (tmp_path / "config.json").write_text(json.dumps(dict(LLAMA2, model_type="gpt_neox")))
    (tmp_path / "model.safetensors").write_bytes(b"not a safetensors file")
    import safetensors

    def no_read(*a, **k):
        raise AssertionError("a weight file was opened")
    monkeypatch.setattr(safetensors, "safe_open", no_read)
    monkeypatch.setattr(reader.B200Llama, "__init__", lambda *a, **k: (_ for _ in ()).throw(AssertionError("allocated")))
    with pytest.raises(AttributeError, match="model_type"):
        reader.load_reader(str(tmp_path))


def test_sharded_and_single_file_listing(tmp_path):
    with pytest.raises(FileNotFoundError):
        reader._shard_files(str(tmp_path))
    (tmp_path / "model.safetensors").write_bytes(b"")
    assert reader._shard_files(str(tmp_path)) == [str(tmp_path / "model.safetensors")]
    index = {"weight_map": {"a": "model-00002-of-00002.safetensors", "b": "model-00001-of-00002.safetensors",
                            "c": "model-00001-of-00002.safetensors"}}
    (tmp_path / "model.safetensors.index.json").write_text(json.dumps(index))
    assert reader._shard_files(str(tmp_path)) == [str(tmp_path / f"model-0000{i}-of-00002.safetensors") for i in (1, 2)]


def test_expected_keys():
    keys = reader.expected_keys(reader.llama_geometry(dict(LLAMA2, num_hidden_layers=2)))
    assert len(keys) == 3 + 2 * 9 and "lm_head.weight" in keys
    tied = reader.expected_keys(reader.llama_geometry(dict(LLAMA2, num_hidden_layers=2, tie_word_embeddings=True)))
    assert "lm_head.weight" not in tied and len(tied) == 2 + 2 * 9
    assert set(keys) == set(F.seeded_state_dict(dict(F.CONFIG, num_hidden_layers=2)))


def test_llm_abi_refusals_need_no_device():
    from retrieval_scaling_b200 import _lib
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "rsb.h")).read(), flags=re.S)
    decl = re.search(r"int\s+rsb_llm_create\s*\(([^)]*)\)", header).group(1)
    assert [p.split()[-1] for p in decl.split(",")][:-1] == [
        "family", "dtype", "layers", "hidden", "heads", "kv_heads", "intermediate", "vocab", "max_pos", "rotary_dims",
        "rope_theta", "eps", "clip_qkv", "tied"]
    L = _lib.lib()
    h = ctypes.c_void_p(0)
    f = ctypes.c_float
    LL, z = (_lib.RSB_LLM_LLAMA, _lib.RSB_DTYPE_F16), f(0.0)
    ok = (*LL, 2, 512, 4, 1, 1024, 1000, 4096, 128, f(1e4), f(1e-5), z, 0)
    assert L.rsb_llm_create(*ok, None) == _lib.RSB_ERR_INVALID
    bad = [
        ((*LL, 2, 512, 8, 1, 1024, 1000, 4096, 128, f(1e4), f(1e-5), z, 0), _lib.RSB_ERR_UNSUPPORTED, b"head_dim"),   # 64
        ((*LL, 2, 512, 4, 3, 1024, 1000, 4096, 128, f(1e4), f(1e-5), z, 0), _lib.RSB_ERR_UNSUPPORTED, b"num_key_value_heads"),
        ((*LL, 2, 512, 4, 1, 1000, 1000, 4096, 128, f(1e4), f(1e-5), z, 0), _lib.RSB_ERR_UNSUPPORTED, b"intermediate_size"),
        ((*LL, 0, 512, 4, 1, 1024, 1000, 4096, 128, f(1e4), f(1e-5), z, 0), _lib.RSB_ERR_INVALID, b"positive"),
        ((*LL, 2, 512, 4, 1, 1024, 0, 4096, 128, f(1e4), f(1e-5), z, 0), _lib.RSB_ERR_INVALID, b"positive"),
        ((*LL, 2, 512, 4, 1, 1024, 1000, 4096, 128, f(0.0), f(1e-5), z, 0), _lib.RSB_ERR_INVALID, b"rope_theta"),
        ((*LL, 2, 512, 4, 1, 1024, 1000, 4096, 128, f(1e4), f(1e-5), z, 2), _lib.RSB_ERR_INVALID, b"tied"),
        # combinations only the one constructor can express
        ((*LL, 2, 512, 4, 1, 1024, 1000, 4096, 64, f(1e4), f(1e-5), z, 0), _lib.RSB_ERR_INVALID, b"rotary_dims"),
        ((*LL, 2, 512, 4, 1, 1024, 1000, 4096, 128, f(1e4), f(1e-5), f(8.0), 0), _lib.RSB_ERR_INVALID, b"clip_qkv"),
    ]
    for args, rc, msg in bad:
        assert L.rsb_llm_create(*args, ctypes.byref(h)) == rc, args
        assert msg in L.rsb_llm_last_error()
        assert h.value is None
    p = ctypes.c_void_p(16)              # never dereferenced: the arguments are refused first
    assert L.rsb_llm_nll(None, p, p, 1, 1, 1, p, p, p, 1 << 20, None) == _lib.RSB_ERR_INVALID
    assert L.rsb_llm_load(None, b"model.norm.weight", p, 512, None) == _lib.RSB_ERR_INVALID
    assert L.rsb_llm_attention(None, p, p, 1, 1, 1, p, None) == _lib.RSB_ERR_INVALID
    assert L.rsb_llm_hidden_states(None, p, p, 1, 1, 1, p, p, 1 << 20, None) == _lib.RSB_ERR_INVALID
    assert b"null" in L.rsb_llm_last_error()
    assert L.rsb_llm_workspace_bytes(None, 10, 10) == 0
    assert L.rsb_llm_free(None) == _lib.RSB_OK
