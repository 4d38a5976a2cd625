"""CPU checks of the OLMo / OLMo-2 reader: the fp64 oracle against transformers, the committed golden against the
oracle, config parsing of the published OLMo geometries in both config forms, the refusals (geometry and C-ABI)
without a device, dispatch and the expected keys."""
import ctypes
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import olmo_fixture as F  # noqa: E402
import olmo_oracle as O  # noqa: E402
from retrieval_scaling_b200 import reader  # noqa: E402

# published geometries: (model_type, hidden, heads, kv heads, intermediate, layers, vocab, max_pos, rope_theta,
# clip_qkv, tie_word_embeddings, rms_norm_eps)
OLMO = {
    "OLMo-1B-hf": ("olmo", 2048, 16, 16, 8192, 16, 50304, 2048, 10000.0, None, True, None),
    "OLMo-7B-hf": ("olmo", 4096, 32, 32, 11008, 32, 50304, 2048, 10000.0, None, False, None),
    "OLMo-7B-0424-hf": ("olmo", 4096, 32, 32, 11008, 32, 50304, 4096, 10000.0, 8.0, False, None),
    "OLMo-2-0425-1B": ("olmo2", 2048, 16, 16, 8192, 16, 100352, 4096, 500000.0, None, False, 1e-6),
    "OLMo-2-1124-7B": ("olmo2", 4096, 32, 32, 11008, 32, 100352, 4096, 500000.0, None, False, 1e-6),
    "OLMo-2-1124-13B": ("olmo2", 5120, 40, 40, 13824, 40, 100352, 4096, 500000.0, None, False, 1e-6),
    "OLMo-2-0325-32B": ("olmo2", 5120, 40, 8, 27648, 64, 100352, 4096, 500000.0, None, False, 1e-6),
}


def hub_config(name):
    mt, H, nh, kv, I, L, V, P, theta, clip, tied, eps = OLMO[name]
    cfg = dict(model_type=mt, hidden_size=H, num_attention_heads=nh, num_key_value_heads=kv, intermediate_size=I,
               num_hidden_layers=L, vocab_size=V, max_position_embeddings=P, rope_theta=theta, rope_scaling=None,
               hidden_act="silu", attention_bias=False, tie_word_embeddings=tied, pad_token_id=1, eos_token_id=50279)
    if mt == "olmo":
        cfg["clip_qkv"] = clip
    else:
        cfg["rms_norm_eps"] = eps
    return cfg


@pytest.mark.parametrize("kind, change", [
    ("olmo", {}),                                                   # clip_qkv active, tied, rope_theta 1e4
    ("olmo", dict(clip_qkv=None, tie_word_embeddings=False, rope_theta=500000.0)),
    ("olmo2", {}),                                                  # GQA 4:1, untied, rope_theta 5e5
    ("olmo2", dict(num_key_value_heads=4, tie_word_embeddings=True, rope_theta=10000.0)),
])
def test_oracle_matches_transformers_fp32(kind, change):
    cfg = F.config(kind, **change)
    sd = F.seeded_state_dict(cfg, seed=11)
    model = F.hf_model(cfg, dtype=torch.float32, sd=sd)
    ids = np.random.default_rng(3).integers(0, cfg["vocab_size"], 80)
    stats = {}
    ours = O.token_nll(sd, cfg, ids, stats=stats)
    assert np.abs(ours - F.hf_token_nll(model, ids)).max() < 1e-4
    if cfg.get("clip_qkv") and kind == "olmo":
        assert stats["clipped"] >= F.MIN_CLIPPED * stats["qkv"]


@pytest.mark.parametrize("kind", ["olmo", "olmo2"])
def test_golden_matches_oracle(kind):
    g = np.load(F.GOLDEN)
    cfg = F.CONFIGS[kind]
    assert json.loads(str(g[f"{kind}_config"])) == cfg
    cu, sd, windows = g[f"{kind}_cu_seqlens"], F.seeded_state_dict(cfg), F.window_ids(kind)
    assert [int(cu[b + 1] - cu[b]) for b in range(len(cu) - 1)] == list(F.LENGTHS)
    stats = {}
    for b in (0, 1, 4, 7, 10):                   # the golden's windows up to 129 tokens
        ours = O.token_nll(sd, cfg, windows[b], stats=stats)
        assert np.abs(ours - g[f"{kind}_nll"][cu[b]:cu[b + 1]]).max() < 2e-5   # float32 storage of ~10-nat values
    assert np.all(g[f"{kind}_nll"][cu[:-1]] == 0)
    if kind == "olmo":                           # the clamp really acts in the golden's forward
        assert float(g["olmo_clipped"]) >= F.MIN_CLIPPED and stats["clipped"] >= F.MIN_CLIPPED * stats["qkv"]


@pytest.mark.parametrize("name", sorted(OLMO))
def test_published_configs_in_both_forms(name):
    import transformers
    mt, H, nh, kv, I, L, V, P, theta, clip, tied, eps = OLMO[name]
    hub = hub_config(name)
    g = reader.olmo_geometry(hub)
    assert g["version"] == (2 if mt == "olmo2" else 1)
    assert (g["hidden_size"], g["num_attention_heads"], g["num_key_value_heads"], g["intermediate_size"]) == (H, nh, kv, I)
    assert (g["num_hidden_layers"], g["vocab_size"], g["max_position_embeddings"]) == (L, V, P)
    assert g["rope_theta"] == theta and g["clip_qkv"] == (clip or 0.0) and g["tie_word_embeddings"] == tied
    assert g["eps"] == (1e-5 if mt == "olmo" else eps)
    # transformers 5 writes rope_parameters instead of rope_theta
    cls = transformers.Olmo2Config if mt == "olmo2" else transformers.OlmoConfig
    new = dict(cls(**{k: v for k, v in hub.items() if k != "model_type"}).to_dict(), model_type=mt)
    assert isinstance(new.get("rope_parameters"), dict)
    assert reader.olmo_geometry(new) == g
    assert reader.READERS[mt] == (reader.olmo_geometry, reader.B200Olmo)


@pytest.mark.parametrize("name, change, field", [
    ("OLMo-7B-hf", dict(hidden_act="gelu"), "hidden_act"),
    ("OLMo-7B-hf", dict(attention_bias=True), "attention_bias"),
    ("OLMo-2-1124-7B", dict(attention_bias=True), "attention_bias"),
    ("OLMo-7B-hf", dict(head_dim=64), "head_dim"),
    ("OLMo-2-1124-7B", dict(hidden_size=4000), "head_dim"),
    ("OLMo-2-1124-7B", dict(num_key_value_heads=3), "num_key_value_heads"),
    ("OLMo-2-0325-32B", dict(num_key_value_heads=-8), "num_key_value_heads"),
    ("OLMo-7B-hf", dict(intermediate_size=11000), "intermediate_size"),
    ("OLMo-7B-hf", dict(hidden_size=10240, num_attention_heads=80, num_key_value_heads=80), "hidden_size"),
    ("OLMo-7B-hf", dict(rope_scaling={"rope_type": "linear", "factor": 2.0}), "rope"),
    ("OLMo-2-1124-7B", dict(rope_parameters={"rope_type": "yarn", "rope_theta": 5e5, "factor": 4.0}), "rope_parameters"),
    ("OLMo-7B-0424-hf", dict(clip_qkv=-1.0), "clip_qkv"),
    ("OLMo-7B-0424-hf", dict(clip_qkv=0.0), "clip_qkv"),
    ("OLMo-7B-hf", dict(vocab_size=0), "vocab_size"),
    ("OLMo-2-1124-7B", dict(num_hidden_layers=0), "num_hidden_layers"),
    ("OLMo-7B-hf", dict(model_type="llama"), "model_type"),
])
def test_geometry_refusals_name_the_field(name, change, field):
    cfg = dict(hub_config(name), **change)
    with pytest.raises(AttributeError, match=field) as e:
        reader.olmo_geometry(cfg)
    assert str(e.value).startswith(f"model_type {cfg['model_type']!r}: ")


def test_olmo2_ignores_clip_qkv_and_olmo_ignores_rms_norm_eps():
    """Olmo2ForCausalLM never reads clip_qkv, and OlmoLayerNorm's eps is fixed at 1e-5 whatever rms_norm_eps says."""
    g2 = reader.olmo_geometry(dict(hub_config("OLMo-2-1124-7B"), clip_qkv=8.0))
    assert g2["clip_qkv"] == 0.0
    g1 = reader.olmo_geometry(dict(hub_config("OLMo-7B-hf"), rms_norm_eps=1e-6))
    assert g1["eps"] == 1e-5


@pytest.mark.parametrize("mt", ["hf_olmo", "olmo3", "olmoe"])
def test_other_olmo_model_types_are_refused(tmp_path, mt):
    (tmp_path / "config.json").write_text(json.dumps(dict(hub_config("OLMo-7B-hf"), model_type=mt)))
    with pytest.raises(AttributeError, match=f"model_type {mt!r}"):
        reader.load_reader(str(tmp_path))


def test_load_reader_refuses_before_opening_a_weight_file(tmp_path, monkeypatch):
    (tmp_path / "config.json").write_text(json.dumps(dict(hub_config("OLMo-2-1124-7B"), hidden_act="gelu")))
    (tmp_path / "model.safetensors").write_bytes(b"not a safetensors file")
    import safetensors

    def no_read(*a, **k):
        raise AssertionError("a weight file was opened")
    monkeypatch.setattr(safetensors, "safe_open", no_read)
    monkeypatch.setattr(torch, "load", no_read)
    monkeypatch.setattr(reader.B200Olmo, "__init__", lambda *a, **k: (_ for _ in ()).throw(AssertionError("allocated")))
    with pytest.raises(AttributeError, match="hidden_act"):
        reader.load_reader(str(tmp_path))


@pytest.mark.parametrize("kind, tied", [("olmo", True), ("olmo", False), ("olmo2", True), ("olmo2", False)])
def test_expected_keys(kind, tied):
    cfg = F.config(kind, tie_word_embeddings=tied)
    keys = reader.olmo_expected_keys(reader.olmo_geometry(cfg))
    per_layer = 7 if kind == "olmo" else 11
    assert len(keys) == 1 + (kind == "olmo2") + (not tied) + 2 * per_layer and len(set(keys)) == len(keys)
    assert set(keys) == set(F.seeded_state_dict(cfg))
    if kind == "olmo":
        assert not any("norm" in k for k in keys)


def test_olmo_abi_refusals_need_no_device():
    import re
    from retrieval_scaling_b200 import _lib
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "rsb.h")).read(), flags=re.S)
    decl = re.search(r"int\s+rsb_llm_create\s*\(([^)]*)\)", header).group(1)
    assert [p.split()[-1] for p in decl.split(",")][:-1] == [
        "family", "dtype", "layers", "hidden", "heads", "kv_heads", "intermediate", "vocab", "max_pos", "rotary_dims",
        "rope_theta", "eps", "clip_qkv", "tied"]
    L = _lib.lib()
    h = ctypes.c_void_p(0)
    f = ctypes.c_float
    F16 = _lib.RSB_DTYPE_F16
    O1, O2 = (_lib.RSB_LLM_OLMO, F16), (_lib.RSB_LLM_OLMO2, F16)
    ok = (2, 4096, 32, 32, 11008, 50304, 2048, 128, f(1e4), f(1e-5))
    assert L.rsb_llm_create(*O1, *ok, f(0.0), 0, None) == _lib.RSB_ERR_INVALID
    bad = [
        ((-1, F16, *ok, f(0.0), 0), _lib.RSB_ERR_INVALID, b"family"),
        ((4, F16, *ok, f(0.0), 0), _lib.RSB_ERR_INVALID, b"family"),
        ((*O1, *ok, f(-1.0), 0), _lib.RSB_ERR_INVALID, b"clip_qkv"),
        ((*O1, *ok, f(float("nan")), 0), _lib.RSB_ERR_INVALID, b"clip_qkv"),
        ((*O1, *ok, f(float("inf")), 0), _lib.RSB_ERR_INVALID, b"clip_qkv"),
        ((*O2, *ok, f(8.0), 0), _lib.RSB_ERR_INVALID, b"clip_qkv"),
        ((*O1, 2, 10240, 80, 80, 11008, 50304, 2048, 128, f(1e4), f(1e-5), f(0.0), 0), _lib.RSB_ERR_UNSUPPORTED, b"hidden"),
        ((*O2, 2, 4000, 32, 32, 11008, 50304, 2048, 128, f(1e4), f(1e-5), f(0.0), 0), _lib.RSB_ERR_UNSUPPORTED, b"head_dim"),
        ((*O2, 2, 4096, 32, 3, 11008, 50304, 2048, 128, f(1e4), f(1e-5), f(0.0), 0), _lib.RSB_ERR_UNSUPPORTED,
         b"num_key_value_heads"),
        ((*O1, 2, 4096, 32, 32, 11000, 50304, 2048, 128, f(1e4), f(1e-5), f(0.0), 0), _lib.RSB_ERR_UNSUPPORTED,
         b"intermediate"),
        ((*O1, 0, 4096, 32, 32, 11008, 50304, 2048, 128, f(1e4), f(1e-5), f(0.0), 0), _lib.RSB_ERR_INVALID, b"positive"),
        ((*O2, 2, 4096, 32, 32, 11008, 0, 2048, 128, f(1e4), f(1e-5), f(0.0), 0), _lib.RSB_ERR_INVALID, b"positive"),
        ((*O2, *ok[:-1], f(0.0), f(0.0), 0), _lib.RSB_ERR_INVALID, b"positive"),
        ((*O1, *ok, f(0.0), 2), _lib.RSB_ERR_INVALID, b"tied"),
        # combinations only the one constructor can express
        ((*O2, 2, 4096, 32, 32, 11008, 50304, 2048, 64, f(1e4), f(1e-5), f(0.0), 0), _lib.RSB_ERR_INVALID, b"rotary_dims"),
    ]
    for args, rc, msg in bad:
        assert L.rsb_llm_create(*args, ctypes.byref(h)) == rc, args
        assert msg in L.rsb_llm_last_error(), (args, L.rsb_llm_last_error())
        assert h.value is None
    # the OLMo-2 norm diagnostic: refused before any launch (the pointers are never dereferenced)
    p = ctypes.c_void_p(16)
    norm = [
        ((0, f(1e-6), p, p, None, 4, p, None), _lib.RSB_ERR_UNSUPPORTED, b"hidden"),
        ((500, f(1e-6), p, p, None, 4, p, None), _lib.RSB_ERR_UNSUPPORTED, b"hidden"),
        ((512, f(1e-6), None, p, None, 4, p, None), _lib.RSB_ERR_INVALID, b"null"),
        ((512, f(1e-6), p, p, None, 4, None, None), _lib.RSB_ERR_INVALID, b"null"),
        ((512, f(1e-6), p, None, None, 4, p, None), _lib.RSB_ERR_INVALID, b"null"),
        ((512, f(1e-6), p, p, None, -1, p, None), _lib.RSB_ERR_INVALID, b"n_rows"),
        ((512, f(0.0), p, p, None, 4, p, None), _lib.RSB_ERR_INVALID, b"eps"),
    ]
    for args, rc, msg in norm:
        assert L.rsb_llm_olmo2_norm(*args, None) == rc, args
        assert msg in L.rsb_llm_last_error(), (args, L.rsb_llm_last_error())
    assert L.rsb_llm_olmo2_norm(512, f(1e-6), p, p, None, 0, p, None, None) == _lib.RSB_OK   # no rows
