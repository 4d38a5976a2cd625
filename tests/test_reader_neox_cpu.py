"""CPU checks of the GPT-NeoX reader: the fp64 oracle against transformers, the committed golden against the oracle,
config parsing of the released Pythia configs in both forms, the refusals (geometry and C-ABI) without a device, the
expected keys and the query_key_value row permutation."""
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

import neox_fixture as F  # noqa: E402
import neox_oracle as O  # noqa: E402
from retrieval_scaling_b200 import reader  # noqa: E402

# the released Pythia configs (Hub form): (hidden, heads, intermediate, layers, vocab)
PYTHIA = {"70m": (512, 8, 2048, 6, 50304), "160m": (768, 12, 3072, 12, 50304), "410m": (1024, 16, 4096, 24, 50304),
          "1b": (2048, 8, 8192, 16, 50304), "1.4b": (2048, 16, 8192, 24, 50304), "2.8b": (2560, 32, 10240, 32, 50304),
          "6.9b": (4096, 32, 16384, 32, 50432), "12b": (5120, 40, 20480, 36, 50688)}


def hub_config(name):
    H, nh, I, L, V = PYTHIA[name]
    return dict(model_type="gpt_neox", architectures=["GPTNeoXForCausalLM"], hidden_size=H, num_attention_heads=nh,
                intermediate_size=I, num_hidden_layers=L, vocab_size=V, max_position_embeddings=2048, rotary_pct=0.25,
                rotary_emb_base=10000, layer_norm_eps=1e-5, hidden_act="gelu", use_parallel_residual=True,
                tie_word_embeddings=False, bos_token_id=0, eos_token_id=0, initializer_range=0.02, use_cache=True)


@pytest.mark.parametrize("head_dim", [64, 80, 128, 256])
@pytest.mark.parametrize("pct", [0.25, 1.0])
def test_oracle_matches_transformers_fp32(head_dim, pct):
    cfg = dict(F.CONFIG, hidden_size=2 * head_dim, num_attention_heads=2, intermediate_size=512, rotary_pct=pct,
               vocab_size=300)
    sd = F.seeded_state_dict(cfg, seed=head_dim)
    model = F.hf_model(cfg, dtype=torch.float32, seed=head_dim)
    ids = np.random.default_rng(head_dim).integers(0, 300, 70)
    ours = O.token_nll(sd, cfg, ids)
    hf = F.hf_token_nll(model, ids)
    assert np.abs(ours - hf).max() < 1e-4


def test_golden_matches_oracle():
    g = np.load(F.GOLDEN)
    assert json.loads(str(g["config"])) == F.CONFIG
    cu, sd = g["cu_seqlens"], F.seeded_state_dict()
    assert [int(cu[b + 1] - cu[b]) for b in range(len(cu) - 1)] == list(F.LENGTHS)
    for b in (0, 1, 4, 7, 10):                   # the golden's windows up to 129 tokens
        ids = g["ids"][cu[b]:cu[b + 1]]
        assert np.array_equal(ids, F.window_ids()[b])
        # the float64 transformers model and the oracle agree to ~6e-7 here, as for the Llama golden (1e-5 there)
        assert np.abs(O.token_nll(sd, F.CONFIG, ids) - g["nll"][cu[b]:cu[b + 1]]).max() < 1e-5
    assert np.all(g["nll"][cu[:-1]] == 0)


@pytest.mark.parametrize("name", sorted(PYTHIA))
def test_released_configs_in_both_forms(name):
    import transformers
    H, nh, I, L, V = PYTHIA[name]
    hub = hub_config(name)
    g = reader.neox_geometry(hub)
    assert (g["hidden_size"], g["num_attention_heads"], g["intermediate_size"], g["num_hidden_layers"]) == (H, nh, I, L)
    assert g["vocab_size"] == V and g["rotary_ndims"] == H // nh // 4 and g["rotary_emb_base"] == 10000.0
    assert g["head_dim"] == H // nh and g["layer_norm_eps"] == 1e-5 and g["max_position_embeddings"] == 2048
    # transformers 5 writes rope_parameters instead of rotary_pct / rotary_emb_base
    new = transformers.GPTNeoXConfig(**{k: v for k, v in hub.items() if k != "model_type"}).to_dict()
    assert "rope_parameters" in new
    assert reader.neox_geometry(new) == g


@pytest.mark.parametrize("change, field", [
    (dict(hidden_act="gelu_new"), "hidden_act"),
    (dict(hidden_size=6144, num_attention_heads=64, intermediate_size=24576), "head_dim"),   # GPT-NeoX-20B, 96
    (dict(hidden_size=512, num_attention_heads=3), "num_attention_heads"),
    (dict(intermediate_size=2000), "intermediate_size"),
    (dict(hidden_size=10240, num_attention_heads=40, intermediate_size=40960), "hidden_size"),   # > 8192, head_dim 256
    (dict(hidden_size=10240, num_attention_heads=80, intermediate_size=40960), "hidden_size"),   # > 8192, head_dim 128
    (dict(hidden_size=240, num_attention_heads=3), "hidden_size"),                          # head_dim 80, 240 % 128
    (dict(rotary_pct=0.0), "rotary_ndims"),
    (dict(rotary_pct=0.3), "rotary_ndims"),                                                   # 76.8 -> 76: even
    (dict(rotary_pct=0.1), "rotary_ndims"),                                                   # 25.6 -> 25: odd
    (dict(rope_scaling={"rope_type": "linear", "factor": 2.0}), "rope"),
    (dict(rope_parameters={"rope_type": "dynamic", "rope_theta": 1e4, "factor": 2.0}), "rope_parameters"),
    (dict(use_parallel_residual=False), "use_parallel_residual"),
    (dict(attention_bias=False), "attention_bias"),
    (dict(tie_word_embeddings=True), "tie_word_embeddings"),
    (dict(vocab_size=0), "vocab_size"),
    (dict(model_type="llama"), "model_type"),
])
def test_geometry_refusals_name_the_field(change, field):
    cfg = dict(hub_config("1b"), **change)
    if field == "rotary_ndims" and change["rotary_pct"] == 0.3:
        assert reader.neox_geometry(cfg)["rotary_ndims"] == 76
        return
    with pytest.raises(AttributeError, match=field) as e:
        reader.neox_geometry(cfg)
    assert str(e.value).startswith(f"model_type {cfg['model_type']!r}: ")


def test_load_reader_refuses_before_opening_a_weight_file(tmp_path, monkeypatch):
    (tmp_path / "config.json").write_text(json.dumps(dict(hub_config("1b"), use_parallel_residual=False)))
    (tmp_path / "pytorch_model.bin").write_bytes(b"not a pickle")
    (tmp_path / "model.safetensors").write_bytes(b"not a safetensors file")
    import safetensors

    def no_read(*a, **k):
        raise AssertionError("a weight file was opened")
    monkeypatch.setattr(safetensors, "safe_open", no_read)
    monkeypatch.setattr(torch, "load", no_read)
    monkeypatch.setattr(reader.B200NeoX, "__init__", lambda *a, **k: (_ for _ in ()).throw(AssertionError("allocated")))
    with pytest.raises(AttributeError, match="use_parallel_residual"):
        reader.load_reader(str(tmp_path))


def test_pickle_listing(tmp_path):
    (tmp_path / "pytorch_model.bin").write_bytes(b"")
    assert reader._shard_files(str(tmp_path)) == [str(tmp_path / "pytorch_model.bin")]
    index = {"weight_map": {"a": "pytorch_model-00002-of-00002.bin", "b": "pytorch_model-00001-of-00002.bin"}}
    (tmp_path / "pytorch_model.bin.index.json").write_text(json.dumps(index))
    assert reader._shard_files(str(tmp_path)) == [str(tmp_path / f"pytorch_model-0000{i}-of-00002.bin") for i in (1, 2)]
    (tmp_path / "model.safetensors").write_bytes(b"")              # safetensors first when both are present
    assert reader._shard_files(str(tmp_path)) == [str(tmp_path / "model.safetensors")]


def test_pickle_fixture_reads_back(tmp_path):
    F.build_dir(str(tmp_path), pickle=True)
    names = dict(reader._tensors(str(tmp_path / "pytorch_model.bin")))
    sd = F.seeded_state_dict()
    assert set(names) == set(sd) | set(F.legacy_buffers())
    assert all(torch.equal(names[k], v) for k, v in sd.items())
    skipped = [k for k in names if k.endswith(reader.B200NeoX._buffers)]
    assert sorted(skipped) == sorted(F.legacy_buffers())


def test_expected_keys():
    keys = reader.neox_expected_keys(reader.neox_geometry(F.CONFIG))
    assert len(keys) == 4 + 2 * 12 and len(set(keys)) == len(keys)
    assert set(keys) == set(F.seeded_state_dict())
    assert not any(k.endswith(reader.B200NeoX._buffers) for k in keys)


def test_neox_abi_refusals_need_no_device():
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
    NX, z = (_lib.RSB_LLM_NEOX, _lib.RSB_DTYPE_F16), f(0.0)
    ok = (*NX, 2, 512, 2, 2, 2048, 1000, 2048, 64, f(1e4), f(1e-5), z, 0)
    assert L.rsb_llm_create(*ok, None) == _lib.RSB_ERR_INVALID
    bad = [
        ((*NX, 2, 6144, 64, 64, 24576, 1000, 2048, 24, f(1e4), f(1e-5), z, 0), _lib.RSB_ERR_UNSUPPORTED, b"head_dim"),   # 96
        ((*NX, 2, 512, 3, 3, 2048, 1000, 2048, 64, f(1e4), f(1e-5), z, 0), _lib.RSB_ERR_UNSUPPORTED, b"head_dim"),
        ((*NX, 2, 512, 1, 1, 2048, 1000, 2048, 64, f(1e4), f(1e-5), z, 0), _lib.RSB_ERR_UNSUPPORTED, b"head_dim"),     # 512
        ((*NX, 2, 512, 2, 2, 2048, 1000, 2048, 63, f(1e4), f(1e-5), z, 0), _lib.RSB_ERR_UNSUPPORTED, b"rotary"),
        ((*NX, 2, 512, 2, 2, 2048, 1000, 2048, 0, f(1e4), f(1e-5), z, 0), _lib.RSB_ERR_INVALID, b"rotary"),
        ((*NX, 2, 512, 2, 2, 2048, 1000, 2048, 258, f(1e4), f(1e-5), z, 0), _lib.RSB_ERR_INVALID, b"rotary"),
        ((*NX, 2, 512, 2, 2, 2000, 1000, 2048, 64, f(1e4), f(1e-5), z, 0), _lib.RSB_ERR_UNSUPPORTED, b"intermediate"),
        ((*NX, 2, 10240, 40, 40, 40960, 1000, 2048, 64, f(1e4), f(1e-5), z, 0), _lib.RSB_ERR_UNSUPPORTED, b"hidden"),
        ((*NX, 2, 10240, 80, 80, 40960, 1000, 2048, 32, f(1e4), f(1e-5), z, 0), _lib.RSB_ERR_UNSUPPORTED, b"hidden"),
        ((*NX, 0, 512, 2, 2, 2048, 1000, 2048, 64, f(1e4), f(1e-5), z, 0), _lib.RSB_ERR_INVALID, b"positive"),
        ((*NX, 2, 512, 2, 2, 2048, 0, 2048, 64, f(1e4), f(1e-5), z, 0), _lib.RSB_ERR_INVALID, b"positive"),
        ((*NX, 2, 512, 2, 2, 2048, 1000, 2048, 64, f(0.0), f(1e-5), z, 0), _lib.RSB_ERR_INVALID, b"rotary_base"),
        ((*NX, 2, 512, 2, 2, 2048, 1000, 2048, 64, f(1e4), f(0.0), z, 0), _lib.RSB_ERR_INVALID, b"ln_eps"),
        # combinations only the one constructor can express
        ((*NX, 2, 512, 2, 1, 2048, 1000, 2048, 64, f(1e4), f(1e-5), z, 0), _lib.RSB_ERR_UNSUPPORTED, b"kv_heads"),
        ((*ok[:-1], 1), _lib.RSB_ERR_UNSUPPORTED, b"tied"),
        ((*ok[:-2], f(8.0), 0), _lib.RSB_ERR_INVALID, b"clip_qkv"),
    ]
    for args, rc, msg in bad:
        assert L.rsb_llm_create(*args, ctypes.byref(h)) == rc, args
        assert msg in L.rsb_llm_last_error(), (args, L.rsb_llm_last_error())
        assert h.value is None
    # the LayerNorm diagnostic: refused before any launch (the pointers are never dereferenced)
    p = ctypes.c_void_p(16)
    ln = [
        ((8192 + 8, f(1e-5), p, None, None, 4, p, p, None, None, p, None), _lib.RSB_ERR_UNSUPPORTED, b"hidden"),
        ((502, f(1e-5), p, None, None, 4, p, p, None, None, p, None), _lib.RSB_ERR_UNSUPPORTED, b"hidden"),
        ((0, f(1e-5), p, None, None, 4, p, p, None, None, p, None), _lib.RSB_ERR_UNSUPPORTED, b"hidden"),
        ((512, f(1e-5), None, None, None, 4, p, p, None, None, p, None), _lib.RSB_ERR_INVALID, b"null"),
        ((512, f(1e-5), p, None, None, 4, p, None, None, None, p, None), _lib.RSB_ERR_INVALID, b"null"),
        ((512, f(1e-5), p, None, None, 4, p, p, p, p, p, None), _lib.RSB_ERR_INVALID, b"null"),
        ((512, f(1e-5), p, None, None, 4, None, None, p, p, p, p), _lib.RSB_ERR_INVALID, b"null"),
        ((512, f(1e-5), p, None, None, -1, p, p, None, None, p, None), _lib.RSB_ERR_INVALID, b"n_rows"),
        ((512, f(0.0), p, None, None, 4, p, p, None, None, p, None), _lib.RSB_ERR_INVALID, b"eps"),
    ]
    for args, rc, msg in ln:
        assert L.rsb_llm_layernorm(*args, None) == rc, args
        assert msg in L.rsb_llm_last_error(), (args, L.rsb_llm_last_error())
    assert L.rsb_llm_layernorm(512, f(1e-5), p, p, None, 0, p, p, p, p, p, p, None) == _lib.RSB_OK   # no rows


@pytest.mark.parametrize("heads, head_dim", [(2, 256), (8, 64), (32, 80), (16, 128)])
def test_qkv_permutation(heads, head_dim):
    """The loader's three strided copies restated in numpy: part p of head h lands at rows p * hidden + h * head_dim,
    which is what the oracle's view(S, heads, 3 * head_dim) chunking reads."""
    H = heads * head_dim
    w = np.arange(3 * H * 4).reshape(3 * H, 4)
    perm = O.qkv_permutation(heads, head_dim)
    copied = np.empty_like(w)
    for p in range(3):                            # cudaMemcpy2DAsync(dst + p H, head_dim rows, src + p head_dim, 3 head_dim)
        for h in range(heads):
            copied[p * H + h * head_dim:p * H + (h + 1) * head_dim] = w[(3 * h + p) * head_dim:(3 * h + p + 1) * head_dim]
    assert np.array_equal(copied, w[perm])
    x = np.random.default_rng(0).standard_normal((5, 3 * H))      # one projected row per token
    q, k, v = (x.reshape(5, heads, 3 * head_dim)[..., i * head_dim:(i + 1) * head_dim].reshape(5, H) for i in range(3))
    assert np.array_equal(x[:, perm], np.concatenate([q, k, v], axis=1))
