"""bf16 readers, host side: the dtype argument of `load_reader` / `_Reader` and the `model.lm_dtype` key, each refused
before any weight file is opened or device memory allocated; `rsb_llm_create`'s dtype refusals before any CUDA call;
the index creators' refusal of RSB_DTYPE_BF16; and `main_ric.py`'s plumbing of `+model.lm_dtype=bfloat16` to
`load_reader`."""
import ctypes
import importlib.util
import json
import os
import sys

import numpy as np
import pytest
import torch

from retrieval_scaling_b200 import _lib, reader

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CONF = os.path.join(ROOT, "ric", "conf")
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

import llama_fixture as F  # noqa: E402

BAD = [torch.float32, torch.float64, torch.int8, "fp16", "bf16", "half", "float32", None, 16]


@pytest.mark.parametrize("dtype, want", [(torch.float16, torch.float16), ("float16", torch.float16),
                                         (torch.bfloat16, torch.bfloat16), ("bfloat16", torch.bfloat16)])
def test_reader_dtype_accepts_torch_dtypes_and_names(dtype, want):
    assert reader.reader_dtype(dtype) == want


@pytest.mark.parametrize("dtype", BAD)
def test_reader_dtype_refuses_everything_else(dtype):
    with pytest.raises(ValueError, match="dtype"):
        reader.reader_dtype(dtype)


def _no_reads(monkeypatch):
    import safetensors

    def no_read(*a, **k):
        raise AssertionError("a weight file was opened")
    monkeypatch.setattr(safetensors, "safe_open", no_read)
    monkeypatch.setattr(torch, "load", no_read)
    for cls in (reader.B200Llama, reader.B200NeoX, reader.B200Olmo):
        monkeypatch.setattr(cls, "_create", lambda *a, **k: (_ for _ in ()).throw(AssertionError("allocated")))


@pytest.mark.parametrize("dtype", [torch.float32, "bf16", None])
def test_load_reader_refuses_a_dtype_before_reading_weights(tmp_path, monkeypatch, dtype):
    (tmp_path / "config.json").write_text(json.dumps(F.CONFIG))
    (tmp_path / "model.safetensors").write_bytes(b"not a safetensors file")
    _no_reads(monkeypatch)
    with pytest.raises(ValueError, match="dtype"):
        reader.load_reader(str(tmp_path), dtype=dtype)


@pytest.mark.parametrize("cls, cfg", [(reader.B200Llama, F.CONFIG),
                                      (reader.B200NeoX, dict(model_type="gpt_neox", num_hidden_layers=1,
                                                             hidden_size=512, num_attention_heads=2,
                                                             intermediate_size=2048, vocab_size=1000)),
                                      (reader.B200Olmo, dict(F.CONFIG, model_type="olmo2"))])
def test_reader_constructor_refuses_a_dtype_first(monkeypatch, cls, cfg):
    """ValueError before the geometry is read and before the CUDA check: a bad config or a CPU-only host would raise
    something else."""
    _no_reads(monkeypatch)
    with pytest.raises(ValueError, match="dtype"):
        cls(cfg, dtype=torch.float32)
    with pytest.raises(ValueError, match="dtype"):
        cls(dict(cfg, model_type="bert"), dtype="float64")


def test_create_dtype_refusals_before_any_cuda_call():
    L = _lib.lib()
    h = ctypes.c_void_p(0)
    geometry = (2, 512, 4, 1, 1024, 1000, 4096, 128, ctypes.c_float(1e4), ctypes.c_float(1e-5), ctypes.c_float(0.0), 0)
    for dtype in (7, _lib.RSB_DTYPE_F32):
        for out in (None, ctypes.byref(h)):
            assert L.rsb_llm_create(_lib.RSB_LLM_LLAMA, dtype, *geometry, out) == _lib.RSB_ERR_INVALID
        assert b"dtype" in L.rsb_llm_last_error()
        assert h.value is None
    assert _lib.RSB_DTYPE_BF16 == 3


def test_index_creators_refuse_bf16():
    L = _lib.lib()
    h = ctypes.c_void_p(0)
    BF16 = _lib.RSB_DTYPE_BF16
    assert L.rsb_flat_create(768, BF16, ctypes.byref(h)) == _lib.RSB_ERR_INVALID
    assert L.rsb_ivfflat_create(768, 16, BF16, ctypes.byref(h)) == _lib.RSB_ERR_INVALID
    assert not h.value
    assert L.rsb_refine_workspace_bytes(4, 10, 5, 768, BF16, 100, 100, 0) == 0


def _ppl_cfg(tmp_path, extra):
    from retrieval_scaling_b200 import config as C
    d = F.build_dir(str(tmp_path / "reader"), dict(num_hidden_layers=1, max_position_embeddings=40), seed=4)
    rng = np.random.default_rng(2)
    eval_path = tmp_path / "eval.jsonl"
    with open(eval_path, "w") as f:
        f.write(json.dumps({"text": " ".join(f"w{i}" for i in rng.integers(2, 1000, 50))}) + "\n")
    ov = ["datastore.domain=d", "evaluation.domain=d", f"evaluation.data.eval_data={eval_path}", f"model.lm_model={d}",
          "evaluation.data.max_eval_data_seq_length=24", "evaluation.data.eval_stride=12",
          "tasks.eval.inference=true", *extra]
    return C.load_config("perplexity", CONF, ov)


@pytest.mark.parametrize("value", ["float32", "fp16", "bf16"])
def test_lm_dtype_key_is_refused_before_the_reader_loads(tmp_path, monkeypatch, value):
    from retrieval_scaling_b200 import perplexity as P
    from retrieval_scaling_b200 import search
    cfg = _ppl_cfg(tmp_path, [f"+model.lm_dtype={value}"])
    monkeypatch.setattr(reader, "load_reader", lambda *a, **k: (_ for _ in ()).throw(AssertionError("loaded")))
    monkeypatch.setattr(search, "load_eval_data", lambda *a, **k: (_ for _ in ()).throw(AssertionError("read data")))
    with pytest.raises(ValueError, match="model.lm_dtype"):
        P.evaluate_perplexity(cfg)


@pytest.mark.parametrize("extra, want", [([], torch.float16), (["+model.lm_dtype=float16"], torch.float16),
                                         (["+model.lm_dtype=bfloat16"], torch.bfloat16)])
def test_main_ric_carries_lm_dtype_to_load_reader(tmp_path, monkeypatch, extra, want):
    """ric/main_ric.py's main() with tasks.eval.inference=true: the reader is loaded with the key's dtype (float16
    when the key is absent), and its losses are what the run summarises."""
    seen = []

    class FakeReader:
        max_position_embeddings = 40

        def loss(self, ids, labels):
            return [1.0 for _ in ids]

    def fake_load_reader(path, device=None, dtype=torch.float16):
        seen.append((path, dtype))
        return FakeReader()
    monkeypatch.setattr(reader, "load_reader", fake_load_reader)
    cfg = _ppl_cfg(tmp_path, extra + [f"evaluation.results_only_log_file={tmp_path / 'res.log'}"])
    spec = importlib.util.spec_from_file_location("main_ric_under_test", os.path.join(ROOT, "ric", "main_ric.py"))
    main_ric = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(main_ric)
    main_ric.main(cfg)
    assert [d for _, d in seen] == [want] and seen[0][0] == cfg.model.lm_model
    assert "perplexity" in open(tmp_path / "res.log").read()


def test_perplexity_conf_documents_the_key():
    text = open(os.path.join(CONF, "perplexity.yaml")).read()
    assert "+model.lm_dtype=bfloat16" in text
