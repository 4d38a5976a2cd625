"""GPU query encoder with the reference's call protocol (`src/search.py:239-258,83-96`):

    model, tokenizer, _ = load_retriever(name)            # contriever/src/contriever.py:103-138
    model.eval().to(device).half()                        # no-ops here: the CUDA path is always fp16 / inference
    emb = model(input_ids=..., attention_mask=..., token_type_ids=...)   # -> Tensor[B, 768] fp16

The forward pass is librsb's `rsb_bert_forward` (wgmma tensor-core GEMMs fed by TMA with fused bias / GELU /
residual epilogues, fused embedding+LayerNorm, shared-memory attention, mean / CLS pooling) on the un-padded
token stream.  No CPU / eager-PyTorch fallback: constructing the model without CUDA raises.
"""
from __future__ import annotations

import ctypes
from typing import Dict, Optional

import torch

from . import _lib

BERT_BASE = dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
                 vocab_size=30522, max_position_embeddings=512, type_vocab_size=2, layer_norm_eps=1e-12)


def _cfg_get(config, key):
    if isinstance(config, dict):
        return config.get(key, BERT_BASE[key])
    return getattr(config, key, BERT_BASE[key])


def expected_keys(num_hidden_layers: int):
    """Every weight the forward pass reads (HF BertModel names, SURVEY.md App. B)."""
    keys = ["embeddings.word_embeddings.weight", "embeddings.position_embeddings.weight",
            "embeddings.token_type_embeddings.weight", "embeddings.LayerNorm.weight", "embeddings.LayerNorm.bias"]
    for i in range(num_hidden_layers):
        p = f"encoder.layer.{i}."
        for nm in ("attention.self.query", "attention.self.key", "attention.self.value", "attention.output.dense",
                   "intermediate.dense", "output.dense", "attention.output.LayerNorm", "output.LayerNorm"):
            keys += [p + nm + ".weight", p + nm + ".bias"]
    return keys


class B200Contriever:
    """`Contriever(BertModel)` (pooling="average", contriever.py:11-55) or plain HF BERT + CLS row (pooling="cls")."""

    # Sequences per forward that `search.embed_queries` may group: the kernels run on the un-padded token stream,
    # so the batch composition does not change any sequence's output; 2048 is where the GEMMs fill the GPU.
    encode_group = 2048

    def __init__(self, config=None, pooling: str = "average", device=None):
        if not torch.cuda.is_available():
            raise RuntimeError("B200Contriever needs a CUDA device (sm_90a): there is no CPU path")
        if pooling not in ("average", "cls"):
            raise ValueError(f"unknown pooling {pooling!r}")
        self.L = _lib.lib()
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.config = {k: _cfg_get(config or {}, k) for k in BERT_BASE}
        self.pooling = pooling
        self._h = ctypes.c_void_p(0)
        c = self.config
        with torch.cuda.device(self.device):
            rc = self.L.rsb_bert_create(c["hidden_size"], c["num_hidden_layers"], c["num_attention_heads"],
                                        c["intermediate_size"], c["vocab_size"], c["max_position_embeddings"],
                                        c["type_vocab_size"], ctypes.c_float(c["layer_norm_eps"]), ctypes.byref(self._h))
        self._check(rc)
        self._ws: Optional[torch.Tensor] = None
        self.loaded = set()

    def _check(self, rc):
        if rc == _lib.RSB_OK:
            return
        msg = self.L.rsb_bert_last_error().decode("utf-8", "replace")
        if rc == _lib.RSB_ERR_INVALID:
            raise ValueError(msg)
        if rc == _lib.RSB_ERR_UNSUPPORTED:
            raise NotImplementedError(msg)
        if rc == _lib.RSB_ERR_OOM:
            raise MemoryError(msg)
        raise _lib.RsbError(f"librsb encoder error {rc}: {msg}")

    def __del__(self):
        try:
            if getattr(self, "_h", None) and self._h.value:
                self.L.rsb_bert_free(self._h)
                self._h = ctypes.c_void_p(0)
        except Exception:
            pass

    # -- nn.Module-like surface used by the reference -----------------------------------------------------------
    def eval(self):
        return self

    def half(self):
        return self

    def to(self, *a, **k):
        return self

    def cuda(self, *a, **k):
        return self

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        """HF BertModel keys (SURVEY.md App. B); a leading 'bert.' / 'encoder_q.' style prefix is not stripped
        here (contriever.load_retriever does that before calling, `contriever.py:121-125`)."""
        stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        unexpected = []
        with torch.cuda.device(self.device):
            for name, t in sd.items():
                if name.endswith("position_ids") or name.startswith("pooler."):
                    continue
                w = t.detach().to(device=self.device, dtype=torch.float16).contiguous()
                rc = self.L.rsb_bert_load(self._h, name.encode(), ctypes.c_void_p(w.data_ptr()), w.numel(), stream)
                if rc == _lib.RSB_ERR_INVALID and b"unknown weight" in self.L.rsb_bert_last_error():
                    unexpected.append(name)
                    continue
                self._check(rc)
                self.loaded.add(name)
            torch.cuda.current_stream().synchronize()
        if strict and unexpected:
            raise KeyError(f"unexpected keys in state_dict: {unexpected[:5]}")
        return unexpected

    # -- forward ------------------------------------------------------------------------------------------------
    def forward_varlen(self, ids: torch.Tensor, cu_seqlens: torch.Tensor, max_seqlen: int,
                       token_types: Optional[torch.Tensor] = None, total_tokens: Optional[int] = None) -> torch.Tensor:
        B = cu_seqlens.numel() - 1
        T = int(ids.numel()) if total_tokens is None else int(total_tokens)
        out = torch.empty((B, self.config["hidden_size"]), dtype=torch.float16, device=self.device)
        need = self.L.rsb_bert_workspace_bytes(self._h, T)
        if self._ws is None or self._ws.numel() < need:
            self._ws = None
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        tt = ctypes.c_void_p(token_types.data_ptr()) if token_types is not None else ctypes.c_void_p(0)
        rc = self.L.rsb_bert_forward(self._h, ctypes.c_void_p(ids.data_ptr()), tt, ctypes.c_void_p(cu_seqlens.data_ptr()),
                                     B, T, int(max_seqlen), 0 if self.pooling == "average" else 1,
                                     ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(self._ws.data_ptr()),
                                     self._ws.numel(), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        self._check(rc)
        return out

    def __call__(self, input_ids=None, attention_mask=None, token_type_ids=None, **_unused) -> torch.Tensor:
        with torch.cuda.device(self.device):
            input_ids = input_ids.to(self.device)
            Bsz, S = input_ids.shape
            if attention_mask is None:
                attention_mask = torch.ones_like(input_ids)
            mask = attention_mask.to(self.device).bool()
            lens = mask.sum(dim=1, dtype=torch.int32)
            cu = torch.zeros(Bsz + 1, dtype=torch.int32, device=self.device)
            cu[1:] = torch.cumsum(lens, 0)
            ids = input_ids[mask].to(torch.int32).contiguous()           # right-padded batches: order is preserved
            tts = None
            if token_type_ids is not None:
                tts = token_type_ids.to(self.device)[mask].to(torch.int32).contiguous()
            return self.forward_varlen(ids, cu, S, tts)

    forward = __call__

    def expected_keys(self):
        return expected_keys(self.config["num_hidden_layers"])

    def missing_keys(self):
        return [k for k in self.expected_keys() if k not in self.loaded]

    def require_all_weights(self, source: str = "state_dict"):
        """librsb allocates the weights with plain cudaMalloc: a checkpoint whose keys do not match would leave them
        uninitialised and the model would return garbage without any error -- refuse instead."""
        missing = self.missing_keys()
        if missing:
            raise KeyError(f"{source}: {len(missing)} of {len(self.expected_keys())} encoder weights were not found "
                           f"(first missing: {missing[:4]}); keys must follow HF BertModel naming after the reference's "
                           f"'encoder_q.' / 'encoder.' / 'bert.' prefix stripping")

    @property
    def launches(self) -> int:
        return int(self.L.rsb_bert_launches(self._h))


def random_state_dict(config=None, seed: int = 0, device="cpu") -> Dict[str, torch.Tensor]:
    """Seeded random-init weights with the HF key names (benchmarks run without pretrained checkpoints)."""
    c = {k: _cfg_get(config or {}, k) for k in BERT_BASE}
    g = torch.Generator(device="cpu").manual_seed(seed)
    H, I = c["hidden_size"], c["intermediate_size"]

    def n(*shape, std):
        return (torch.randn(*shape, generator=g) * std).to(device)

    sd = {
        "embeddings.word_embeddings.weight": n(c["vocab_size"], H, std=0.5),
        "embeddings.position_embeddings.weight": n(c["max_position_embeddings"], H, std=0.3),
        "embeddings.token_type_embeddings.weight": n(c["type_vocab_size"], H, std=0.3),
        "embeddings.LayerNorm.weight": 1.0 + n(H, std=0.1),
        "embeddings.LayerNorm.bias": n(H, std=0.1),
    }
    for i in range(c["num_hidden_layers"]):
        p = f"encoder.layer.{i}."
        for nm, (o, k_) in {"attention.self.query": (H, H), "attention.self.key": (H, H), "attention.self.value": (H, H),
                            "attention.output.dense": (H, H), "intermediate.dense": (I, H), "output.dense": (H, I)}.items():
            sd[p + nm + ".weight"] = n(o, k_, std=0.04)
            sd[p + nm + ".bias"] = n(o, std=0.02)
        for nm in ("attention.output.LayerNorm", "output.LayerNorm"):
            sd[p + nm + ".weight"] = 1.0 + n(H, std=0.1)
            sd[p + nm + ".bias"] = n(H, std=0.1)
    return sd


def strip_wrapper_prefix(sd: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    """Checkpoint key names -> HF BertModel key names.

    The reference (`contriever.py:121-125`) keeps the keys containing 'encoder_q.' (MoCo wrapper: query tower) or else
    'encoder.' (in-batch wrapper) and removes that substring with `str.replace` -- which removes EVERY occurrence, so
    an in-batch checkpoint's 'encoder.encoder.layer.N...' keys become 'layer.N...' and are silently dropped by
    `load_state_dict(strict=False)`.  That quirk is not copied: only the LEADING wrapper prefix is stripped, and
    `load_retriever` refuses a checkpoint that does not provide every encoder weight."""
    keys = list(sd.keys())
    if any(k.startswith("encoder_q.") for k in keys):
        return {k[len("encoder_q."):]: v for k, v in sd.items() if k.startswith("encoder_q.")}
    if any(k.startswith("encoder.embeddings.") or k.startswith("encoder.encoder.") for k in keys):
        return {k[len("encoder."):]: v for k, v in sd.items() if k.startswith("encoder.")}
    if any(k.startswith("bert.") for k in keys):
        return {k[len("bert."):]: v for k, v in sd.items() if k.startswith("bert.")}
    return dict(sd)


def read_retriever_files(model_path: str, tokenizer_name: Optional[str] = None):
    """(state_dict with HF BertModel keys, config, tokenizer, retriever_model_id) from a local `checkpoint.pth`
    directory (`contriever.py:105-126`) or an HF model directory / cache entry (`:127-136`).  Pure host code."""
    import os

    import transformers

    def load_hf(cls, name):            # reference `utils.load_hf`: local files first
        try:
            return cls.from_pretrained(name, local_files_only=True)
        except Exception:
            return cls.from_pretrained(name, local_files_only=False)

    ckpt = os.path.join(model_path, "checkpoint.pth")
    if os.path.exists(ckpt):
        blob = torch.load(ckpt, map_location="cpu", weights_only=False)
        opt = blob["opt"]
        model_id = getattr(opt, "retriever_model_id", "bert-base-multilingual-cased")
        sd = strip_wrapper_prefix(blob["model"])
        cfg = load_hf(transformers.AutoConfig, model_id)
        tokenizer = load_hf(transformers.AutoTokenizer, model_id)
    else:
        model_id = model_path
        cfg = load_hf(transformers.AutoConfig, model_path)
        tokenizer = load_hf(transformers.AutoTokenizer, tokenizer_name or model_path)
        hf = load_hf(transformers.AutoModel, model_path)
        sd = strip_wrapper_prefix(hf.state_dict())
    if getattr(cfg, "model_type", "bert") != "bert":
        raise AttributeError(f"{model_path}: only BERT-architecture encoders run on the GPU path")
    return sd, cfg, tokenizer, model_id


def load_retriever(model_path: str, tokenizer_name: Optional[str] = None, pooling: str = "average", fp16: bool = True,
                   random_init: bool = False):
    """(model, tokenizer, retriever_model_id) like `contriever.src.contriever.load_retriever` (:103-138).
    Needs the checkpoint / tokenizer on local disk or in the HF cache (this image has no network)."""
    if random_init:
        model = B200Contriever(BERT_BASE, pooling)
        model.load_state_dict(random_state_dict(BERT_BASE, 0))
        return model, None, model_path
    sd, cfg, tokenizer, model_id = read_retriever_files(model_path, tokenizer_name)
    if not fp16:
        import warnings
        warnings.warn("no_fp16 / fp16=False was requested, but the encoder computes in fp16 with fp32 accumulation "
                      "only (the reference's default path, src/search.py:257-258); continuing in fp16")
    model = B200Contriever(cfg, pooling)
    model.load_state_dict(sd, strict=False)
    model.require_all_weights(model_path)
    return model, tokenizer, model_id
