"""GPU query encoder with the reference's call protocol (`src/search.py:239-258,83-96`):

    model, tokenizer, _ = load_retriever(name)            # contriever/src/contriever.py:103-138
    model.eval().to(device).half()                        # no-ops here: the CUDA path is always fp16 / inference
    emb = model(input_ids=..., attention_mask=..., token_type_ids=...)   # -> Tensor[B, 768] fp16

The forward pass is librsb's `rsb_bert_forward` (wgmma tensor-core GEMMs fed by TMA with fused bias / GELU /
residual epilogues, fused embedding+LayerNorm, shared-memory attention, mean / CLS pooling) on the un-padded
token stream.  No CPU / eager-PyTorch fallback: constructing the model without CUDA raises.  An HF checkpoint whose
`model_type` is "roberta" (DRAGON-RoBERTa's query and context encoders) loads as `B200Roberta`: the same layers behind
RoBERTa's embedding positions (`rsb_roberta_create`).

The same library runs the sentence-transformers retrievers the reference loads with `SentenceTransformer(name)`
(`src/search.py:49-61`, `src/embed.py:25-40`): `load_sentence_transformer(path)` reads the model directory into a
`SentenceTransformerEncoder` whose transformer is a T5 encoder (`B200T5Encoder`, GTR-T5) or a BERT-base model
(`B200Contriever`, e5-base), with the Pooling -> Dense -> Normalize head run by `rsb_bert_forward` as well.
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

    def __init__(self, config=None, pooling: str = "average", device=None, dense: bool = False, normalize: bool = False):
        """`dense` / `normalize` add the sentence-transformers head after the pooling: a 768 x 768 Linear
        (`dense.weight`, optional `dense.bias`) and L2 normalisation."""
        if not torch.cuda.is_available():
            raise RuntimeError(f"{type(self).__name__} needs a CUDA device (sm_90a): there is no CPU path")
        if pooling not in ("average", "cls"):
            raise ValueError(f"unknown pooling {pooling!r}")
        self.L = _lib.lib()
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.pooling, self.dense, self.normalize = pooling, bool(dense), bool(normalize)
        self._pool_flags = ((_lib.POOL_MEAN if pooling == "average" else _lib.POOL_CLS)
                            | (_lib.POOL_DENSE if dense else 0) | (_lib.POOL_NORMALIZE if normalize else 0))
        self._h = ctypes.c_void_p(0)
        self._ws: Optional[torch.Tensor] = None
        self.loaded = set()
        with torch.cuda.device(self.device):
            self._create(config)

    def _create(self, config):
        self.config = {k: _cfg_get(config or {}, k) for k in BERT_BASE}
        c = self.config
        rc = self.L.rsb_bert_create(c["hidden_size"], c["num_hidden_layers"], c["num_attention_heads"],
                                    c["intermediate_size"], c["vocab_size"], c["max_position_embeddings"],
                                    c["type_vocab_size"], ctypes.c_float(c["layer_norm_eps"]), ctypes.byref(self._h))
        self._check(rc)

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

    _ALIASES: Dict[str, str] = {}

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
                self.loaded.add(self._ALIASES.get(name, name))
            torch.cuda.current_stream().synchronize()
        if strict and unexpected:
            raise KeyError(f"unexpected keys in state_dict: {unexpected[:5]}")
        return unexpected

    # -- forward ------------------------------------------------------------------------------------------------
    def forward_varlen(self, ids: torch.Tensor, cu_seqlens: torch.Tensor, max_seqlen: int,
                       token_types: Optional[torch.Tensor] = None, total_tokens: Optional[int] = None,
                       pool_flags: Optional[int] = None) -> torch.Tensor:
        """[B, 768] fp16 with the model's pooling and head, or [T, 768] with pool_flags=_lib.POOL_TOKENS."""
        B = cu_seqlens.numel() - 1
        T = int(ids.numel()) if total_tokens is None else int(total_tokens)
        flags = self._pool_flags if pool_flags is None else int(pool_flags)
        rows = T if flags == _lib.POOL_TOKENS else B
        out = torch.empty((rows, self.config["hidden_size"]), dtype=torch.float16, device=self.device)
        need = self.L.rsb_bert_workspace_bytes(self._h, T)
        if self._ws is None or self._ws.numel() < need:
            self._ws = None
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        tt = ctypes.c_void_p(token_types.data_ptr()) if token_types is not None else ctypes.c_void_p(0)
        rc = self.L.rsb_bert_forward(self._h, ctypes.c_void_p(ids.data_ptr()), tt, ctypes.c_void_p(cu_seqlens.data_ptr()),
                                     B, T, int(max_seqlen), flags,
                                     ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(self._ws.data_ptr()),
                                     self._ws.numel(), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        self._check(rc)
        return out

    def _unpad(self, input_ids, attention_mask, token_type_ids):
        input_ids = input_ids.to(self.device)
        Bsz, S = input_ids.shape
        if attention_mask is None:
            attention_mask = torch.ones_like(input_ids)
        mask = attention_mask.to(self.device).bool()
        lens = mask.sum(dim=1, dtype=torch.int32)
        cu = torch.zeros(Bsz + 1, dtype=torch.int32, device=self.device)
        cu[1:] = torch.cumsum(lens, 0)
        ids = input_ids[mask].to(torch.int32).contiguous()               # right-padded batches: order is preserved
        tts = None
        if token_type_ids is not None:
            tts = token_type_ids.to(self.device)[mask].to(torch.int32).contiguous()
        return ids, cu, S, tts

    def __call__(self, input_ids=None, attention_mask=None, token_type_ids=None, **_unused) -> torch.Tensor:
        with torch.cuda.device(self.device):
            ids, cu, S, tts = self._unpad(input_ids, attention_mask, token_type_ids)
            return self.forward_varlen(ids, cu, S, tts)

    forward = __call__

    def hidden_states(self, input_ids=None, attention_mask=None, token_type_ids=None):
        """Diagnostic (tests): the final hidden states of the real tokens, before any pooling -- BERT after the last
        LayerNorm, T5 after final_layer_norm -- as ([T, 768] fp16 rows in batch order, cu_seqlens [B + 1] int32)."""
        with torch.cuda.device(self.device):
            ids, cu, S, tts = self._unpad(input_ids, attention_mask, token_type_ids)
            return self.forward_varlen(ids, cu, S, tts, pool_flags=_lib.POOL_TOKENS), cu

    def expected_keys(self):
        return expected_keys(self.config["num_hidden_layers"]) + (["dense.weight"] if self.dense else [])

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
    """Checkpoint key names -> HF BertModel key names (RobertaModel uses the same names, behind 'roberta.').

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
    for prefix in ("bert.", "roberta."):
        if any(k.startswith(prefix) for k in keys):
            return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}
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
    model_type = getattr(cfg, "model_type", "bert")
    if model_type == "roberta":
        _roberta_config(cfg)
    elif model_type != "bert":
        raise AttributeError(f"{model_path}: only BERT-architecture encoders (BERT, RoBERTa-base) run on the GPU path")
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
    cls = B200Roberta if getattr(cfg, "model_type", "bert") == "roberta" else B200Contriever
    model = cls(cfg, pooling)
    model.load_state_dict(sd, strict=False)
    model.require_all_weights(model_path)
    return model, tokenizer, model_id


# ----------------------------------------------------------------------------------------------------------------
# RoBERTa-base (DRAGON-RoBERTa's query and context encoders)
# ----------------------------------------------------------------------------------------------------------------
ROBERTA_BASE = dict(BERT_BASE, vocab_size=50265, max_position_embeddings=514, type_vocab_size=1, layer_norm_eps=1e-5,
                    pad_token_id=1)


def _roberta_config(config) -> dict:
    """The RoBERTa geometry the kernels run (hidden 768, 12 heads, erf GELU), or AttributeError."""
    get = (lambda k, d=None: config.get(k, d)) if isinstance(config, dict) else (lambda k, d=None: getattr(config, k, d))
    geom = dict(hidden_size=get("hidden_size", 768), num_attention_heads=get("num_attention_heads", 12),
                hidden_act=get("hidden_act", "gelu"))
    if geom != dict(hidden_size=768, num_attention_heads=12, hidden_act="gelu"):
        raise AttributeError(f"unsupported RoBERTa geometry {geom}: only RoBERTa-base (hidden 768, 12 heads, GELU) "
                             f"runs on the GPU path")
    c = {k: get(k, ROBERTA_BASE[k]) for k in ROBERTA_BASE}
    if c["pad_token_id"] is None:
        raise AttributeError("RoBERTa config without pad_token_id: its positions are counted from padding_idx")
    return c


class B200Roberta(B200Contriever):
    """HF `RobertaModel` (RoBERTa-base geometry) + CLS row or mean pooling on librsb (`rsb_roberta_create`): the BERT
    layers behind RoBERTa's positions, padding_idx + the count of non-pad ids up to each token.  Same call surface
    and HF key names as `B200Contriever`; token_type_ids other than 0 on a type_vocab_size 1 model raise ValueError,
    as HF raises on them."""

    def _create(self, config):
        self.config = _roberta_config(config or {})
        c = self.config
        rc = self.L.rsb_roberta_create(c["num_hidden_layers"], c["intermediate_size"], c["vocab_size"],
                                       c["max_position_embeddings"], c["type_vocab_size"],
                                       ctypes.c_float(c["layer_norm_eps"]), int(c["pad_token_id"]), ctypes.byref(self._h))
        self._check(rc)

    def require_all_weights(self, source: str = "state_dict"):
        missing = self.missing_keys()
        if missing:
            raise KeyError(f"{source}: {len(missing)} of {len(self.expected_keys())} RoBERTa encoder weights were not "
                           f"found (first missing: {missing[:4]}); keys must follow HF RobertaModel naming after the "
                           f"'roberta.' prefix stripping")


# ----------------------------------------------------------------------------------------------------------------
# T5 encoder (GTR-T5) and the sentence-transformers model directory
# ----------------------------------------------------------------------------------------------------------------
T5_BASE = dict(num_layers=12, d_ff=3072, vocab_size=32128, relative_attention_num_buckets=32,
               relative_attention_max_distance=128, layer_norm_epsilon=1e-6)
T5_MAX_REL = 511            # relative positions -511..511 cover every pair of a 512-token sequence


def t5_bucket_table(num_buckets: int, max_distance: int) -> torch.Tensor:
    """int32 [1023]: the bucket of relative position r = key - query at index r + 511.  HF T5Attention's
    `_relative_position_bucket` (bidirectional encoder), with its fp32 log expression evaluated once on the host so
    that the device never rounds a logarithm differently."""
    import math
    r = torch.arange(-T5_MAX_REL, T5_MAX_REL + 1, dtype=torch.long)
    nb = num_buckets // 2
    buckets = (r > 0).to(torch.long) * nb
    a = torch.abs(r)
    max_exact = nb // 2
    large = max_exact + (torch.log(a.float() / max_exact) / math.log(max_distance / max_exact)
                         * (nb - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, nb - 1))
    return (buckets + torch.where(a < max_exact, a, large)).to(torch.int32)


def t5_expected_keys(num_layers: int):
    """Every weight the T5 forward reads (HF T5EncoderModel names)."""
    keys = ["shared.weight", "encoder.final_layer_norm.weight",
            "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight"]
    for i in range(num_layers):
        p = f"encoder.block.{i}.layer."
        keys += [p + f"0.SelfAttention.{m}.weight" for m in "qkvo"]
        keys += [p + "0.layer_norm.weight", p + "1.DenseReluDense.wi.weight", p + "1.DenseReluDense.wo.weight",
                 p + "1.layer_norm.weight"]
    return keys


def _t5_config(config) -> dict:
    """The T5 geometry the kernels run (d_model 768, 12 heads of 64, ReLU feed-forward), or AttributeError."""
    get = (lambda k, d=None: config.get(k, d)) if isinstance(config, dict) else (lambda k, d=None: getattr(config, k, d))
    geom = dict(d_model=get("d_model", 768), num_heads=get("num_heads", 12), d_kv=get("d_kv", 64),
                feed_forward_proj=get("feed_forward_proj", "relu"))
    if geom != dict(d_model=768, num_heads=12, d_kv=64, feed_forward_proj="relu"):
        raise AttributeError(f"unsupported T5 geometry {geom}: only d_model 768, 12 heads of 64 and "
                             f"feed_forward_proj 'relu' (T5 v1.0, GTR-T5-base) run on the GPU path")
    return {k: get(k, T5_BASE[k]) for k in T5_BASE}


class B200T5Encoder(B200Contriever):
    """HF `T5EncoderModel` (fp16, d_model 768, 12 heads of 64, ReLU feed-forward) + mean / first-token pooling and the
    optional sentence-transformers Dense / Normalize head, on librsb (`rsb_t5_create`).  Same call surface as
    `B200Contriever`; `token_type_ids` are ignored.  The relative-position bucket table is uploaded at construction."""

    _ALIASES = {"encoder.embed_tokens.weight": "shared.weight"}     # tied embeddings: either name loads them

    def _create(self, config):
        self.config = dict(_t5_config(config or {}), hidden_size=768)     # hidden_size: the output width
        c = self.config
        rc = self.L.rsb_t5_create(c["num_layers"], c["d_ff"], c["vocab_size"], c["relative_attention_num_buckets"],
                                  c["relative_attention_max_distance"], ctypes.c_float(c["layer_norm_epsilon"]),
                                  ctypes.byref(self._h))
        self._check(rc)
        table = t5_bucket_table(c["relative_attention_num_buckets"], c["relative_attention_max_distance"]).to(self.device)
        rc = self.L.rsb_bert_load(self._h, b"relative_position_bucket", ctypes.c_void_p(table.data_ptr()), table.numel(),
                                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        self._check(rc)

    def expected_keys(self):
        return t5_expected_keys(self.config["num_layers"]) + (["dense.weight"] if self.dense else [])

    def require_all_weights(self, source: str = "state_dict"):
        missing = self.missing_keys()
        if missing:
            raise KeyError(f"{source}: {len(missing)} of {len(self.expected_keys())} T5 encoder weights were not found "
                           f"(first missing: {missing[:4]}); keys must follow HF T5EncoderModel naming")


def random_t5_state_dict(config=None, seed: int = 0, device="cpu", head: bool = True) -> Dict[str, torch.Tensor]:
    """Seeded random-init T5 encoder weights with HF T5EncoderModel names, plus the sentence-transformers Dense
    head (`dense.weight`, `dense.bias`) when `head` (benchmarks run without pretrained checkpoints)."""
    c = _t5_config(config or {})
    g = torch.Generator(device="cpu").manual_seed(seed)
    H, F = 768, c["d_ff"]

    def n(*shape, std):
        return (torch.randn(*shape, generator=g) * std).to(device)

    sd = {"shared.weight": n(c["vocab_size"], H, std=0.5),
          "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight":
              n(c["relative_attention_num_buckets"], 12, std=0.5)}
    for i in range(c["num_layers"]):
        p = f"encoder.block.{i}.layer."
        sd[p + "0.SelfAttention.q.weight"] = n(H, H, std=0.02)
        for m in "kvo":
            sd[p + f"0.SelfAttention.{m}.weight"] = n(H, H, std=0.04)
        sd[p + "0.layer_norm.weight"] = 1.0 + n(H, std=0.1)
        sd[p + "1.DenseReluDense.wi.weight"] = n(F, H, std=0.04)
        sd[p + "1.DenseReluDense.wo.weight"] = n(H, F, std=0.02)
        sd[p + "1.layer_norm.weight"] = 1.0 + n(H, std=0.1)
    sd["encoder.final_layer_norm.weight"] = 1.0 + n(H, std=0.1)
    if head:
        sd["dense.weight"] = n(H, H, std=0.04)
        sd["dense.bias"] = n(H, std=0.02)
    return sd


_ST_MODULE = "sentence_transformers.models."
_OTHER_FAMILIES = ("Qwen3", "drama", "ReasonIR", "GRIT")


def is_sentence_transformers_name(name: str) -> bool:
    """The reference's name dispatch (`src/search.py:49,244`, `src/embed.py:25,130`) for the family this project
    runs: "sentence-transformers" or "e5" in the name; Qwen3 and the other decoder-LLM embedders are not run here."""
    return ("sentence-transformers" in name or "e5" in name) and not any(t in name for t in _OTHER_FAMILIES)


class SentenceTransformerEncoder:
    """A sentence-transformers model (`SentenceTransformer(path)`, reference `src/search.py:244-246`) on the GPU:
    host tokenisation as its Transformer module does it (strip, optional lower-casing, truncation to
    `max_seq_length`), then one `rsb_bert_forward` that runs the transformer, the pooling and the head."""

    def __init__(self, model: B200Contriever, tokenizer, max_seq_length: int, do_lower_case: bool, path: str = ""):
        self.model, self.tokenizer = model, tokenizer
        self.max_seq_length, self.do_lower_case, self.path = int(max_seq_length), bool(do_lower_case), path

    @property
    def encode_group(self) -> int:
        return self.model.encode_group

    def eval(self):
        return self

    def half(self):
        return self

    def to(self, *a, **k):
        return self

    def encode_batch(self, texts) -> torch.Tensor:
        """list[str] -> fp16 [n, 768] on the device."""
        texts = [str(t).strip() for t in texts]
        if self.do_lower_case:
            texts = [t.lower() for t in texts]
        enc = self.tokenizer(texts, return_tensors="pt", max_length=self.max_seq_length, padding=True, truncation=True)
        return self.model(input_ids=enc["input_ids"], attention_mask=enc["attention_mask"],
                          token_type_ids=enc.get("token_type_ids"))


def _read_json(path: str) -> dict:
    import json
    with open(path) as f:
        return json.load(f)


def _read_weights(directory: str) -> Dict[str, torch.Tensor]:
    import os
    st = os.path.join(directory, "model.safetensors")
    if os.path.exists(st):
        from safetensors.torch import load_file
        return load_file(st)
    pt = os.path.join(directory, "pytorch_model.bin")
    if os.path.exists(pt):
        return torch.load(pt, map_location="cpu", weights_only=True)
    raise AttributeError(f"{directory}: neither model.safetensors nor pytorch_model.bin is present")


def _resolve_model_dir(path: str) -> str:
    import os
    if os.path.isdir(path):
        return path
    try:
        from huggingface_hub import snapshot_download
        return snapshot_download(path, local_files_only=True)
    except Exception as e:  # noqa: BLE001 -- any failure means the files are not available locally
        raise FileNotFoundError(f"{path}: not a local directory and not in the Hugging Face cache ({e})") from e


def read_sentence_transformer(path: str) -> dict:
    """Validates a sentence-transformers directory against what the GPU path runs and returns its description:
    {"dir", "arch" ("t5" | "bert"), "config", "max_seq_length", "do_lower_case", "pooling" ("average" | "cls"),
    "dense" (None or {"in_features", "out_features", "bias", "dir"}), "normalize"}.  Pure host code; anything it
    does not support raises AttributeError naming it."""
    import os
    root = _resolve_model_dir(path)
    mpath = os.path.join(root, "modules.json")
    if not os.path.exists(mpath):
        raise AttributeError(f"{path}: modules.json not found, not a sentence-transformers directory")
    mods = sorted(_read_json(mpath), key=lambda m: int(m.get("idx", 0)))
    kinds = [str(m.get("type", "")).replace(_ST_MODULE, "") for m in mods]
    if kinds[:2] != ["Transformer", "Pooling"] or kinds[2:] not in ([], ["Dense"], ["Normalize"], ["Dense", "Normalize"]):
        raise AttributeError(f"{path}: unsupported module stack {kinds}; supported: Transformer, Pooling, "
                             f"optionally Dense, optionally Normalize")
    mdir = [os.path.join(root, m.get("path", "")) for m in mods]
    # 1. Transformer
    sbc = os.path.join(mdir[0], "sentence_bert_config.json")
    st_cfg = _read_json(sbc) if os.path.exists(sbc) else {}
    max_len = int(st_cfg.get("max_seq_length") or 512)
    if max_len > 512:
        raise AttributeError(f"{path}: max_seq_length {max_len} > 512 is not supported")
    cfg = _read_json(os.path.join(mdir[0], "config.json"))
    arch = cfg.get("model_type")
    if arch == "t5":
        _t5_config(cfg)
    elif arch == "bert":
        geom = {k: cfg.get(k) for k in ("hidden_size", "num_attention_heads", "hidden_act")}
        if geom != dict(hidden_size=768, num_attention_heads=12, hidden_act="gelu") or int(cfg.get("intermediate_size", 0)) % 128:
            raise AttributeError(f"{path}: unsupported BERT geometry {geom}: only BERT-base (hidden 768, 12 heads, "
                                 f"GELU) runs on the GPU path")
    else:
        raise AttributeError(f"{path}: transformer model_type {arch!r} is not supported (T5 encoder or BERT-base only)")
    # 2. Pooling
    pc = _read_json(os.path.join(mdir[1], "config.json"))
    modes = sorted(k for k, v in pc.items() if k.startswith("pooling_mode_") and v)
    if modes == ["pooling_mode_mean_tokens"]:
        pooling = "average"
    elif modes == ["pooling_mode_cls_token"]:
        pooling = "cls"
    else:
        raise AttributeError(f"{path}: unsupported pooling modes {modes}; exactly one of pooling_mode_mean_tokens "
                             f"or pooling_mode_cls_token")
    if int(pc.get("word_embedding_dimension", 768)) != 768:
        raise AttributeError(f"{path}: pooling dimension {pc.get('word_embedding_dimension')} is not 768")
    # 3. Dense
    dense = None
    if "Dense" in kinds:
        i = kinds.index("Dense")
        dc = _read_json(os.path.join(mdir[i], "config.json"))
        act = str(dc.get("activation_function", "torch.nn.modules.linear.Identity"))
        if (int(dc.get("in_features", 0)), int(dc.get("out_features", 0))) != (768, 768):
            raise AttributeError(f"{path}: Dense {dc.get('in_features')} -> {dc.get('out_features')} is not supported "
                                 f"(768 -> 768 only)")
        if not act.endswith("Identity"):
            raise AttributeError(f"{path}: Dense activation {act} is not supported (Identity only)")
        dense = dict(in_features=768, out_features=768, bias=bool(dc.get("bias", True)), dir=mdir[i])
    return dict(dir=mdir[0], arch=arch, config=cfg, max_seq_length=max_len,
                do_lower_case=bool(st_cfg.get("do_lower_case", False)), pooling=pooling, dense=dense,
                normalize="Normalize" in kinds)


def load_sentence_transformer(path: str, device=None) -> SentenceTransformerEncoder:
    """`SentenceTransformer(path)` for the supported stacks (see `read_sentence_transformer`): weights and tokenizer
    from the local directory or the Hugging Face cache (no download)."""
    import transformers
    d = read_sentence_transformer(path)
    sd = _read_weights(d["dir"])
    if d["dense"] is not None:
        hw = _read_weights(d["dense"]["dir"])
        sd["dense.weight"] = hw["linear.weight"]
        if d["dense"]["bias"]:
            sd["dense.bias"] = hw["linear.bias"]
    cls = B200T5Encoder if d["arch"] == "t5" else B200Contriever
    if d["arch"] == "bert":
        sd = strip_wrapper_prefix(sd)
    else:
        sd = {k: v for k, v in sd.items() if not k.startswith("decoder.") and not k.startswith("lm_head.")}
    model = cls(d["config"], d["pooling"], device=device, dense=d["dense"] is not None, normalize=d["normalize"])
    model.load_state_dict(sd, strict=False)
    model.require_all_weights(path)
    tokenizer = transformers.AutoTokenizer.from_pretrained(d["dir"], local_files_only=True)
    return SentenceTransformerEncoder(model, tokenizer, d["max_seq_length"], d["do_lower_case"], path)
