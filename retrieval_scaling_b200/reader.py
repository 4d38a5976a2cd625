"""GPU reader LM for perplexity evaluation in fp16 (the default) or bf16 on librsb: HF `LlamaForCausalLM` (Llama-2 MHA, Llama-3 GQA),
HF `GPTNeoXForCausalLM` (the Pythia suite, whose pythia-1b is the reference's default `model.lm_model`) and HF
`OlmoForCausalLM` / `Olmo2ForCausalLM` (OLMo, OLMo-1.7 and OLMo-2).

The reference loads its reader with `AutoModelForCausalLM.from_pretrained(cfg.model.lm_model, torch_dtype=bfloat16)`
and calls `lm(input_ids, labels=labels)` one window at a time (`src/evaluate_perplexity.py:98-134`).  Here

    model = load_reader(path)                                   # local directory or HF cache, no download
    model = load_reader(path, dtype=torch.bfloat16)             # the reference's reader dtype
    nll = model.nll([ids_0, ids_1, ...], [labels_0, ...])       # per-token NLL, many windows per forward
    losses = model.loss([ids_0, ...], [labels_0, ...])          # HF's per-window mean loss
    new_ids = model.generate([prompt_0, ...], 256, eos_ids)      # greedy decoding with a KV cache (rsb_llm_generate)
    ll = model.loglikelihood([(ctx_0, cont_0), ...], 2048)      # (log p(cont | ctx), is_greedy) (rsb_llm_loglikelihood)

runs `rsb_llm_nll`: a prefill-only forward over packed, un-padded windows whose LM head runs only on the rows whose
next token is a label.  `load_reader` picks `B200Llama`, `B200NeoX` or `B200Olmo` from the config's `model_type`.  No CPU /
eager-PyTorch fallback: constructing the model without CUDA raises.  A checkpoint the kernels do not run (another
`model_type`, another head_dim, RoPE scaling, a sequential residual, ...) raises AttributeError naming the field before
any weight is read or device memory is allocated.
"""
from __future__ import annotations

import ctypes
import json
import math
import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib

IGNORE = -100


def _get(cfg, key, default=None):
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


def _refuse(msg):
    raise AttributeError(msg)


def _rope_parameters(cfg, refuse, **fields):
    """`fields` (rope_parameters key -> value read outside it) as the config gives them: transformers >= 5 folds them
    and rope_scaling into rope_parameters.  Anything but the default RoPE is refused."""
    rp = _get(cfg, "rope_parameters")
    if isinstance(rp, dict):
        if rp.get("rope_type", "default") != "default":
            refuse(f"rope_parameters {rp}: only the default RoPE is implemented (rope_scaling null)")
        fields = {k: rp.get(k, v) for k, v in fields.items()}
    if _get(cfg, "rope_scaling") is not None and not (isinstance(rp, dict) and _get(cfg, "rope_scaling") == rp):
        refuse(f"rope_scaling {_get(cfg, 'rope_scaling')}: only rope_scaling null is implemented")
    return fields


def _positive_sizes(cfg, refuse, *keys):
    """The values of `keys`, each refused unless a positive size."""
    for key in keys:
        if not _get(cfg, key) or _get(cfg, key) <= 0:
            refuse(f"{key} {_get(cfg, key)} is not a positive size")
    return [_get(cfg, key) for key in keys]


def llama_geometry(cfg) -> dict:
    """The reader geometry the kernels run, from an HF config (dict or object), or AttributeError naming the field."""
    mt = _get(cfg, "model_type")
    if mt != "llama":
        why = (" (GPT-NeoX / Pythia needs head_dim-256 attention, partial rotary and a parallel residual)"
               if mt == "gpt_neox" else "")
        raise AttributeError(f"model_type {mt!r}: only 'llama' readers run on the GPU path{why}")
    hidden, heads = _get(cfg, "hidden_size"), _get(cfg, "num_attention_heads")
    kv = _get(cfg, "num_key_value_heads") or heads
    head_dim = _get(cfg, "head_dim") or (hidden // heads if hidden and heads else None)
    if head_dim != 128 or hidden != heads * 128:
        raise AttributeError(f"head_dim {head_dim} (hidden_size {hidden}, num_attention_heads {heads}): only head_dim "
                             f"128 with hidden_size = 128 x num_attention_heads is implemented")
    if heads % kv:
        raise AttributeError(f"num_key_value_heads {kv} does not divide num_attention_heads {heads}")
    if _get(cfg, "hidden_act", "silu") != "silu":
        raise AttributeError(f"hidden_act {_get(cfg, 'hidden_act')!r}: only 'silu' is implemented")
    inter = _get(cfg, "intermediate_size")
    if hidden % 128 or not inter or inter % 128:
        raise AttributeError(f"hidden_size {hidden} / intermediate_size {inter}: both must be multiples of 128")
    for key in ("attention_bias", "mlp_bias"):
        if _get(cfg, key, False):
            raise AttributeError(f"{key} is set: only bias-free Llama layers are implemented")
    theta = _rope_parameters(cfg, _refuse, rope_theta=_get(cfg, "rope_theta"))["rope_theta"]
    vocab, = _positive_sizes(cfg, _refuse, "vocab_size")
    return dict(num_hidden_layers=_get(cfg, "num_hidden_layers"), hidden_size=hidden, num_attention_heads=heads,
                num_key_value_heads=kv, intermediate_size=inter, vocab_size=vocab,
                max_position_embeddings=_get(cfg, "max_position_embeddings", 2048),
                rope_theta=float(theta if theta is not None else 10000.0),
                rms_norm_eps=float(_get(cfg, "rms_norm_eps", 1e-6)),
                tie_word_embeddings=bool(_get(cfg, "tie_word_embeddings", False)))


NEOX_HEAD_DIMS = (64, 80, 128, 256)
NEOX_MAX_HIDDEN = 8192                           # ln_rows_kernel's widest row


def neox_geometry(cfg) -> dict:
    """The GPT-NeoX reader geometry the kernels run, from an HF config in the Hub's form (`rotary_pct`,
    `rotary_emb_base`) or transformers 5's (`rope_parameters`), or AttributeError naming the field."""
    mt = _get(cfg, "model_type")

    def refuse(msg):
        raise AttributeError(f"model_type {mt!r}: {msg}")
    if mt != "gpt_neox":
        refuse("only 'gpt_neox' readers run on this path")
    act = _get(cfg, "hidden_act", "gelu")
    if act != "gelu":
        refuse(f"hidden_act {act!r}: only the exact-erf 'gelu' is implemented")
    hidden, heads = _get(cfg, "hidden_size"), _get(cfg, "num_attention_heads")
    if not hidden or not heads or hidden <= 0 or heads <= 0 or hidden % heads:
        refuse(f"hidden_size {hidden} is not a multiple of num_attention_heads {heads}")
    head_dim = hidden // heads
    if head_dim not in NEOX_HEAD_DIMS:
        refuse(f"head_dim {head_dim} (hidden_size {hidden} / num_attention_heads {heads}): only head_dim "
               f"{', '.join(map(str, NEOX_HEAD_DIMS))} is implemented")
    if hidden > NEOX_MAX_HIDDEN:
        refuse(f"hidden_size {hidden}: the LayerNorm kernel holds rows of at most {NEOX_MAX_HIDDEN} (Pythia-12B: 5120)")
    inter = _get(cfg, "intermediate_size")
    if hidden % 128 or not inter or inter % 128:
        refuse(f"hidden_size {hidden} / intermediate_size {inter}: both must be multiples of 128")
    rope = _rope_parameters(cfg, refuse, partial_rotary_factor=_get(cfg, "rotary_pct", 0.25),
                            rope_theta=_get(cfg, "rotary_emb_base", 10000.0))
    pct, base = rope["partial_rotary_factor"], rope["rope_theta"]
    rot = int(head_dim * pct)
    if rot <= 0 or rot % 2 or rot > head_dim:
        refuse(f"rotary_ndims {rot} (rotary_pct {pct} x head_dim {head_dim}) must be even and in [2, head_dim]")
    if not (base and base > 0):
        refuse(f"rotary_emb_base {base} is not positive")
    for key, want in (("use_parallel_residual", True), ("attention_bias", True), ("tie_word_embeddings", False)):
        if bool(_get(cfg, key, want)) != want:
            refuse(f"{key} {_get(cfg, key)}: only {key} {want} (every Pythia model) is implemented")
    vocab, layers = _positive_sizes(cfg, refuse, "vocab_size", "num_hidden_layers")
    return dict(num_hidden_layers=layers, hidden_size=hidden, num_attention_heads=heads, head_dim=head_dim,
                intermediate_size=inter, vocab_size=vocab, max_position_embeddings=_get(cfg, "max_position_embeddings", 2048),
                rotary_ndims=rot, rotary_emb_base=float(base), layer_norm_eps=float(_get(cfg, "layer_norm_eps", 1e-5)))


def neox_expected_keys(geom: dict) -> List[str]:
    """Every weight the GPT-NeoX forward reads (HF GPTNeoXForCausalLM names)."""
    keys = ["gpt_neox.embed_in.weight", "gpt_neox.final_layer_norm.weight", "gpt_neox.final_layer_norm.bias",
            "embed_out.weight"]
    for i in range(geom["num_hidden_layers"]):
        keys += [f"gpt_neox.layers.{i}.{n}.{p}" for n in (
            "input_layernorm", "post_attention_layernorm", "attention.query_key_value", "attention.dense",
            "mlp.dense_h_to_4h", "mlp.dense_4h_to_h") for p in ("weight", "bias")]
    return keys


OLMO_MAX_HIDDEN = 8192                           # OLMo's LayerNorm runs on ln_rows_kernel


def olmo_geometry(cfg) -> dict:
    """The OLMo (`model_type` 'olmo', version 1) or OLMo-2 ('olmo2', version 2) reader geometry the kernels run, from an
    HF config in either the `rope_theta` or transformers 5's `rope_parameters` form, or AttributeError naming the
    field.  The non-HF 'hf_olmo' repos and 'olmo3' are other model_types and are refused by `load_reader`."""
    mt = _get(cfg, "model_type")

    def refuse(msg):
        raise AttributeError(f"model_type {mt!r}: {msg}")
    if mt not in ("olmo", "olmo2"):
        refuse("only 'olmo' and 'olmo2' readers run on this path")
    act = _get(cfg, "hidden_act", "silu")
    if act != "silu":
        refuse(f"hidden_act {act!r}: only 'silu' is implemented")
    if _get(cfg, "attention_bias", False):
        refuse("attention_bias is set: only bias-free attention is implemented")
    hidden, heads = _get(cfg, "hidden_size"), _get(cfg, "num_attention_heads")
    kv = _get(cfg, "num_key_value_heads") or heads
    head_dim = _get(cfg, "head_dim") or (hidden // heads if hidden and heads else None)
    if head_dim != 128 or not heads or hidden != heads * 128:
        refuse(f"head_dim {head_dim} (hidden_size {hidden}, num_attention_heads {heads}): only head_dim 128 with "
               f"hidden_size = 128 x num_attention_heads is implemented")
    if kv <= 0 or heads % kv:
        refuse(f"num_key_value_heads {kv} does not divide num_attention_heads {heads}")
    inter = _get(cfg, "intermediate_size")
    if not inter or inter <= 0 or inter % 128:
        refuse(f"intermediate_size {inter}: must be a positive multiple of 128 (hidden_size {hidden} is)")
    if mt == "olmo" and hidden > OLMO_MAX_HIDDEN:
        refuse(f"hidden_size {hidden}: the LayerNorm kernel holds rows of at most {OLMO_MAX_HIDDEN}")
    theta = _rope_parameters(cfg, refuse, rope_theta=_get(cfg, "rope_theta"))["rope_theta"]
    theta = float(theta if theta is not None else 10000.0)
    if not theta > 0:
        refuse(f"rope_theta {theta} is not positive")
    clip = _get(cfg, "clip_qkv") if mt == "olmo" else None   # Olmo2ForCausalLM never reads clip_qkv
    if clip is not None and not clip > 0:
        refuse(f"clip_qkv {clip}: must be null or positive")
    vocab, layers = _positive_sizes(cfg, refuse, "vocab_size", "num_hidden_layers")
    # OlmoLayerNorm's eps is 1e-5 in the model code; OLMo-2 reads rms_norm_eps
    eps = 1e-5 if mt == "olmo" else float(_get(cfg, "rms_norm_eps", 1e-5))
    return dict(version=1 if mt == "olmo" else 2, num_hidden_layers=layers, hidden_size=hidden,
                num_attention_heads=heads, num_key_value_heads=kv, intermediate_size=inter, vocab_size=vocab,
                max_position_embeddings=_get(cfg, "max_position_embeddings", 2048), rope_theta=theta, eps=eps,
                clip_qkv=float(clip or 0.0), tie_word_embeddings=bool(_get(cfg, "tie_word_embeddings", False)))


def olmo_expected_keys(geom: dict) -> List[str]:
    """Every weight the OLMo / OLMo-2 forward reads (HF OlmoForCausalLM / Olmo2ForCausalLM names); OLMo has no norm
    weights."""
    v2 = geom["version"] == 2
    keys = ["model.embed_tokens.weight"] + (["model.norm.weight"] if v2 else [])
    if not geom["tie_word_embeddings"]:
        keys.append("lm_head.weight")
    names = ["self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj", "mlp.gate_proj",
             "mlp.up_proj", "mlp.down_proj"]
    if v2:
        names += ["self_attn.q_norm", "self_attn.k_norm", "post_attention_layernorm", "post_feedforward_layernorm"]
    for i in range(geom["num_hidden_layers"]):
        keys += [f"model.layers.{i}.{n}.weight" for n in names]
    return keys


def expected_keys(geom: dict) -> List[str]:
    """Every weight the forward reads (HF LlamaForCausalLM names)."""
    keys = ["model.embed_tokens.weight", "model.norm.weight"]
    if not geom["tie_word_embeddings"]:
        keys.append("lm_head.weight")
    for i in range(geom["num_hidden_layers"]):
        keys += [f"model.layers.{i}.{n}.weight" for n in (
            "self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj", "mlp.gate_proj",
            "mlp.up_proj", "mlp.down_proj", "input_layernorm", "post_attention_layernorm")]
    return keys


READER_DTYPES = {torch.float16: "float16", torch.bfloat16: "bfloat16"}


def reader_dtype(dtype) -> torch.dtype:
    """torch.float16 or torch.bfloat16 from either torch dtype or its name ('float16', 'bfloat16'); ValueError
    otherwise."""
    for t, name in READER_DTYPES.items():
        if (isinstance(dtype, torch.dtype) and dtype == t) or (isinstance(dtype, str) and dtype == name):
            return t
    raise ValueError(f"reader dtype {dtype!r}: only torch.float16 / 'float16' and torch.bfloat16 / 'bfloat16' are "
                     f"implemented")


def scored_positions(labels: Sequence[int]) -> List[int]:
    """Positions whose label enters HF's shifted loss: every position after the first whose label is not -100."""
    return [t for t in range(1, len(labels)) if labels[t] != IGNORE]


class _Reader:
    """A causal-LM reader on librsb (`rsb_llm_*`): everything but the geometry and the constructor's arguments."""

    # tokens per forward that `nll` packs: the GEMMs fill the GPU well before this, and the activations of a
    # Llama-3-8B forward stay near 3 GB
    token_budget = 16384
    # non-weight buffers of HF checkpoints, skipped by name before any conversion
    _buffers = ("rotary_emb.inv_freq",)

    def __init__(self, config, device=None, dtype=torch.float16):
        self.dtype = reader_dtype(dtype)
        self.geom = self._geometry(config)
        if not torch.cuda.is_available():
            raise RuntimeError(f"{type(self).__name__} needs a CUDA device (sm_90a): there is no CPU path")
        self.L = _lib.lib()
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self._h = ctypes.c_void_p(0)
        self._ws: Optional[torch.Tensor] = None
        self.loaded = set()
        with torch.cuda.device(self.device):
            self._check(self._create(self.geom))

    def _create(self, g):
        dtype = _lib.RSB_DTYPE_BF16 if self.dtype == torch.bfloat16 else _lib.RSB_DTYPE_F16
        return self.L.rsb_llm_create(self.family, dtype, *self._create_args(g), ctypes.byref(self._h))

    def _check(self, rc):
        if rc == _lib.RSB_OK:
            return
        msg = self.L.rsb_llm_last_error().decode("utf-8", "replace")
        if rc == _lib.RSB_ERR_INVALID:
            raise ValueError(msg)
        if rc == _lib.RSB_ERR_UNSUPPORTED:
            raise NotImplementedError(msg)
        if rc == _lib.RSB_ERR_OOM:
            raise MemoryError(msg)
        raise _lib.RsbError(f"librsb reader error {rc}: {msg}")

    def __del__(self):
        try:
            if getattr(self, "_h", None) and self._h.value:
                self.L.rsb_llm_free(self._h)
                self._h = ctypes.c_void_p(0)
        except Exception:
            pass

    @property
    def max_position_embeddings(self) -> int:
        return self.geom["max_position_embeddings"]

    def load_weight(self, name: str, t: torch.Tensor) -> bool:
        """Uploads one HF weight in the reader's dtype (round to nearest even, as `from_pretrained(torch_dtype=...)`
        converts); False for a name the reader does not use.  A weight that does not stay finite in that dtype (in
        fp16, a bf16 value beyond 65504) is refused."""
        if name.endswith(self._buffers):
            return False
        w = t.detach().to(device=self.device, dtype=self.dtype).contiguous()
        if not bool(torch.isfinite(w).all()):
            raise ValueError(f"weight {name} does not stay finite in {READER_DTYPES[self.dtype]}")
        stream = ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        rc = self.L.rsb_llm_load(self._h, name.encode(), ctypes.c_void_p(w.data_ptr()), w.numel(), stream)
        if rc == _lib.RSB_ERR_INVALID and b"unknown weight" in self.L.rsb_llm_last_error():
            return False
        self._check(rc)
        torch.cuda.current_stream(self.device).synchronize()
        self.loaded.add(name)
        return True

    def load_state_dict(self, sd: Dict[str, torch.Tensor], strict: bool = True):
        with torch.cuda.device(self.device):
            unexpected = [n for n, t in sd.items() if not self.load_weight(n, t) and not n.endswith(self._buffers)]
        if strict and unexpected:
            raise KeyError(f"unexpected keys in state_dict: {unexpected[:5]}")
        if strict:
            self.require_all_weights()
        return unexpected

    def missing_keys(self):
        return [k for k in self._expected_keys(self.geom) if k not in self.loaded]

    def require_all_weights(self, source: str = "state_dict"):
        missing = self.missing_keys()
        if missing:
            raise KeyError(f"{source} lacks {len(missing)} reader weights, e.g. {missing[:3]}")

    # -- forward ------------------------------------------------------------------------------------------------
    def _nll_packed(self, ids: Sequence[Sequence[int]], labels: Sequence[Sequence[int]]) -> List[torch.Tensor]:
        lens = [len(x) for x in ids]
        T = sum(lens)
        n_label = sum(len(scored_positions(lb)) for lb in labels)
        cu = [0]
        for n in lens:
            cu.append(cu[-1] + n)
        dev = self.device
        flat_ids = torch.tensor([v for x in ids for v in x], dtype=torch.int32, device=dev)
        flat_lab = torch.tensor([v for x in labels for v in x], dtype=torch.int32, device=dev)
        cu_t = torch.tensor(cu, dtype=torch.int32, device=dev)
        out = torch.empty(T, dtype=torch.float32, device=dev)
        need = self.L.rsb_llm_workspace_bytes(self._h, T, n_label)
        if self._ws is None or self._ws.numel() < need:
            self._ws = None
            self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            rc = self.L.rsb_llm_nll(self._h, ctypes.c_void_p(flat_ids.data_ptr()), ctypes.c_void_p(cu_t.data_ptr()),
                                    len(lens), T, max(lens), ctypes.c_void_p(flat_lab.data_ptr()),
                                    ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(self._ws.data_ptr()),
                                    self._ws.numel(), ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
        self._check(rc)
        host = out.cpu()
        if not bool(torch.isfinite(host).all()):
            raise self._overflow("per-token NLL")
        return [host[cu[i]:cu[i + 1]].clone() for i in range(len(lens))]

    def _overflow(self, what: str) -> FloatingPointError:
        if self.dtype == torch.float16:
            return FloatingPointError(f"non-finite {what}: the fp16 activations overflowed (|x| > 65504); this "
                                      f"checkpoint needs a bf16 reader (load_reader(..., dtype=torch.bfloat16), "
                                      f"model.lm_dtype=bfloat16)")
        return FloatingPointError(f"non-finite {what}: the bf16 activations overflowed (|x| > 3.39e38) or the "
                                  f"checkpoint's weights produce NaN")

    def nll(self, input_ids_list, labels_list, max_tokens: Optional[int] = None) -> List[torch.Tensor]:
        """Per-token NLL of each window, fp32 [len(ids)] on the host: position t holds -log p(labels[t] | ids[:t])
        where t > 0 and labels[t] != -100, 0 elsewhere.  Consecutive windows are packed into one forward up to
        `max_tokens` (default `token_budget`); the kernels treat every window on its own, so the values are the
        same as one call per window."""
        ids = [[int(v) for v in x] for x in input_ids_list]
        labels = [[int(v) for v in x] for x in labels_list]
        if len(ids) != len(labels) or any(len(a) != len(b) for a, b in zip(ids, labels)):
            raise ValueError("every window needs one label per token")
        if any(len(x) == 0 for x in ids):
            raise ValueError("empty window")
        budget = self.token_budget if max_tokens is None else int(max_tokens)
        out: List[torch.Tensor] = []
        i = 0
        while i < len(ids):
            j, tokens = i, 0
            while j < len(ids) and (j == i or tokens + len(ids[j]) <= budget):
                tokens += len(ids[j])
                j += 1
            out += self._nll_packed(ids[i:j], labels[i:j])
            i = j
        return out

    # -- multiple-choice scoring (rsb_llm_loglikelihood) ----------------------------------------------------------
    def _loglikelihood_packed(self, windows: Sequence[Sequence[int]], targets: Sequence[Sequence[Tuple[int, int]]]):
        """fp32 log-probabilities and greedy flags (numpy, in target order) of the (row within its window, token)
        targets of each window, one forward over the packed windows."""
        lens = [len(w) for w in windows]
        cu = [0] + np.cumsum(lens).tolist()
        T = cu[-1]
        rows = [cu[b] + r for b, ts in enumerate(targets) for r, _ in ts]
        toks = [t for ts in targets for _, t in ts]
        n = len(rows)
        dev = self.device
        i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=dev)   # noqa: E731
        flat_ids, cu_t, d_row, d_tok = i32([v for w in windows for v in w]), i32(cu), i32(rows), i32(toks)
        lp = torch.empty(n, dtype=torch.float32, device=dev)
        greedy = torch.empty(n, dtype=torch.int32, device=dev)
        need = self.L.rsb_llm_loglikelihood_workspace_bytes(self._h, T, n)
        if self._ws is None or self._ws.numel() < need:
            self._ws = None
            self._ws = torch.empty(need, dtype=torch.uint8, device=dev)
        p = lambda t: ctypes.c_void_p(t.data_ptr())   # noqa: E731
        with torch.cuda.device(dev):
            rc = self.L.rsb_llm_loglikelihood(self._h, p(flat_ids), p(cu_t), len(lens), T, max(lens), p(d_row), p(d_tok),
                                              n, p(lp), p(greedy), p(self._ws), self._ws.numel(),
                                              ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
        self._check(rc)
        lp, greedy = lp.cpu().numpy(), greedy.cpu().numpy()
        if not np.isfinite(lp).all():
            raise self._overflow("log-likelihood")
        return lp, greedy

    def loglikelihood(self, requests, max_length: int, max_tokens: Optional[int] = None) -> List[Tuple[float, bool]]:
        """(log p(continuation | context), is_greedy) per (context_ids, continuation_ids) request, in input order: the
        lm-eval fork's HFLM._loglikelihood_tokens (lm_eval/models/huggingface.py:948-1162) for a causal LM.

        The input window is (context + continuation)[-(max_length + 1):][:-1], and the continuation is scored on its
        last len(continuation) rows (:1030-1046); the log-likelihood is the fp64 sum of the tokens' fp32 log-softmax
        (:1106, :1147-1153), and is_greedy holds when every continuation token is its row's argmax (:1128, :1144).
        Requests with identical windows share one forward, as the fork's group_by="contexts" cache shares the logits of
        one-token continuations (:968-984), so an MMLU question costs one window for its four choices.  Windows run
        longest first (:957-967), packed up to `max_tokens` (default `token_budget`) per forward.  An empty context or
        continuation, or a continuation longer than max_length, raises ValueError; non-finite values raise
        FloatingPointError."""
        max_length = int(max_length)
        windows: Dict[tuple, int] = {}
        scored = []                              # per request: (window, first scored row, continuation)
        for ctx, cont in requests:
            ctx, cont = [int(v) for v in ctx], [int(v) for v in cont]
            if not ctx:
                raise ValueError("empty context: the harness scores an empty context after its prefix token (BOS, "
                                 "else EOS)")
            if not cont:
                raise ValueError("empty continuation")
            if len(cont) > max_length:
                raise ValueError(f"a continuation of {len(cont)} tokens is longer than max_length {max_length}")
            inp = tuple((ctx + cont)[-(max_length + 1):][:-1])
            w = windows.setdefault(inp, len(windows))
            scored.append((w, len(inp) - len(cont), cont))
        wins = list(windows)
        targets: List[List[Tuple[int, int]]] = [[] for _ in wins]
        first: List[Tuple[int, int]] = []        # per request: (window, index of its first target in the window)
        for w, r0, cont in scored:
            first.append((w, len(targets[w])))
            targets[w] += [(r0 + j, t) for j, t in enumerate(cont)]
        order = sorted(range(len(wins)), key=lambda w: -len(wins[w]))
        budget = self.token_budget if max_tokens is None else int(max_tokens)
        lp: List = [None] * len(wins)
        greedy: List = [None] * len(wins)
        i = 0
        while i < len(order):
            j, tokens = i, 0
            while j < len(order) and (j == i or tokens + len(wins[order[j]]) <= budget):
                tokens += len(wins[order[j]])
                j += 1
            batch = order[i:j]
            l_all, g_all = self._loglikelihood_packed([wins[w] for w in batch], [targets[w] for w in batch])
            k = 0
            for w in batch:
                lp[w], greedy[w] = l_all[k:k + len(targets[w])], g_all[k:k + len(targets[w])]
                k += len(targets[w])
            i = j
        res = []
        for (w, t0), (_, _, cont) in zip(first, scored):
            sl = slice(t0, t0 + len(cont))
            res.append((float(lp[w][sl].astype(np.float64).sum()), bool(greedy[w][sl].all())))
        return res

    # -- greedy generation (rsb_llm_generate) ---------------------------------------------------------------------
    # share of the free device memory one generate call's workspace (KV cache, activations, partials) may take
    generate_memory_share = 0.8

    def _generate_batch(self, prompts, max_new: int, eos: List[int]):
        lens = [len(p) for p in prompts]
        B, T = len(prompts), sum(lens)
        dev = self.device
        ids = torch.tensor([v for p in prompts for v in p], dtype=torch.int32, device=dev)
        cu = torch.tensor([0] + list(np.cumsum(lens)), dtype=torch.int32, device=dev)
        toks = torch.empty((B, max_new), dtype=torch.int32, device=dev)
        out_lens = torch.empty(B, dtype=torch.int32, device=dev)
        lp = torch.empty((B, max_new), dtype=torch.float32, device=dev)
        ws = torch.empty(self.L.rsb_llm_generate_workspace_bytes(self._h, B, T, max(lens), max_new), dtype=torch.uint8,
                         device=dev)
        eos_arr = (ctypes.c_int32 * max(len(eos), 1))(*eos)
        with torch.cuda.device(dev):
            rc = self.L.rsb_llm_generate(self._h, ctypes.c_void_p(ids.data_ptr()), ctypes.c_void_p(cu.data_ptr()), B, T,
                                         max(lens), max_new, eos_arr, len(eos), ctypes.c_void_p(toks.data_ptr()),
                                         ctypes.c_void_p(out_lens.data_ptr()), ctypes.c_void_p(lp.data_ptr()),
                                         ctypes.c_void_p(ws.data_ptr()), ws.numel(),
                                         ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
        self._check(rc)
        n = out_lens.cpu().tolist()
        toks, lp = toks.cpu(), lp.cpu()
        out = [(toks[b, :n[b]].tolist(), lp[b, :n[b]].clone()) for b in range(B)]
        if not all(bool(torch.isfinite(x).all()) for _, x in out):
            raise FloatingPointError(f"non-finite logits while generating: the {READER_DTYPES[self.dtype]} activations "
                                     f"overflowed or the checkpoint's weights produce NaN"
                                     + (" (a bf16 reader may evaluate it)" if self.dtype == torch.float16 else ""))
        return out

    def generate(self, prompt_ids, max_new_tokens: int, eos_token_ids=(), return_logprobs: bool = False):
        """Greedy continuation of every prompt (HF `generate(do_sample=False)` with `eos_token_id=eos_token_ids`): per
        prompt, in input order, the new ids, ending after the first id of `eos_token_ids` (included) or after
        `max_new_tokens` ids.  With return_logprobs, also each id's fp32 log-softmax (a float32 tensor per prompt).
        Prompts run longest first, as many per call as the workspace (KV cache included) fits in
        `generate_memory_share` of the free device memory; a prompt's ids do not depend on the others.  Raises
        FloatingPointError on non-finite logits; a prompt plus max_new_tokens past max_position_embeddings raises
        NotImplementedError."""
        prompts = [[int(v) for v in p] for p in prompt_ids]
        max_new = int(max_new_tokens)
        if max_new <= 0:
            raise ValueError(f"max_new_tokens {max_new_tokens} must be positive")
        if any(len(p) == 0 for p in prompts):
            raise ValueError("empty prompt")
        eos = [int(eos_token_ids)] if isinstance(eos_token_ids, int) else [int(e) for e in (eos_token_ids or ())]
        order = sorted(range(len(prompts)), key=lambda i: -len(prompts[i]))
        with torch.cuda.device(self.device):
            free = torch.cuda.mem_get_info(self.device)[0] + torch.cuda.memory_reserved(self.device) \
                - torch.cuda.memory_allocated(self.device)
        budget = self.generate_memory_share * free
        res: List = [None] * len(prompts)
        i = 0
        while i < len(order):
            j, T = i + 1, len(prompts[order[i]])
            longest = T
            while j < len(order) and self.L.rsb_llm_generate_workspace_bytes(
                    self._h, j + 1 - i, T + len(prompts[order[j]]), longest, max_new) <= budget:
                T += len(prompts[order[j]])
                j += 1
            for k, r in zip(order[i:j], self._generate_batch([prompts[k] for k in order[i:j]], max_new, eos)):
                res[k] = r
            i = j
        if return_logprobs:
            return [r[0] for r in res], [r[1] for r in res]
        return [r[0] for r in res]

    # -- diagnostics (rsb_llm_attention / rsb_llm_hidden_states), not used by nll / loss ----------------------------
    def attention(self, qkv: torch.Tensor, cu_seqlens: torch.Tensor, max_seqlen: int, ctx: torch.Tensor):
        """One attention step of the forward: RoPE in place on the Q / K heads of qkv [T, (heads + 2 kv_heads)
        head_dim] in the reader's dtype (GPT-NeoX: [Q heads | K heads | V heads], only the first rotary_ndims of each
        head rotated), then causal attention into ctx [T, hidden] of the same dtype for the windows of cu_seqlens
        (int32 [B + 1], empty windows allowed, may end below T).  Rows outside the windows are left as they are."""
        for what, t in (("qkv", qkv), ("ctx", ctx)):
            if t.dtype != self.dtype:
                raise ValueError(f"{what} is {t.dtype}; this reader runs in {self.dtype}")
        with torch.cuda.device(self.device):
            rc = self.L.rsb_llm_attention(self._h, ctypes.c_void_p(qkv.data_ptr()), ctypes.c_void_p(cu_seqlens.data_ptr()),
                                          cu_seqlens.numel() - 1, qkv.shape[0], int(max_seqlen),
                                          ctypes.c_void_p(ctx.data_ptr()),
                                          ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream))
        self._check(rc)

    def decode_attention(self, qkv: torch.Tensor, slot: torch.Tensor, pos: torch.Tensor, k_cache: torch.Tensor,
                         v_cache: torch.Tensor, ctx: torch.Tensor):
        """One decode step of generate's attention: row i of qkv [n, (heads + 2 kv_heads) head_dim] is rotated in place
        at position pos[i] (int32 [n] on the device), its K and V are stored in k_cache / v_cache [slots, kv_heads, cap,
        head_dim] at (slot[i], :, pos[i]), and ctx [n, hidden] receives its attention over positions 0 .. pos[i] of the
        slot.  Every tensor in the reader's dtype but slot / pos."""
        for what, t in (("qkv", qkv), ("k_cache", k_cache), ("v_cache", v_cache), ("ctx", ctx)):
            if t.dtype != self.dtype:
                raise ValueError(f"{what} is {t.dtype}; this reader runs in {self.dtype}")
        g = self.geom
        H, heads = g["hidden_size"], g["num_attention_heads"]
        kv, d = g.get("num_key_value_heads", heads), H // heads
        n = qkv.shape[0]
        shapes = {"qkv": (qkv, (n, (heads + 2 * kv) * d)), "ctx": (ctx, (n, H)), "slot": (slot, (n,)), "pos": (pos, (n,)),
                  "v_cache": (v_cache, tuple(k_cache.shape))}
        if k_cache.dim() != 4 or tuple(k_cache.shape[1::2]) != (kv, d):
            raise ValueError(f"k_cache is {tuple(k_cache.shape)}, not [slots, {kv}, cap, {d}]")
        for what, (t, want) in shapes.items():
            if tuple(t.shape) != want or not t.is_contiguous():
                raise ValueError(f"{what} is {tuple(t.shape)}, not a contiguous {want}")
        if slot.dtype != torch.int32 or pos.dtype != torch.int32:
            raise ValueError("slot and pos must be int32")
        p = lambda t: ctypes.c_void_p(t.data_ptr())   # noqa: E731
        with torch.cuda.device(self.device):
            rc = self.L.rsb_llm_decode_attention(self._h, p(qkv), p(slot), p(pos), qkv.shape[0], p(k_cache), p(v_cache),
                                                 k_cache.shape[0], k_cache.shape[2], p(ctx),
                                                 ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream))
        self._check(rc)

    def hidden_states(self, ids: torch.Tensor, cu_seqlens: torch.Tensor, max_seqlen: int) -> torch.Tensor:
        """The residual stream after the last layer, before the final norm: [T, hidden] in the reader's dtype for the
        packed int32 ids [T] and cu_seqlens [B + 1] on the device."""
        T = ids.numel()
        out = torch.empty((T, self.geom["hidden_size"]), dtype=self.dtype, device=self.device)
        ws = torch.empty(self.L.rsb_llm_workspace_bytes(self._h, T, 0), dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            rc = self.L.rsb_llm_hidden_states(self._h, ctypes.c_void_p(ids.data_ptr()),
                                              ctypes.c_void_p(cu_seqlens.data_ptr()), cu_seqlens.numel() - 1, T,
                                              int(max_seqlen), ctypes.c_void_p(out.data_ptr()),
                                              ctypes.c_void_p(ws.data_ptr()), ws.numel(),
                                              ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream))
        self._check(rc)
        return out

    def loss(self, input_ids_list, labels_list, max_tokens: Optional[int] = None) -> List[float]:
        """`lm(input_ids, labels=labels).loss` per window: the mean NLL over the scored positions, NaN for a window
        without any (HF's mean over zero tokens)."""
        res = []
        for nll, lb in zip(self.nll(input_ids_list, labels_list, max_tokens), labels_list):
            pos = scored_positions([int(v) for v in lb])
            res.append(float(nll[pos].double().sum() / len(pos)) if pos else math.nan)
        return res


class B200Llama(_Reader):
    """An HF LlamaForCausalLM reader on librsb (`rsb_llm_*`)."""

    _geometry = staticmethod(llama_geometry)
    _expected_keys = staticmethod(expected_keys)
    family = _lib.RSB_LLM_LLAMA

    def _create_args(self, g):                   # rsb_llm_create's arguments after family and dtype
        return (g["num_hidden_layers"], g["hidden_size"], g["num_attention_heads"], g["num_key_value_heads"],
                g["intermediate_size"], g["vocab_size"], g["max_position_embeddings"], 128, g["rope_theta"],
                g["rms_norm_eps"], 0.0, int(g["tie_word_embeddings"]))


class B200NeoX(_Reader):
    """An HF GPTNeoXForCausalLM reader (Pythia) on librsb (`rsb_llm_*`)."""

    _geometry = staticmethod(neox_geometry)
    _expected_keys = staticmethod(neox_expected_keys)
    family = _lib.RSB_LLM_NEOX
    # older checkpoints also carry the causal mask (a 2048 x 2048 bool) and the masked-score constant
    _buffers = ("rotary_emb.inv_freq", ".attention.bias", ".attention.masked_bias")

    def _create_args(self, g):
        return (g["num_hidden_layers"], g["hidden_size"], g["num_attention_heads"], g["num_attention_heads"],
                g["intermediate_size"], g["vocab_size"], g["max_position_embeddings"], g["rotary_ndims"],
                g["rotary_emb_base"], g["layer_norm_eps"], 0.0, 0)


class B200Olmo(_Reader):
    """An HF OlmoForCausalLM / Olmo2ForCausalLM reader on librsb (`rsb_llm_*`).  Diagnostics: `attention` runs layer
    0's clip_qkv / QK-norm prologue in place of RoPE, then the same attention."""

    _geometry = staticmethod(olmo_geometry)
    _expected_keys = staticmethod(olmo_expected_keys)

    @property
    def family(self):
        return _lib.RSB_LLM_OLMO if self.geom["version"] == 1 else _lib.RSB_LLM_OLMO2

    def _create_args(self, g):
        return (g["num_hidden_layers"], g["hidden_size"], g["num_attention_heads"], g["num_key_value_heads"],
                g["intermediate_size"], g["vocab_size"], g["max_position_embeddings"], 128, g["rope_theta"], g["eps"],
                g["clip_qkv"], int(g["tie_word_embeddings"]))


READERS = {"llama": (llama_geometry, B200Llama), "gpt_neox": (neox_geometry, B200NeoX),
           "olmo": (olmo_geometry, B200Olmo), "olmo2": (olmo_geometry, B200Olmo)}


def _shard_files(directory: str) -> List[str]:
    index = os.path.join(directory, "model.safetensors.index.json")
    if os.path.exists(index):
        with open(index) as f:
            files = sorted(set(json.load(f)["weight_map"].values()))
        return [os.path.join(directory, fn) for fn in files]
    single = os.path.join(directory, "model.safetensors")
    if os.path.exists(single):
        return [single]
    # PyTorch pickles, as the Pythia suite publishes its intermediate-step revisions
    index = os.path.join(directory, "pytorch_model.bin.index.json")
    if os.path.exists(index):
        with open(index) as f:
            files = sorted(set(json.load(f)["weight_map"].values()))
        return [os.path.join(directory, fn) for fn in files]
    single = os.path.join(directory, "pytorch_model.bin")
    if os.path.exists(single):
        return [single]
    raise FileNotFoundError(f"{directory}: neither model.safetensors nor model.safetensors.index.json is present "
                            f"(nor pytorch_model.bin / pytorch_model.bin.index.json)")


def _tensors(fn: str):
    """(name, tensor) of one weight file, safetensors or a PyTorch pickle (read with weights_only=True)."""
    if fn.endswith(".safetensors"):
        from safetensors import safe_open
        with safe_open(fn, framework="pt") as f:
            for name in f.keys():
                yield name, f.get_tensor(name)
    else:
        yield from torch.load(fn, weights_only=True, map_location="cpu").items()


def load_reader(path: str, device=None, dtype=torch.float16):
    """The reader of `cfg.model.lm_model` from a local directory or the Hugging Face cache (never downloaded):
    `B200Llama` for model_type 'llama', `B200NeoX` for 'gpt_neox', `B200Olmo` for 'olmo' and 'olmo2'.  Single-file or sharded safetensors weights, or
    PyTorch `pytorch_model.bin` files when no safetensors file is present, converted to `dtype`: torch.float16 (the
    default) or torch.bfloat16 (the reference's reader dtype; also 'float16' / 'bfloat16').  Any other dtype raises
    ValueError before any file is read."""
    dtype = reader_dtype(dtype)
    from .encoder import _resolve_model_dir
    directory = _resolve_model_dir(path)
    with open(os.path.join(directory, "config.json")) as f:
        cfg = json.load(f)
    geometry, cls = READERS.get(cfg.get("model_type"), READERS["llama"])
    geometry(cfg)                                # refuses before any weight is read or device memory allocated
    files = _shard_files(directory)
    model = cls(cfg, device=device, dtype=dtype)
    with torch.cuda.device(model.device):
        for fn in files:
            for name, t in _tensors(fn):
                model.load_weight(name, t)
    model.require_all_weights(directory)
    return model
