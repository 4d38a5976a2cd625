"""Deterministic local sentence-transformers model directories, rebuilt on demand (nothing large is committed):

    <root>/sentence-transformers-t5-fixture/   modules.json: Transformer (2-layer T5 encoder, d_model 768, Unigram
                                               tokenizer.json), 1_Pooling (mean), 2_Dense (768 -> 768, bias),
                                               3_Normalize -- the GTR-T5 stack
    <root>/e5-bert-fixture/                    modules.json: Transformer (2-layer BERT, the WordPiece vocabulary of
                                               retriever_fixture), 1_Pooling (mean), 2_Normalize -- the e5-base stack

Weights come from `oracle.t5_oracle.seeded_state_dict` / `oracle.bert_oracle.seeded_state_dict` (CPU generator:
identical on every machine).  The directory names carry "sentence-transformers" / "e5", the reference's name dispatch."""
import json
import os

import torch

T5_CONFIG = dict(d_model=768, num_heads=12, d_kv=64, d_ff=3072, num_layers=2, vocab_size=2048,
                 relative_attention_num_buckets=32, relative_attention_max_distance=128, layer_norm_epsilon=1e-6,
                 feed_forward_proj="relu")
T5_SEED, BERT_SEED = 41, 42
MAX_SEQ_LENGTH = 256
WORDS = ["the", "of", "who", "what", "when", "how", "is", "in", "a", "did", "does", "many", "large", "and", "its",
         "capital", "wall", "fall", "moon", "mountain", "south", "america", "tall", "est", "wrote", "origin", "species",
         "australia", "berlin", "saturn", "largest", "band", "width", "cache", "have", "mega", "bytes", "title", "text"]


def unigram_vocab(size: int):
    """(piece, log-probability) pairs: the specials, then whole words, single characters, and filler pieces."""
    vocab = [("<pad>", 0.0), ("</s>", 0.0), ("<unk>", 0.0)]
    vocab += [("▁" + w, -5.0 - 0.01 * i) for i, w in enumerate(WORDS)]
    vocab += [("▁", -6.0)] + [(c, -9.0) for c in "abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789?.,!'-"]
    i = 0
    while len(vocab) < size:
        vocab.append((f"▁w{i}", -12.0))
        i += 1
    return vocab[:size]


def _write_json(path, obj):
    with open(path, "w") as f:
        json.dump(obj, f, indent=1)


def _save(path, sd):
    from safetensors.torch import save_file
    save_file({k: v.contiguous() for k, v in sd.items()}, path)


def _modules(root, stack):
    names = {"Transformer": "", "Pooling": "1_Pooling", "Dense": "2_Dense", "Normalize": f"{len(stack) - 1}_Normalize"}
    mods = [{"idx": i, "name": str(i), "path": names[k], "type": "sentence_transformers.models." + k}
            for i, k in enumerate(stack)]
    _write_json(os.path.join(root, "modules.json"), mods)
    for m in mods[1:]:
        os.makedirs(os.path.join(root, m["path"]), exist_ok=True)
    _write_json(os.path.join(root, "1_Pooling", "config.json"),
                {"word_embedding_dimension": 768, "pooling_mode_cls_token": False, "pooling_mode_mean_tokens": True,
                 "pooling_mode_max_tokens": False, "pooling_mode_mean_sqrt_len_tokens": False,
                 "pooling_mode_weightedmean_tokens": False, "pooling_mode_lasttoken": False,
                 "include_prompt": True})
    return mods


def build_t5(root: str) -> dict:
    from tokenizers import Tokenizer, decoders, models, normalizers, pre_tokenizers, processors

    from oracle.t5_oracle import seeded_state_dict
    d = os.path.join(root, "sentence-transformers-t5-fixture")
    os.makedirs(d, exist_ok=True)
    _modules(d, ["Transformer", "Pooling", "Dense", "Normalize"])
    _write_json(os.path.join(d, "sentence_bert_config.json"), {"max_seq_length": MAX_SEQ_LENGTH, "do_lower_case": False})
    _write_json(os.path.join(d, "config.json"),
                {"model_type": "t5", "architectures": ["T5EncoderModel"], "is_encoder_decoder": False,
                 "dropout_rate": 0.0, "pad_token_id": 0, "eos_token_id": 1, "decoder_start_token_id": 0,
                 "use_cache": False, **T5_CONFIG})
    tok = Tokenizer(models.Unigram(unigram_vocab(T5_CONFIG["vocab_size"]), unk_id=2))
    tok.normalizer = normalizers.Sequence([normalizers.NFKC(), normalizers.Replace("  ", " ")])
    tok.pre_tokenizer = pre_tokenizers.Metaspace(replacement="▁", prepend_scheme="always")
    tok.decoder = decoders.Metaspace(replacement="▁", prepend_scheme="always")
    tok.post_processor = processors.TemplateProcessing(single="$A </s>", pair="$A </s> $B </s>",
                                                       special_tokens=[("</s>", 1)])
    tok.save(os.path.join(d, "tokenizer.json"))
    _write_json(os.path.join(d, "tokenizer_config.json"),
                {"tokenizer_class": "PreTrainedTokenizerFast", "model_max_length": 512, "pad_token": "<pad>",
                 "eos_token": "</s>", "unk_token": "<unk>"})
    sd = seeded_state_dict(T5_CONFIG, T5_SEED)
    _save(os.path.join(d, "model.safetensors"),
          {k: v for k, v in sd.items() if not k.startswith("dense.") and k != "encoder.embed_tokens.weight"})
    _write_json(os.path.join(d, "2_Dense", "config.json"),
                {"in_features": 768, "out_features": 768, "bias": True,
                 "activation_function": "torch.nn.modules.linear.Identity"})
    _save(os.path.join(d, "2_Dense", "model.safetensors"), {"linear.weight": sd["dense.weight"], "linear.bias": sd["dense.bias"]})
    return {"dir": d, "state_dict": sd, "config": T5_CONFIG}


def build_bert(root: str) -> dict:
    from oracle.bert_oracle import seeded_state_dict

    from .retriever_fixture import CONFIG, vocab_tokens
    d = os.path.join(root, "e5-bert-fixture")
    os.makedirs(d, exist_ok=True)
    _modules(d, ["Transformer", "Pooling", "Normalize"])
    _write_json(os.path.join(d, "sentence_bert_config.json"), {"max_seq_length": MAX_SEQ_LENGTH, "do_lower_case": False})
    _write_json(os.path.join(d, "config.json"),
                {"model_type": "bert", "architectures": ["BertModel"], "hidden_act": "gelu", "pad_token_id": 0,
                 "position_embedding_type": "absolute", **CONFIG})
    with open(os.path.join(d, "vocab.txt"), "w") as f:
        f.write("\n".join(vocab_tokens()) + "\n")
    _write_json(os.path.join(d, "tokenizer_config.json"),
                {"do_lower_case": True, "tokenizer_class": "BertTokenizer", "model_max_length": 512})
    sd = seeded_state_dict(CONFIG, BERT_SEED)
    _save(os.path.join(d, "model.safetensors"), sd)
    return {"dir": d, "state_dict": sd, "config": CONFIG}


def build(root: str) -> dict:
    return {"t5": build_t5(root), "bert": build_bert(root)}
