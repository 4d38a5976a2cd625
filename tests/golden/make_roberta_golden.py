"""Writes tests/golden/roberta_golden.npz: HF transformers' own RobertaModel -- the class the reference's
`AutoModel.from_pretrained(name)` builds for the DRAGON-RoBERTa checkpoints (src/search.py:241-243,
src/embed.py:123-126) -- run in fp32 on the CPU on the two encoders of roberta_fixture.py, for the fixed query set
QUERIES (see `queries`), tokenised by the fixture's tokenizer as the reference does (padding to the longest,
truncation to 512).

Stored: the query texts, the padded input_ids / attention_mask, and the CLS rows `last_hidden_state[:, 0, :]` of the
query encoder (cls_query) and of the context encoder (cls_context).

    python tests/golden/make_roberta_golden.py
"""
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import roberta_fixture as RF  # noqa: E402

MAX_LENGTH = 512


def _n_tokens(tok, text):
    return len(tok(text)["input_ids"])


def _exactly(tok, n):
    """Words from RF.WORDS appended until the tokenised text is exactly n tokens (<s> and </s> included)."""
    words, i = [], 0
    while True:
        text = " ".join(words)
        k = _n_tokens(tok, text)
        if k == n:
            return text
        if k > n:                                         # the last word overshot: try the next one instead
            words.pop()
        words.append(RF.WORDS[i % len(RF.WORDS)])
        i += 1
        if i > 10 * n:
            raise RuntimeError(f"no text of exactly {n} tokens")


def queries(tok):
    """The fixed query set: empty, one word, 31 / 32 / 33 tokens, one truncated at 512 tokens, two holding the literal
    text <pad> (tokenised to id 1 inside the sequence), non-ASCII text, and a few ordinary questions."""
    long_text = " ".join(f"{RF.WORDS[i % len(RF.WORDS)]}{i % 7}" for i in range(700))
    return ["", "moon", "a", _exactly(tok, 31), _exactly(tok, 32), _exactly(tok, 33), long_text,
            "ab <pad> c", "who wrote <pad> the origin of <pad><pad> species",
            "Zürich – straße, 東京の川 🌙 ¿qué?", "when did the berlin wall fall",
            "largest moon of saturn", "How many bytes have the cache and its width?"]


def main():
    import transformers
    tok = RF.tokenizer()
    texts = queries(tok)
    enc = tok(texts, return_tensors="pt", padding=True, truncation=True, max_length=MAX_LENGTH)
    assert "token_type_ids" not in enc
    out = {"texts": np.array(texts), "input_ids": enc["input_ids"].numpy().astype(np.int32),
           "attention_mask": enc["attention_mask"].numpy().astype(np.int8),
           "transformers_version": np.array(transformers.__version__)}
    with tempfile.TemporaryDirectory() as tmp:
        fx = RF.build(tmp)
        for which in ("query", "context"):
            model = transformers.AutoModel.from_pretrained(fx[which]["dir"], local_files_only=True).eval().float()
            assert type(model).__name__ == "RobertaModel", type(model)
            with torch.no_grad():
                h = model(input_ids=enc["input_ids"], attention_mask=enc["attention_mask"]).last_hidden_state
            out[f"cls_{which}"] = h[:, 0, :].numpy().astype(np.float32)
    lens = out["attention_mask"].sum(1)
    print("token counts:", lens.tolist())
    np.savez_compressed(os.path.join(HERE, "roberta_golden.npz"), **out)


if __name__ == "__main__":
    main()
