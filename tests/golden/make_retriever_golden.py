"""Generates tests/golden/retriever_ckpt.npz with the REFERENCE's own loader and model
(`contriever.src.contriever.load_retriever`, contriever/src/contriever.py:103-138 of the reference checkout) on the
deterministic checkpoint directory of retriever_fixture.py.  Needs a checkout of the reference project, named by
REFERENCE_ROOT:

    REFERENCE_ROOT=<reference checkout> python tests/golden/make_retriever_golden.py
"""
import os
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.environ["REFERENCE_ROOT"])
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from contriever.src.contriever import load_retriever  # noqa: E402  (the reference loader)

import retriever_fixture as RF  # noqa: E402


def main():
    # The reference calls torch.load(path, map_location="cpu") (contriever.py:107); torch >= 2.6 defaults to
    # weights_only=True, which rejects the argparse.Namespace every Contriever checkpoint stores under "opt".
    # Allow-listing that class is the environment fix a user of the reference needs too (the reference is unmodified).
    import argparse
    torch.serialization.add_safe_globals([argparse.Namespace])
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        paths = RF.build(tmp)
        for branch in ("ckpt", "hf"):
            model, tokenizer, model_id = load_retriever(paths[branch])
            model.eval()
            enc = tokenizer(RF.QUERIES, return_tensors="pt", max_length=512, padding=True, truncation=True)
            with torch.no_grad():
                emb = model(**enc)
            out[f"{branch}_input_ids"] = enc["input_ids"].numpy()
            out[f"{branch}_attention_mask"] = enc["attention_mask"].numpy()
            out[f"{branch}_emb"] = emb.float().numpy()
            print(branch, "model id:", os.path.basename(model_id), "emb", tuple(emb.shape), "norm", float(emb.norm(dim=1).mean()))
    assert np.array_equal(out["ckpt_input_ids"], out["hf_input_ids"])
    print("max |ckpt - hf| =", float(np.abs(out["ckpt_emb"] - out["hf_emb"]).max()))
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "retriever_ckpt.npz"), **out)


if __name__ == "__main__":
    main()
