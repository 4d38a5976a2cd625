"""Per-shard-group re-ranking under torchrun: `ric/main_ric.py tasks.eval.search=true` over index_shard_ids=[[0],[1]]
with datastore.index.refine_k_factor set.  Each rank re-ranks its own group's candidates before the cross-rank merge,
so the merged result must equal the single-process flow (per-group refined search + post-hoc merge, reference
src/search.py:312-373), and every returned score must be the exact inner product with the passage's embedding."""
import json
import os
import pickle
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")]


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_torchrun_per_group_refine_equals_single_process(tmp_path):
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_gpu_indexer import D as DIM, ROOT, _make_datastore
    embs, q = _make_datastore(str(tmp_path))
    eval_path = tmp_path / "nq.jsonl"
    with open(eval_path, "w") as f:
        for i in range(12):
            f.write(json.dumps({"query": f"question {i}"}) + "\n")
    qcache = tmp_path / "q.pkl"
    with open(qcache, "wb") as f:
        pickle.dump(q, f)
    common = ["--config-name", "default", f"datastore.datastore_root_dir={tmp_path}", "datastore.domain=dom",
              "model.datastore_encoder=enc", "datastore.embedding.num_shards=2", "datastore.index.index_type=IVFPQ",
              "datastore.index.ncentroids=16", "datastore.index.probe=4", "datastore.index.sample_train_size=4000",
              "datastore.index.n_subquantizers=16", "+datastore.index.refine_k_factor=8",
              "datastore.index.index_shard_ids=[[0],[1]]", f"datastore.index.projection_size={DIM}",
              "evaluation.search.n_docs=5", "evaluation.domain=dom", f"evaluation.data.eval_data={eval_path}",
              "tasks.eval.search=true", "tasks.eval.task_name=lm-eval", "+evaluation.search.cache_query_embedding=true",
              f"+evaluation.search.query_embedding_save_path={qcache}"]
    main = os.path.join(ROOT, "ric", "main_ric.py")
    out_a, out_b = tmp_path / "out_single", tmp_path / "out_torchrun"
    r = subprocess.run([sys.executable, main] + common + [f"evaluation.eval_output_dir={out_a}"], cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
                        "127.0.0.1", "--master-port", str(_free_port()), main] + common + [f"evaluation.eval_output_dir={out_b}"],
                       cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    a = [json.loads(l) for l in open(out_a / "0-1" / "nq_retrieved_results.jsonl")]
    b = [json.loads(l) for l in open(out_b / "0-1" / "nq_retrieved_results.jsonl")]
    assert len(a) == len(b) == 12
    for i, (ea, eb) in enumerate(zip(a, b)):
        assert [c["id"] for c in ea["ctxs"]] == [c["id"] for c in eb["ctxs"]]
        sa = [float(c["retrieval score"]) for c in ea["ctxs"]]
        assert np.allclose(sa, [float(c["retrieval score"]) for c in eb["ctxs"]], rtol=1e-6, atol=1e-6)
        assert sa == sorted(sa, reverse=True)
