"""Path derivation and the on-disk passage store (reference: `src/indicies/index_utils.py`).

Artefact layout kept identical to the reference so existing `scaling_out/` trees load unchanged:
  embeddings   {embedding_dir}/{prefix}_{shard:02d}.pkl        pickle (ids, ndarray[n, d] fp16|fp32)   (:20)
  index dir    {embedding_dir}/index_{type}/{ids joined by _}                                          (:24-25)
  passages     {passages_dir}/raw_passages-{i}-of-{n}.jsonl    one JSON per line                       (:103)
  offset map   passage_pos_id_map.pkl : {shard_id: {chunk_id: [path, byte_offset]}}                    (:71-134)

Deliberate differences from the reference (SURVEY.md App. D quirks 1-2): nested `index_shard_ids`
(`[[0],[1]]`) and `index_shard_ids: null` are handled instead of raising.
"""
from __future__ import annotations

import glob
import json
import os
import pickle
import re
from typing import Dict, List, Sequence, Tuple

import numpy as np


def _as_int_list(x) -> List[int]:
    return sorted(int(i) for i in x)


def get_index_dir_and_embedding_paths(cfg, index_shard_ids=None) -> Tuple[str, List[str]]:
    emb, idx = cfg.datastore.embedding, cfg.datastore.index
    index_type = idx.index_type
    if index_shard_ids is None:
        index_shard_ids = idx.get("index_shard_ids", None)
    if index_shard_ids:
        if isinstance(index_shard_ids[0], (list, tuple)):      # nested form: caller should pass one group
            if len(index_shard_ids) != 1:
                raise ValueError("pass one shard group (e.g. [0, 1]) per index; got a nested list of several")
            index_shard_ids = index_shard_ids[0]
        shard_ids = _as_int_list(index_shard_ids)
        paths = [os.path.join(emb.embedding_dir, f"{emb.prefix}_{s:02d}.pkl") for s in shard_ids]
        index_dir = os.path.join(os.path.dirname(paths[0]), f"index_{index_type}", "_".join(map(str, shard_ids)))
        return index_dir, paths
    paths = glob.glob(idx.passages_embeddings)
    if not paths:
        raise FileNotFoundError(f"no embedding files match {idx.passages_embeddings}")
    key = lambda p: int(re.search(r"_(\d+)\.pkl$", os.path.basename(p)).group(1))  # noqa: E731
    paths = sorted(paths, key=key)
    nsub = idx.get("num_subsampled_embedding_files", -1)
    if nsub is not None and nsub != -1:
        paths = paths[:nsub]
    return os.path.join(os.path.dirname(paths[0]), f"index_{index_type}"), paths


def shard_id_of_embedding_path(path: str) -> int:
    m = re.search(r"_(\d+)\.pkl$", os.path.basename(path))
    if not m:
        raise ValueError(f"cannot read a shard id from {path}")
    return int(m.group(1))


def load_embedding_shard(path: str, dtype=np.float32) -> np.ndarray:
    """(ids, embeddings) pickle -> [n, d] in `dtype` (None: as stored, fp16 when the embedding task wrote it); the
    ids inside the pickle are ignored, row order defines chunk_id (reference `flat.py:59,86`)."""
    with open(path, "rb") as f:
        _ids, emb = pickle.load(f)
    emb = np.asarray(emb)
    return np.ascontiguousarray(emb, dtype=emb.dtype if dtype is None else dtype)


def convert_pkl_to_jsonl(passage_dir: str) -> None:
    """Legacy passage pickles -> JSONL next to them (reference :38-68)."""
    if os.path.isdir(passage_dir):
        files = [os.path.join(passage_dir, f) for f in os.listdir(passage_dir) if f.endswith(".pkl") and "pos_id_map" not in f]
    elif os.path.isfile(passage_dir) and passage_dir.endswith(".pkl"):
        files = [passage_dir]
    else:
        raise AssertionError(f"{passage_dir} does not exist or is neither a file nor a directory.")
    for fp in files:
        out = fp[:-4] + ".jsonl"
        if os.path.exists(out):
            continue
        with open(fp, "rb") as f:
            data = pickle.load(f)
        with open(out, "w") as f:
            for item in data:
                f.write(json.dumps(item) + "\n")


def _scan_offsets(file_path: str) -> Dict[int, list]:
    out, pos, doc = {}, 0, 0
    with open(file_path, "rb") as f:       # binary: tell() is the byte offset `seek` needs
        for line in f:
            out[doc] = [file_path, pos]
            pos += len(line)
            doc += 1
    return out


def get_passage_pos_ids(passage_dir: str, pos_map_save_path: str) -> Dict[int, Dict[int, list]]:
    if pos_map_save_path and os.path.exists(pos_map_save_path):
        with open(pos_map_save_path, "rb") as f:
            return pickle.load(f)
    pos_id_map: Dict[int, Dict[int, list]] = {}
    if os.path.isdir(passage_dir):
        for name in sorted(os.listdir(passage_dir)):
            m = re.match(r"raw_passages-(\d+)-of-\d+\.jsonl$", name)
            if m:
                pos_id_map[int(m.group(1))] = _scan_offsets(os.path.join(passage_dir, name))
    elif os.path.isfile(passage_dir) and passage_dir.endswith(".pkl") and os.path.exists(passage_dir[:-4] + ".jsonl"):
        m = re.search(r"-(\d+)-of-\d+\.pkl$", passage_dir)
        assert m, f"Cannot extract shard_id from {passage_dir}"
        pos_id_map[int(m.group(1))] = _scan_offsets(passage_dir[:-4] + ".jsonl")
    else:
        raise AssertionError(f"{passage_dir} does not exist or is neither a file nor a directory.")
    if pos_map_save_path:
        tmp = pos_map_save_path + ".tmp"
        with open(tmp, "wb") as f:
            pickle.dump(pos_id_map, f)
        os.replace(tmp, pos_map_save_path)
    return pos_id_map


try:                                    # optional: msgspec decodes a passage record in half the time of json.loads and
    import msgspec as _msgspec          # returns the same builtin objects (scripts/bench_passage_fetch.py); json is the fallback
    _fast_decode = _msgspec.json.decode
except Exception:                       # not installed: plain json
    _fast_decode = None


def _loads_record(line: bytes):
    if _fast_decode is not None:
        try:
            return _fast_decode(line)
        except Exception:               # let the standard library raise its own error type for a malformed line
            pass
    return json.loads(line)


def fetch_passages(pos_id_map, db_ids: Sequence[Sequence[int]]) -> List[dict]:
    """Batched passage fetch (SURVEY §8f-2): group by file, sort by offset, one open() per file instead of one
    per (query, rank) as in the reference's `_id2psg` (`ivf_pq.py:209-214`).  Returns records in input order."""
    by_file: Dict[str, list] = {}
    for i, (shard, chunk) in enumerate(db_ids):
        path, pos = pos_id_map[int(shard)][int(chunk)]
        by_file.setdefault(path, []).append((pos, i))
    out: List[dict] = [None] * len(db_ids)  # type: ignore
    for path, items in by_file.items():
        items.sort()
        with open(path, "rb") as f:
            for pos, i in items:
                f.seek(pos)
                out[i] = _loads_record(f.readline())
    return out
