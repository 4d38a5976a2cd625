"""Shared machinery of the three indexers: load-or-build with the reference's artefact names, the
index-id -> [shard_id, chunk_id] map, the passage store, and `.search(query_embs, k)` with the reference's
return structure `(scores: list[list[float]], passages: list[list[str]], db_ids: list[list[[shard, chunk]]])`
(`src/indicies/flat.py:138-141`).

Differences kept deliberately (SURVEY.md App. D): results padded with id -1 by the index (fewer than k
candidates) are *dropped* instead of being looked up with a negative Python index (reference quirk 3), and
the id map is two int32 arrays in memory instead of a 100M-element list of lists.  On disk the `.meta` file keeps
the reference's format -- a pickled list of [shard_id, chunk_id] pairs (`flat.py:59-66`) -- so a reference process
pointed at the same index_dir loads it; beyond `DbIdMap.LIST_LIMIT` entries an int32 ndarray [n, 2] is pickled
instead (indexing and unpacking a row behave like the list form; a 100M-element list of lists costs ~10 GB of host
memory to build).
"""
from __future__ import annotations

import os
import pickle
import time
from typing import List, Optional, Sequence

import numpy as np

from .. import index as rsb_index
from . import index_utils as iu


class DbIdMap:
    """index id -> [shard_id, chunk_id]; behaves like the reference's `index_id_to_db_id` list."""

    def __init__(self, shard: Optional[np.ndarray] = None, chunk: Optional[np.ndarray] = None):
        self.shard = np.zeros(0, np.int32) if shard is None else np.asarray(shard, np.int32)
        self.chunk = np.zeros(0, np.int32) if chunk is None else np.asarray(chunk, np.int32)

    def __len__(self):
        return int(self.shard.shape[0])

    def __getitem__(self, i):
        if isinstance(i, slice):
            return [[int(s), int(c)] for s, c in zip(self.shard[i], self.chunk[i])]
        i = int(i)
        if i < 0 or i >= len(self):
            raise IndexError(f"index id {i} out of range (ntotal = {len(self)})")
        return [int(self.shard[i]), int(self.chunk[i])]

    def extend_shard(self, shard_id: int, n: int) -> None:
        self.shard = np.concatenate([self.shard, np.full(n, shard_id, np.int32)])
        self.chunk = np.concatenate([self.chunk, np.arange(n, dtype=np.int32)])

    def lookup(self, ids: np.ndarray) -> np.ndarray:
        return np.stack([self.shard[ids], self.chunk[ids]], axis=-1)

    LIST_LIMIT = 20_000_000

    def dump(self, path: str) -> None:
        pairs = np.stack([self.shard, self.chunk], axis=1) if len(self) else np.zeros((0, 2), np.int32)
        obj = pairs.tolist() if len(self) <= self.LIST_LIMIT else pairs
        tmp = path + ".tmp"
        with open(tmp, "wb") as f:
            pickle.dump(obj, f, protocol=4)
        os.replace(tmp, path)

    @classmethod
    def load(cls, path: str) -> "DbIdMap":
        with open(path, "rb") as f:
            obj = pickle.load(f)
        if isinstance(obj, dict) and obj.get("format") == "rsb-idmap-v1":
            return cls(obj["shard"], obj["chunk"])
        arr = np.asarray(obj)                       # reference format: list of [shard_id, chunk_id]
        if arr.size == 0:
            return cls()
        if arr.ndim == 1:                           # very old metas: chunk ids only (flat.py:127-130)
            return cls(np.zeros(arr.shape[0], np.int32), arr)
        return cls(arr[:, 0], arr[:, 1])


class BaseIndexer:
    index_kind = "Flat"

    def __init__(self, embed_paths, index_path, meta_file, passage_dir=None, pos_map_save_path=None,
                 dimension=768, trained_index_path=None, sample_train_size=1000000, probe=1, storage_dtype=None,
                 device_rows=None, list_device_rows=None):
        self.embed_paths = list(embed_paths) if embed_paths is not None else []
        self.index_path, self.meta_file = index_path, meta_file
        self.trained_index_path = trained_index_path
        self.passage_dir, self.pos_map_save_path = passage_dir, pos_map_save_path
        self.dimension, self.sample_size, self.probe = int(dimension), int(sample_train_size), int(probe)
        self.cuda = True   # informational: unlike the reference (`self.cuda = False`), search runs on the GPU
        # datastore.index.storage_dtype (Flat / IVFFlat): None = fp32 vectors, the reference's upcast-on-load path
        self.storage_dtype = storage_dtype
        # datastore.index.device_rows (Flat, float16): None = every row in device memory, else a tiered index
        self.device_rows = device_rows
        # datastore.index.list_device_rows (IVFFlat): None = every list in device memory, else a tiered IVF index
        self.list_device_rows = list_device_rows
        tier = {} if list_device_rows is None else {"list_device_rows": list_device_rows}

        if os.path.exists(index_path) and os.path.exists(meta_file):
            print("Loading index...")
            self.index = rsb_index.read_index(index_path, storage_dtype=storage_dtype, device_rows=device_rows, **tier)
            self.index_id_to_db_id = DbIdMap.load(meta_file)
        else:
            self.index_id_to_db_id = DbIdMap()
            self.index = self._new_index()
            if not self.index.is_trained:
                if trained_index_path and os.path.exists(trained_index_path):
                    self.index = rsb_index.read_index(trained_index_path, storage_dtype=storage_dtype, **tier)
                else:
                    print("Training index...")
                    self._sample_and_train_index()
            print("Building index...")
            self._add_keys()
        self.index.nprobe = self.probe
        self.psg_pos_id_map = None
        if self.pos_map_save_path is not None:
            self.psg_pos_id_map = self.load_psg_pos_id_map()

    # -- subclass hook ---------------------------------------------------------------------------------------
    def _new_index(self):
        raise NotImplementedError

    # -- build -----------------------------------------------------------------------------------------------
    def _sample_and_train_index(self) -> None:
        """Per-shard uniform sample without replacement, then train (reference `ivf_flat.py:122-140`)."""
        per = max(1, self.sample_size // max(1, len(self.embed_paths)))
        rng = np.random.default_rng(1)
        parts = []
        for p in self.embed_paths:
            emb = iu.load_embedding_shard(p)
            take = min(per, emb.shape[0])
            parts.append(emb[rng.choice(emb.shape[0], size=take, replace=False)])
        t0 = time.time()
        self.index.train(np.concatenate(parts, axis=0))
        print("Finish training (%ds)" % (time.time() - t0))
        if self.trained_index_path:
            rsb_index.write_index(self.index, self.trained_index_path)

    def _add_keys(self) -> None:
        t0 = time.time()
        if self.list_device_rows is not None:
            return self._add_keys_tiered(t0)
        for i, p in enumerate(self.embed_paths):
            shard_id = iu.shard_id_of_embedding_path(p)
            emb = self._load_shard_for_add(p)
            self.index.add(emb)
            self.index_id_to_db_id.extend_shard(shard_id, emb.shape[0])
            print("Added %d / %d shards, (%d min)" % (i + 1, len(self.embed_paths), (time.time() - t0) / 60))
        self._save(t0)

    def _add_keys_tiered(self, t0: float) -> None:
        """A tiered IVF index places every row in its final slot, so it learns its list sizes first: pass 1 assigns
        each shard (the int32 lists stay on the host), then reserve_lists; pass 2 reloads each shard and adds it with
        its kept lists."""
        kept = []
        sizes = np.zeros(self.index.nlist, dtype=np.int64)
        for p in self.embed_paths:
            emb = self._load_shard_for_add(p)
            lists = np.concatenate([self.index.assign(emb[a:a + 65536]).cpu().numpy()
                                    for a in range(0, emb.shape[0], 65536)]) if emb.shape[0] else np.zeros(0, np.int32)
            sizes += np.bincount(lists, minlength=self.index.nlist)
            kept.append(lists)
        self.index.reserve_lists(sizes)
        print("Reserved %d lists, %d rows in device memory (%d min)" % (self.index.nlist, self.index.n_dev,
                                                                        (time.time() - t0) / 60))
        for i, (p, lists) in enumerate(zip(self.embed_paths, kept)):
            shard_id = iu.shard_id_of_embedding_path(p)
            emb = self._load_shard_for_add(p)
            self.index.add_preassigned(emb, lists)
            self.index_id_to_db_id.extend_shard(shard_id, emb.shape[0])
            print("Added %d / %d shards, (%d min)" % (i + 1, len(self.embed_paths), (time.time() - t0) / 60))
        self._save(t0)

    def _save(self, t0: float) -> None:
        self.index.finalize()
        os.makedirs(os.path.dirname(self.index_path) or ".", exist_ok=True)
        rsb_index.write_index(self.index, self.index_path)
        self.index_id_to_db_id.dump(self.meta_file)
        print(f"Total data indexed {len(self.index_id_to_db_id)}")

    def _load_shard_for_add(self, path: str) -> np.ndarray:
        """fp32 rows (the reference's upcast on load), or, with storage_dtype set, the rows as the embedding task
        stored them: fp16 pickles go to the GPU as fp16.  An fp16 index refuses an fp32 shard whose values do not
        round-trip through fp16, since its results would no longer be the reference's."""
        if self.storage_dtype is None:
            return iu.load_embedding_shard(path)
        emb = iu.load_embedding_shard(path, dtype=None)
        if emb.dtype not in (np.float16, np.float32):
            emb = emb.astype(np.float32)
        if self.storage_dtype == "float16":
            emb = rsb_index._as_storage(emb, "float16", f"embedding shard {path}")
        return emb

    # -- passages --------------------------------------------------------------------------------------------
    def load_psg_pos_id_map(self):
        if os.path.exists(self.pos_map_save_path):
            with open(self.pos_map_save_path, "rb") as f:
                return pickle.load(f)
        return self.build_passage_pos_id_map()

    def build_passage_pos_id_map(self):
        iu.convert_pkl_to_jsonl(self.passage_dir)
        return iu.get_passage_pos_ids(self.passage_dir, self.pos_map_save_path)

    def _id2psg(self, shard_id, chunk_id):
        return iu.fetch_passages(self.psg_pos_id_map, [(shard_id, chunk_id)])[0]

    def _get_passage(self, index_id):
        shard_id, chunk_id = self.index_id_to_db_id[index_id]
        return self._id2psg(shard_id, chunk_id)

    def get_retrieved_passages(self, all_indices):
        all_indices = np.asarray(all_indices)
        flat_ids = all_indices.reshape(-1)
        valid = flat_ids >= 0
        pairs = self.index_id_to_db_id.lookup(flat_ids[valid])
        texts: List[Optional[str]] = [None] * int(valid.sum())
        if self.psg_pos_id_map is not None:
            texts = [rec["text"] for rec in iu.fetch_passages(self.psg_pos_id_map, pairs)]
        passages, db_ids, it = [], [], 0
        for row in all_indices:
            nvalid = int((row >= 0).sum())
            passages.append(texts[it:it + nvalid])
            db_ids.append([[int(s), int(c)] for s, c in pairs[it:it + nvalid]])
            it += nvalid
        return passages, db_ids

    # -- search ----------------------------------------------------------------------------------------------
    def search_ids(self, query_embs, k: int):
        """Fast path: CUDA tensor in -> (ids int64 [nq,k], scores float32 [nq,k]) CUDA tensors out."""
        return self.index.search_ids(query_embs, k)

    def search(self, query_embs, k=4096, return_passages: bool = True):
        all_scores, all_indices = self.index.search(np.asarray(query_embs).astype(np.float32), k)
        if not return_passages:
            return all_scores.tolist(), None, [self.index_id_to_db_id.lookup(r[r >= 0]).tolist() for r in all_indices]
        all_passages, db_ids = self.get_retrieved_passages(all_indices)
        scores = [row[: len(ids)].tolist() for row, ids in zip(all_scores, db_ids)]
        return scores, all_passages, db_ids
