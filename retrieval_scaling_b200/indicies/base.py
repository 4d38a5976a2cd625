"""`Indexer(cfg)` -- the drop-in boundary (reference `src/indicies/base.py:12-77`).

Same constructor contract (reads `cfg.datastore.index` / `cfg.datastore.embedding`, derives the index, meta
and passage-offset-map paths with the reference's naming scheme, dispatches on `index_type`) and the same
`search(query_embs, k) -> (all_scores, all_passages, db_ids)`; additionally `search_ids` for the tensor fast
path.  Unknown `index_type` raises NotImplementedError like `base.py:71-72`.
"""
from __future__ import annotations

import logging
import os

from .flat import FlatIndexer
from .index_utils import get_index_dir_and_embedding_paths
from .ivf_flat import IVFFlatIndexer
from .ivf_pq import IVFPQIndexer


class Indexer(object):
    @staticmethod
    def artefact_paths(cfg, index_shard_ids=None):
        """The reference's naming scheme (`base.py:23-30`): index / meta / passage-offset-map paths of a shard group."""
        a = cfg.datastore.index
        index_dir, embedding_paths = get_index_dir_and_embedding_paths(cfg, index_shard_ids)
        if "IVF" in a.index_type:
            name = f"index_{a.index_type}.{a.sample_train_size}.{a.projection_size}.{a.ncentroids}.faiss"
        else:
            name = f"index_{a.index_type}.faiss"
        index_path = os.path.join(index_dir, name)
        return dict(index_dir=index_dir, embed_paths=embedding_paths, index_path=index_path, meta_file=index_path + ".meta",
                    pos_map_save_path=os.path.join(index_dir, "passage_pos_id_map.pkl"))

    @staticmethod
    def refine_options(index_cfg):
        """Optional keys `refine_k_factor` (absent or 0: no re-ranking) and `refine_dtype` (float16 | float32 | sq8; absent:
        the embedding pickles' dtype) -> (k_factor, dtype).  Re-ranking applies to IVFPQ only."""
        k_factor = int(index_cfg.get("refine_k_factor", 0) or 0)
        dtype = index_cfg.get("refine_dtype", None)
        if k_factor < 0:
            raise ValueError(f"datastore.index.refine_k_factor must be >= 0, got {k_factor}")
        if k_factor and index_cfg.index_type != "IVFPQ":
            raise ValueError(f"datastore.index.refine_k_factor re-ranks IVFPQ results; {index_cfg.index_type} scores "
                             f"are already exact")
        if dtype not in (None, "float16", "float32", "sq8"):
            raise ValueError(f"datastore.index.refine_dtype must be float16, float32 or sq8, got {dtype!r}")
        Indexer.refine_device_rows(index_cfg)
        return k_factor, dtype

    @staticmethod
    def _rows_key(index_cfg, key):
        """Optional key `key`: None when absent, else an integer >= 0 (ValueError naming the key otherwise)."""
        rows = index_cfg.get(key, None)
        if rows is not None and (isinstance(rows, bool) or not isinstance(rows, int) or rows < 0):
            raise ValueError(f"datastore.index.{key} must be an integer >= 0, got {rows!r}")
        return rows

    @staticmethod
    def refine_device_rows(index_cfg):
        """Optional key `refine_device_rows` (absent: None, every store row in device memory): an integer >= 0; store rows
        from that id on are kept in pinned host memory (index.IndexRefine(device_rows=...)).  Needs refine_k_factor > 0."""
        rows = Indexer._rows_key(index_cfg, "refine_device_rows")
        if rows is None:
            return None
        if not int(index_cfg.get("refine_k_factor", 0) or 0) > 0:
            raise ValueError("datastore.index.refine_device_rows splits the re-rank store: it needs refine_k_factor > 0")
        return rows

    @staticmethod
    def storage_dtype(index_cfg):
        """Optional key `storage_dtype` (float32 | float16 | sq8; absent: None, today's fp32 path) -> the dtype Flat and
        IVFFlat indexes store their vectors in.  sq8 (IVFFlat only) builds faiss' "IVFn,SQ8": an IndexIVFScalarQuantizer
        with 8-bit codes of the residuals.  IVFPQ stores codes, so the key is refused there."""
        dtype = index_cfg.get("storage_dtype", None)
        if dtype is None:
            return None
        if dtype not in ("float16", "float32", "sq8"):
            raise ValueError(f"datastore.index.storage_dtype must be float16 or float32 (IVFFlat also takes sq8), "
                             f"got {dtype!r}")
        if index_cfg.index_type not in ("Flat", "IVFFlat"):
            raise ValueError(f"datastore.index.storage_dtype applies to Flat and IVFFlat indexes; {index_cfg.index_type} "
                             f"stores PQ codes")
        if dtype == "sq8" and index_cfg.index_type != "IVFFlat":
            raise ValueError(f"datastore.index.storage_dtype sq8 applies to IVFFlat indexes only (IVF-SQ8); "
                             f"{index_cfg.index_type} takes float16 or float32")
        return dtype

    @staticmethod
    def device_rows(index_cfg):
        """Optional key `device_rows` (absent: None, every row in device memory): an integer >= 0; Flat rows from that
        position on are kept in pinned host memory and streamed to the GPU by each search (index.IndexFlatIP(
        device_rows=...)).  Needs index_type Flat with storage_dtype float16."""
        rows = Indexer._rows_key(index_cfg, "device_rows")
        if rows is None:
            return None
        if index_cfg.index_type != "Flat" or index_cfg.get("storage_dtype", None) != "float16":
            raise ValueError(f"datastore.index.device_rows splits a Flat index between device and host memory: it needs "
                             f"index_type Flat and storage_dtype float16 (got {index_cfg.index_type}, "
                             f"{index_cfg.get('storage_dtype', None)})")
        return rows

    @staticmethod
    def list_device_rows(index_cfg):
        """Optional key `list_device_rows` (absent: None, every list in device memory): an integer >= 0; an IVFFlat index
        (any storage_dtype) keeps the rows of its first lists -- as many as fit that many rows -- in device memory and the
        others in pinned host memory, copying only the probed host lists at search time (index.IndexIVFFlat(
        list_device_rows=...)).  Needs index_type IVFFlat."""
        rows = Indexer._rows_key(index_cfg, "list_device_rows")
        if rows is None:
            return None
        if index_cfg.index_type != "IVFFlat":
            raise ValueError(f"datastore.index.list_device_rows splits the inverted lists of an IVFFlat index between "
                             f"device and host memory: it needs index_type IVFFlat (got {index_cfg.index_type})")
        return rows

    def __init__(self, cfg, index_shard_ids=None):
        self.cfg = cfg
        self.args = cfg.datastore.index
        self.index_type = self.args.index_type
        self.refine_options(self.args)
        storage_dtype = self.storage_dtype(self.args)
        device_rows = self.device_rows(self.args)
        list_device_rows = self.list_device_rows(self.args)

        passage_dir = self.cfg.datastore.embedding.passages_dir
        paths = self.artefact_paths(cfg, index_shard_ids)
        index_dir, embedding_paths, index_path = paths["index_dir"], paths["embed_paths"], paths["index_path"]
        os.makedirs(index_dir, exist_ok=True)
        logging.info(f"Indexing for passages: {embedding_paths}")
        a = self.args
        common = dict(embed_paths=embedding_paths, index_path=index_path, meta_file=paths["meta_file"],
                      passage_dir=passage_dir, pos_map_save_path=paths["pos_map_save_path"],
                      dimension=a.projection_size)
        if a.get("overwrite", False):
            for p in (index_path, index_path + ".meta", index_path + ".trained"):
                if os.path.exists(p):
                    os.remove(p)
        if self.index_type == "Flat":
            self.datastore = FlatIndexer(storage_dtype=storage_dtype, device_rows=device_rows, **common)
        elif self.index_type == "IVFFlat":
            self.datastore = IVFFlatIndexer(trained_index_path=index_path + ".trained", sample_train_size=a.sample_train_size,
                                            prev_index_path=None, ncentroids=a.ncentroids, probe=a.probe,
                                            storage_dtype=storage_dtype, list_device_rows=list_device_rows, **common)
        elif self.index_type == "IVFPQ":
            k_factor, refine_dtype = self.refine_options(a)
            self.datastore = IVFPQIndexer(trained_index_path=index_path + ".trained", sample_train_size=a.sample_train_size,
                                          prev_index_path=None, ncentroids=a.ncentroids, probe=a.probe,
                                          n_subquantizers=a.n_subquantizers, code_size=a.n_bits,
                                          refine_k_factor=k_factor, refine_dtype=refine_dtype,
                                          refine_device_rows=self.refine_device_rows(a), **common)
        else:
            raise NotImplementedError

    def search(self, query_embs, k=5):
        all_scores, all_passages, db_ids = self.datastore.search(query_embs, k)
        return all_scores, all_passages, db_ids

    def search_ids(self, query_embs, k=5):
        """(ids int64 [nq,k], scores float32 [nq,k]) as CUDA tensors -- no passage fetch, no host copy."""
        return self.datastore.search_ids(query_embs, k)
