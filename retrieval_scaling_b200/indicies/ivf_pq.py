"""IVFPQIndexer -- inverted file + residual product quantisation, inner product (reference
`src/indicies/ivf_pq.py:35-232`: IndexIVFPQ(IndexFlatIP(d), d, ncentroids, n_subquantizers, code_size,
METRIC_INNER_PRODUCT); note the reference passes `n_bits` as `code_size` = bits per sub-quantizer).

With `refine_k_factor` > 0 the search re-ranks k * refine_k_factor IVF-PQ candidates exactly against the passage
embeddings (index.IndexRefine; the reference's unused `get_knn_scores` path, `ivf_pq.py:119-123`).  The store is
built from the embedding pickles on the GPU, or, with `refine_device_rows`, split between device memory (rows below it)
and pinned host memory (the rest); the `.faiss` file stays the plain IVF-PQ index.  `refine_dtype: sq8` stores 8-bit
scalar-quantizer codes (faiss `Refine(SQ8)`), trained on the first min(ntotal, sample_train_size) store rows in id
order, so a reload from the same pickles rebuilds the same store."""
from __future__ import annotations

import numpy as np

from .. import index as rsb_index
from . import index_utils as iu
from ._common import BaseIndexer


class IVFPQIndexer(BaseIndexer):
    index_kind = "IVFPQ"

    def __init__(self, embed_paths, index_path, meta_file, trained_index_path, passage_dir=None,
                 pos_map_save_path=None, sample_train_size=1000000, prev_index_path=None, dimension=768,
                 dtype=None, ncentroids=4096, probe=2048, num_keys_to_add_at_a_time=1000000,
                 DSTORE_SIZE_BATCH=51200000, n_subquantizers=16, code_size=8, refine_k_factor=0, refine_dtype=None,
                 refine_device_rows=None):
        self.ncentroids = int(ncentroids)
        self.n_subquantizers, self.code_size = int(n_subquantizers), int(code_size)
        self.prev_index_path = prev_index_path
        super().__init__(embed_paths, index_path, meta_file, passage_dir, pos_map_save_path, dimension,
                         trained_index_path=prev_index_path or trained_index_path,
                         sample_train_size=sample_train_size, probe=probe)
        if refine_k_factor:
            self.index = self._build_refine(int(refine_k_factor), refine_dtype, refine_device_rows)

    def _new_index(self):
        return rsb_index.IndexIVFPQ(self.dimension, self.ncentroids, self.n_subquantizers, self.code_size)

    def _build_refine(self, k_factor: int, refine_dtype, device_rows=None):
        """Re-rank store from the embedding pickles in the order `_add_keys` added them (the `.meta` order, so row =
        index id), copied one shard at a time: rows below device_rows (None: all) are uploaded, the rest are copied
        into the pinned host tier without crossing PCIe.  An sq8 store is built in the same single pass: the shards are
        held until the first min(ntotal, sample_train_size) rows have been read, the quantizer is trained on those
        rows, and then every shard is encoded in order."""
        base, meta = self.index, self.index_id_to_db_id
        if len(meta) != base.ntotal:
            raise ValueError(f"{self.meta_file} maps {len(meta)} ids but the index holds {base.ntotal} vectors")
        n_train = min(base.ntotal, self.sample_size)
        held, sample = [], []                           # sq8: shards read before the quantizer is trained
        refine, row = None, 0
        for p in self.embed_paths:
            emb = iu.load_embedding_shard(p, dtype=None)
            n = emb.shape[0]
            shard = iu.shard_id_of_embedding_path(p)
            if (row + n > len(meta) or not np.all(meta.shard[row:row + n] == shard)
                    or not np.array_equal(meta.chunk[row:row + n], np.arange(n))):
                raise ValueError(f"{p} does not match rows [{row}, {row + n}) of {self.meta_file}: the re-rank store "
                                 f"must follow the index's id order")
            if refine is None:
                dtype = refine_dtype or ("float16" if emb.dtype == np.float16 else "float32")
                refine = rsb_index.IndexRefine(base, store_dtype=dtype, k_factor=k_factor, device_rows=device_rows)
                refine.reserve(base.ntotal)                 # MemoryError (with the byte count) before any upload
            if dtype == "sq8" and refine._sq is None:
                held.append(emb)
                sample.append(emb[: max(0, n_train - row)])
                if row + n >= n_train:
                    refine.train_store(np.concatenate(sample))
                    for e in held:
                        refine.add_store(e)
                    held, sample = [], []
            else:
                refine.add_store(emb)
            row += n
        if refine is None or row != base.ntotal or held:
            raise ValueError(f"the embedding shards hold {row} vectors, the index {base.ntotal}")
        return refine
