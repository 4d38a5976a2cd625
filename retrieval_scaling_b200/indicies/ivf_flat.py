"""IVFFlatIndexer -- inverted file over raw fp32 vectors, inner product (reference
`src/indicies/ivf_flat.py:35-227`: IndexIVFFlat(IndexFlatIP(d), d, ncentroids, METRIC_INNER_PRODUCT),
`index.nprobe = probe`).  storage_dtype "sq8" builds faiss' IVFn,SQ8 (IndexIVFScalarQuantizer, by_residual) instead.
list_device_rows tiers the lists between device and pinned host memory (see BaseIndexer._add_keys)."""
from __future__ import annotations

from .. import index as rsb_index
from ._common import BaseIndexer


class IVFFlatIndexer(BaseIndexer):
    index_kind = "IVFFlat"

    def __init__(self, embed_paths, index_path, meta_file, trained_index_path, passage_dir=None,
                 pos_map_save_path=None, sample_train_size=1000000, prev_index_path=None, dimension=768,
                 dtype=None, ncentroids=4096, probe=2048, num_keys_to_add_at_a_time=1000000,
                 DSTORE_SIZE_BATCH=51200000, storage_dtype=None, list_device_rows=None):
        self.ncentroids = int(ncentroids)
        self.prev_index_path = prev_index_path
        self.num_keys_to_add_at_a_time = num_keys_to_add_at_a_time
        super().__init__(embed_paths, index_path, meta_file, passage_dir, pos_map_save_path, dimension,
                         trained_index_path=prev_index_path or trained_index_path,
                         sample_train_size=sample_train_size, probe=probe, storage_dtype=storage_dtype,
                         list_device_rows=list_device_rows)

    def _new_index(self):
        if self.storage_dtype == "sq8":         # faiss index_factory(d, "IVFn,SQ8")
            return rsb_index.IndexIVFScalarQuantizer(self.dimension, self.ncentroids, by_residual=True,
                                                     list_device_rows=self.list_device_rows)
        return rsb_index.IndexIVFFlat(self.dimension, self.ncentroids, dtype=self.storage_dtype or "float32",
                                      list_device_rows=self.list_device_rows)
