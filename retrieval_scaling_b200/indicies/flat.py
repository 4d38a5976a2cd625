"""FlatIndexer -- exact inner-product index (reference `src/indicies/flat.py:18-141`, faiss.IndexFlatIP)."""
from __future__ import annotations

from .. import index as rsb_index
from ._common import BaseIndexer


class FlatIndexer(BaseIndexer):
    index_kind = "Flat"

    def __init__(self, embed_paths=None, index_path=None, meta_file=None, passage_dir=None,
                 pos_map_save_path=None, dimension=768, storage_dtype=None, device_rows=None):
        super().__init__(embed_paths, index_path, meta_file, passage_dir, pos_map_save_path, dimension,
                         storage_dtype=storage_dtype, device_rows=device_rows)

    def _new_index(self):
        return rsb_index.IndexFlatIP(self.dimension, dtype=self.storage_dtype or "float32", device_rows=self.device_rows)
