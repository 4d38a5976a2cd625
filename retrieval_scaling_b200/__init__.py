"""retrieval_scaling_b200 -- H100-native (sm_90a) implementation of the query -> top-k dense-retrieval hot
path of RulinShao/retrieval-scaling: Contriever/BERT query encoding and Flat / IVF-Flat / IVF-PQ
inner-product search behind the reference's `Indexer(cfg).search(query_embs, k)` surface.

Importing the package does not need a GPU; constructing an index or an encoder does (there is no CPU path).
"""
__version__ = "0.1.0"

from . import _lib  # noqa: F401  (ctypes signatures; the shared library is loaded lazily)


def _lazy():
    from . import index as _index
    return _index


def __getattr__(name):
    if name in ("IndexFlatIP", "IndexIVFFlat", "IndexIVFPQ", "IndexIVFScalarQuantizer", "IndexRefine", "read_index", "write_index", "merge_topk", "knn_ip"):
        return getattr(_lazy(), name)
    raise AttributeError(name)
