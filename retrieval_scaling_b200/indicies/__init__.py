"""Drop-in mirror of the reference's `src/indicies` package (same class names, constructor arguments, return
types and on-disk artefact names), backed by the GPU index objects in `retrieval_scaling_b200.index`."""
from .base import Indexer  # noqa: F401
from .flat import FlatIndexer  # noqa: F401
from .ivf_flat import IVFFlatIndexer  # noqa: F401
from .ivf_pq import IVFPQIndexer  # noqa: F401
