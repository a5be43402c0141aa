"""sdbgpu -- H100-native KNN / HNSW / graph-expansion engine behind SurrealDB's operator surface.

Python here is only the host-side mirror of the reference's operator interface (KnnTopK, KnnScan /
HnswIndex.knn_search, GraphEdgeScan) on top of the C ABI in include/sdbgpu.h; all compute is
hand-written sm_90a CUDA in surrealdb_b200/csrc.
"""
from ._lib import SdbError, SO_PATH  # noqa: F401
from .engine import Context, VectorColumn, pack_row_filter  # noqa: F401
from .operators import (Distance, Filter, KnnBruteForceLegacy, KnnContext, KnnScan, KnnTopK, SortTopK,  # noqa: F401
                        TableScan, Union)
from .graph import CsrGraph, GraphEdgeScan, GraphStore  # noqa: F401
from .hnsw import HnswIndex  # noqa: F401

__version__ = "0.1.0"
