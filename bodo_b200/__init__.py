"""bodo_b200 — CUDA-native (H100) streaming hash groupby / hash join / row->rank shuffle behind Bodo's operator API.

The compute path is libbodo_b200.so (hand-written sm_90a CUDA, include/bodo_b200.h); this package is the
thin Python host layer that mirrors the reference's operator interface (bodo/libs/streaming/groupby.py,
join.py, bodo/libs/array.py shuffle_table).  There is no CPU fallback.
"""

from ._lib import B200Error  # noqa: F401
from .table import ArrTypes, Column, CTypes, DeviceArray, Table  # noqa: F401

__all__ = ["B200Error", "Table", "Column", "DeviceArray", "CTypes", "ArrTypes"]
