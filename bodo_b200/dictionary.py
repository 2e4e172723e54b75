"""Dictionary-encoded string key columns: the host side of the reference's DictionaryBuilder
(bodo/libs/_dict_builder.{h,cpp}; used by the streaming groupby / join for DICT key columns,
bodo/libs/streaming/_groupby.cpp:3647-3706 UnifyBuildTableDictionaryArrays).

Every batch arrives with its own dictionary (Arrow DictionaryArray, or a plain string column that is dictionary-encoded per
batch).  The builder keeps ONE growing dictionary per key column; a batch's dictionary is matched against it on the host
(dictionaries are small: distinct strings, not rows) and the batch's index column is rewritten to global ids on the device
(b200_remap_i32: the `transpose` step of UnifyDictionaryArray).  The operators then see an ordinary int32 key column; output
ids are decoded back through the same dictionary.  NA stays NA: a null index and an index to a null dictionary entry both
become a NA row (validity bitmap of the id column).
"""

from __future__ import annotations

import numpy as np

from . import _lib
from ._lib import ffi
from .table import ArrTypes, Column, CTypes


class DictionaryBuilder:
    def __init__(self):
        self.values: list = []      # global id -> string
        self.index: dict = {}       # string -> global id
        self._cache_key = None
        self._cache_map = None

    def _global_ids(self, batch_dictionary) -> np.ndarray:
        """global ids of a batch dictionary (pyarrow string array); new strings are appended (InsertIfNotExists)."""
        ids = np.empty(len(batch_dictionary), dtype=np.int32)
        for j, s in enumerate(batch_dictionary.to_pylist()):
            if s is None:  # null entries get no global id: the rows that use them are NA (unify)
                ids[j] = 0
                continue
            g = self.index.get(s)
            if g is None:
                g = len(self.values)
                self.index[s] = g
                self.values.append(s)
            ids[j] = g
        return ids

    def unify(self, arr, device: int, stream: int = 0) -> Column:
        """pyarrow string / large_string / dictionary<string> array -> device Column of global ids (INT32, nullable)."""
        import pyarrow as pa
        import torch

        if isinstance(arr, pa.ChunkedArray):
            if pa.types.is_dictionary(arr.type) and arr.num_chunks > 1 and any(c.dictionary.null_count for c in arr.chunks):
                # Arrow cannot concatenate dictionaries with null entries: decode the chunks (those entries become null rows)
                arr = pa.chunked_array([c.cast(arr.type.value_type) for c in arr.chunks])
            arr = arr.combine_chunks()
        if not pa.types.is_dictionary(arr.type):
            arr = arr.dictionary_encode()
        idx = arr.indices.cast(pa.int32())
        gmap = self._global_ids(arr.dictionary)
        n = len(idx)
        dev = torch.device("cuda", device)
        bufs = idx.buffers()
        off = idx.offset
        host_idx = np.frombuffer(bufs[1], dtype=np.int32)[off: off + n] if n else np.empty(0, np.int32)
        d_idx = torch.from_numpy(np.ascontiguousarray(host_idx)).to(dev)
        validity = None
        mask = np.asarray(idx.is_valid())
        if arr.dictionary.null_count > 0:  # a row whose dictionary entry is null is NA too
            mask = mask & np.asarray(arr.dictionary.is_valid())[np.where(mask, host_idx, 0)]
        if not mask.all():
            vb = np.packbits(mask, bitorder="little")
            pad = np.zeros((len(vb) + 15) // 8 * 8, dtype=np.uint8)
            pad[: len(vb)] = vb
            validity = torch.from_numpy(pad).to(dev)
        d_map = torch.from_numpy(gmap if len(gmap) else np.zeros(1, np.int32)).to(dev)
        out = torch.empty(n, dtype=torch.int32, device=dev)
        _lib.check(_lib.lib().b200_remap_i32(ffi.cast("int32_t*", d_idx.data_ptr()), ffi.cast("uint8_t*", validity.data_ptr() if validity is not None else 0), n,
                                             ffi.cast("int32_t*", d_map.data_ptr()), len(gmap), ffi.cast("int32_t*", out.data_ptr()), device,
                                             ffi.cast("void*", stream)), "dictionary unification (remap)")
        torch.cuda.current_stream(dev).synchronize() if stream == 0 else None
        return Column(out, validity, CTypes.INT32, ArrTypes.NULLABLE_INT_BOOL, n)

    def decode(self, ids: np.ndarray, valid_mask=None):
        """global ids -> numpy object array of strings (None where NA)."""
        vals = np.array(self.values + [None], dtype=object)
        ids = np.asarray(ids, dtype=np.int64)
        out = vals[np.where((ids >= 0) & (ids < len(self.values)), ids, len(self.values))]
        if valid_mask is not None:
            out = out.copy()
            out[~np.asarray(valid_mask)] = None
        return out
