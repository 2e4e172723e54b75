"""Columnar batches crossing the C ABI: the Python face of b200_table / b200_column.

Mirrors the reference's table_info/array_info data model (bodo/libs/_bodo_common.h:927,1819) restricted to
the fixed-width column kinds the hot path handles: NUMPY (no nulls) and NULLABLE_INT_BOOL (Arrow validity
bitmap).  A column's buffers may live in host memory (numpy / pandas / pyarrow) or on a CUDA device
(torch tensors, or library-owned DeviceArray views); nothing here computes on the data.
"""

from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any, Sequence

import numpy as np

from . import _lib
from ._lib import ffi


class CTypes:
    """Bodo_CTypes codes (reference: bodo/libs/_bodo_common.h:331-359)."""

    INT8, UINT8, INT32, UINT32, INT64, FLOAT32, FLOAT64, UINT64, INT16, UINT16 = range(10)
    STRING, BOOL, DECIMAL, DATE, TIME, DATETIME, TIMEDELTA = 10, 11, 12, 13, 14, 15, 16


class ArrTypes:
    """bodo_array_type codes (reference: bodo/libs/_bodo_common.h:515-532)."""

    NUMPY = 0
    NULLABLE_INT_BOOL = 2


_NP_TO_CT = {
    np.dtype("int8"): CTypes.INT8, np.dtype("uint8"): CTypes.UINT8, np.dtype("int16"): CTypes.INT16,
    np.dtype("uint16"): CTypes.UINT16, np.dtype("int32"): CTypes.INT32, np.dtype("uint32"): CTypes.UINT32,
    np.dtype("int64"): CTypes.INT64, np.dtype("uint64"): CTypes.UINT64, np.dtype("float32"): CTypes.FLOAT32,
    np.dtype("float64"): CTypes.FLOAT64, np.dtype("bool"): CTypes.BOOL,
}
_CT_TO_NP = {v: k for k, v in _NP_TO_CT.items()}
_CT_TO_NP[CTypes.DATETIME] = np.dtype("int64")
_CT_TO_NP[CTypes.TIMEDELTA] = np.dtype("int64")
_CT_TO_NP[CTypes.DATE] = np.dtype("int32")


def ctype_of(np_dtype) -> int:
    dt = np.dtype(np_dtype)
    if dt.kind == "M":
        return CTypes.DATETIME
    if dt.kind == "m":
        return CTypes.TIMEDELTA
    try:
        return _NP_TO_CT[dt]
    except KeyError:
        raise TypeError(f"bodo_b200: unsupported column dtype {dt} (fixed-width numeric columns only)") from None


def np_dtype_of(ctype: int) -> np.dtype:
    return _CT_TO_NP[ctype]


class DeviceArray:
    """A typed view of device memory (owned by a library state object or by a torch tensor).

    Exposes __cuda_array_interface__ so torch.as_tensor(x, device="cuda") wraps it without a copy.
    `owner` keeps whatever owns the memory alive.
    """

    def __init__(self, ptr: int, length: int, dtype, device: int, owner: Any = None):
        self.ptr = int(ptr)
        self.length = int(length)
        self.dtype = np.dtype(dtype)
        self.device = int(device)
        self.owner = owner

    @property
    def nbytes(self) -> int:
        return self.length * self.dtype.itemsize

    @property
    def __cuda_array_interface__(self):
        return {"shape": (self.length,), "typestr": self.dtype.str, "data": (self.ptr if self.length else 0, False),
                "version": 2, "strides": None}

    def to_numpy(self, stream: int = 0) -> np.ndarray:
        out = np.empty(self.length, dtype=self.dtype)
        if self.length:
            L = _lib.lib()
            _lib.check(L.b200_memcpy_d2h(ffi.cast("void*", out.ctypes.data), ffi.cast("void*", self.ptr), self.nbytes,
                                         ffi.cast("void*", stream)), "d2h copy")
        return out

    def __len__(self):
        return self.length


def _is_torch_tensor(x) -> bool:
    return type(x).__module__.startswith("torch") and hasattr(x, "data_ptr")


@dataclass
class Column:
    """One column: `data` is a numpy array (host), a torch CUDA tensor, or a DeviceArray (device)."""

    data: Any
    validity: Any = None  # Arrow validity bitmap (uint8 numpy array / uint8 CUDA tensor / DeviceArray) or None
    c_type: int = -1
    arr_type: int = ArrTypes.NUMPY
    length: int = -1

    def __post_init__(self):
        if self.length < 0:
            self.length = len(self.data)
        if isinstance(self.data, np.ndarray) and self.data.dtype.kind in "Mm":
            # temporal numpy buffers: nanosecond int64 storage, whatever unit they arrive in
            kind = self.data.dtype.kind
            if self.c_type < 0:
                self.c_type = CTypes.DATETIME if kind == "M" else CTypes.TIMEDELTA
            self.data = np.ascontiguousarray(self.data.astype("datetime64[ns]" if kind == "M" else "timedelta64[ns]", copy=False)).view("int64")
        if self.c_type < 0:
            if isinstance(self.data, np.ndarray):
                self.c_type = ctype_of(self.data.dtype)
            elif isinstance(self.data, DeviceArray):
                self.c_type = ctype_of(self.data.dtype)
            elif _is_torch_tensor(self.data):
                self.c_type = ctype_of(str(self.data.dtype).replace("torch.", ""))
            else:
                raise TypeError(f"unsupported column buffer {type(self.data)}")
        if self.validity is not None and self.arr_type == ArrTypes.NUMPY:
            self.arr_type = ArrTypes.NULLABLE_INT_BOOL

    @property
    def device(self) -> int:
        d = self.data
        if isinstance(d, np.ndarray):
            return -1
        if isinstance(d, DeviceArray):
            return d.device
        if _is_torch_tensor(d):
            return d.device.index if d.is_cuda else -1
        raise TypeError(type(d))

    def data_ptr(self) -> int:
        d = self.data
        if isinstance(d, np.ndarray):
            return d.ctypes.data
        if isinstance(d, DeviceArray):
            return d.ptr
        return d.data_ptr()

    def validity_ptr(self) -> int:
        v = self.validity
        if v is None:
            return 0
        if isinstance(v, np.ndarray):
            return v.ctypes.data
        if isinstance(v, DeviceArray):
            return v.ptr
        return v.data_ptr()

    # ---- host materialisation (for results / tests) ----
    def values_numpy(self, stream: int = 0) -> np.ndarray:
        d = self.data
        if isinstance(d, np.ndarray):
            return d[: self.length]
        if isinstance(d, DeviceArray):
            return d.to_numpy(stream)[: self.length]
        return d.cpu().numpy()[: self.length]

    def valid_mask_numpy(self, stream: int = 0):
        """bool array (True = valid) or None when the column has no validity bitmap."""
        v = self.validity
        if v is None:
            return None
        if isinstance(v, DeviceArray):
            v = v.to_numpy(stream)
        elif not isinstance(v, np.ndarray):
            v = v.cpu().numpy()
        bits = np.unpackbits(v.view(np.uint8), bitorder="little")[: self.length]
        return bits.astype(bool)


@dataclass
class Table:
    columns: list[Column]
    names: list[str] = field(default_factory=list)

    def __post_init__(self):
        if not self.names:
            self.names = [f"c{i}" for i in range(len(self.columns))]
        n = {c.length for c in self.columns}
        if len(n) > 1:
            raise ValueError(f"columns have different lengths: {sorted(n)}")

    @property
    def n_rows(self) -> int:
        return self.columns[0].length if self.columns else 0

    @property
    def n_cols(self) -> int:
        return len(self.columns)

    @property
    def device(self) -> int:
        devs = {c.device for c in self.columns}
        if len(devs) > 1:
            raise ValueError(f"columns of one batch live in different memories: {sorted(devs)}")
        return devs.pop() if devs else -1

    def select(self, idx: Sequence[int]) -> "Table":
        return Table([self.columns[i] for i in idx], [self.names[i] for i in idx])

    def slice(self, start: int, stop: int) -> "Table":
        """Row slice of a HOST table (streaming tests feed batch_size-row slices, as the reference's
        table_local_filter loops do, bodo/tests/test_streaming/test_groupby.py:58-66)."""
        cols = []
        stop = min(stop, self.n_rows)
        start = min(start, stop)
        for c in self.columns:
            if not isinstance(c.data, np.ndarray):
                raise TypeError("Table.slice is only provided for host tables")
            v = None
            if c.validity is not None:
                mask = np.unpackbits(c.validity, bitorder="little")[: c.length][start:stop]
                v = np.packbits(mask, bitorder="little")
            cols.append(Column(np.ascontiguousarray(c.data[start:stop]), v, c.c_type, c.arr_type, stop - start))
        return Table(cols, list(self.names))

    # ---- conversions ----
    @staticmethod
    def from_pandas(df) -> "Table":
        import pandas as pd

        cols, names = [], []
        for name in df.columns:
            s = df[name]
            cols.append(column_from_pandas(s))
            names.append(str(name))
        return Table(cols, names)

    @staticmethod
    def from_arrow(tbl) -> "Table":
        """pyarrow Table / RecordBatch -> host Table (zero-copy views of the Arrow buffers)."""
        import pyarrow as pa

        if isinstance(tbl, pa.Table):
            tbl = tbl.combine_chunks()
            arrays = [c.chunk(0) if c.num_chunks else pa.array([], type=c.type) for c in tbl.columns]
        else:
            arrays = list(tbl.columns)
        cols = [column_from_arrow(a) for a in arrays]
        return Table(cols, list(tbl.schema.names))

    def to_pandas(self, stream: int = 0):
        import pandas as pd

        out = {}
        for name, c in zip(self.names, self.columns):
            out[name] = column_to_pandas(c, stream)
        return pd.DataFrame(out)


def column_from_pandas(s) -> Column:
    """pandas Series -> Column.  Nullable extension dtypes (Int64, Float64, boolean) become
    NULLABLE_INT_BOOL columns with an Arrow validity bitmap, numpy dtypes become NUMPY columns — the same
    split bodo::Schema::FromArrowSchema makes for in-memory pandas input (SURVEY.md §8c)."""
    import pandas as pd

    dt = s.dtype
    if isinstance(dt, pd.api.extensions.ExtensionDtype) and hasattr(s.array, "_mask"):
        arr = s.array
        data = np.ascontiguousarray(arr._data)
        mask = np.asarray(arr._mask)
        validity = np.packbits(~mask, bitorder="little")
        return Column(data, validity, ctype_of(data.dtype), ArrTypes.NULLABLE_INT_BOOL)
    if isinstance(dt, pd.ArrowDtype):
        import pyarrow as pa

        return column_from_arrow(pa.chunked_array(s.array._pa_array).combine_chunks())
    a = s.to_numpy()
    if a.dtype.kind in "Mm":
        # DATETIME / TIMEDELTA columns are int64 NANOSECONDS (Bodo_CTypes, _bodo_common.h:331-359): pandas >= 3 hands out
        # datetime64[us] (and [s]/[ms] on request), so the unit is normalised before the storage is reinterpreted
        # NaT is NA (the reference converts every pandas slice to Arrow first, read_pandas.h, and Arrow makes NaT null)
        ct = CTypes.DATETIME if a.dtype.kind == "M" else CTypes.TIMEDELTA
        a = a.astype("datetime64[ns]" if a.dtype.kind == "M" else "timedelta64[ns]", copy=False)
        nat = np.isnat(a)
        if nat.any():
            return Column(np.ascontiguousarray(a.view("int64")), np.packbits(~nat, bitorder="little"), ct, ArrTypes.NULLABLE_INT_BOOL)
        return Column(np.ascontiguousarray(a.view("int64")), None, ct)
    if a.dtype == object:
        raise TypeError(f"bodo_b200: column '{s.name}' has object dtype (strings are a 'next' row, SURVEY.md §8f)")
    return Column(np.ascontiguousarray(a), None, ctype_of(a.dtype))


def column_from_arrow(a) -> Column:
    import pyarrow as pa

    if isinstance(a, pa.ChunkedArray):
        a = a.combine_chunks()
    t = a.type
    # temporal columns travel as their integer storage with the reference's dtype code (Bodo_CTypes DATE = int32 days,
    # DATETIME / TIMEDELTA = int64 nanoseconds, bodo/libs/_bodo_common.h:331-359); other units are brought to ns first
    c_type = None
    if pa.types.is_date32(t):
        a, c_type = a.view(pa.int32()), CTypes.DATE
    elif pa.types.is_timestamp(t) or pa.types.is_duration(t):
        is_ts = pa.types.is_timestamp(t)
        if t.unit != "ns":
            a = a.cast(pa.timestamp("ns", tz=t.tz) if is_ts else pa.duration("ns"))
        a, c_type = a.view(pa.int64()), (CTypes.DATETIME if is_ts else CTypes.TIMEDELTA)
    elif pa.types.is_date64(t):
        a, c_type = a.cast(pa.timestamp("ns")).view(pa.int64()), CTypes.DATETIME
    t = a.type
    if not (pa.types.is_integer(t) or pa.types.is_floating(t)):
        raise TypeError(f"bodo_b200: unsupported Arrow type {t} (fixed-width numeric, date and timestamp columns only; "
                        "strings are a 'next' row, SURVEY.md §8f)")
    np_dt = np.dtype(t.to_pandas_dtype())
    bufs = a.buffers()
    n = len(a)
    if a.offset % 8 != 0:
        a = pa.concat_arrays([a])  # re-base so bitmap slicing stays byte aligned
        bufs = a.buffers()
    off = a.offset
    data = np.frombuffer(bufs[1], dtype=np_dt)[off : off + n] if n else np.empty(0, np_dt)
    validity = None
    if bufs[0] is not None and a.null_count > 0:
        validity = np.frombuffer(bufs[0], dtype=np.uint8)[off // 8 : off // 8 + (n + 7) // 8]
    arr_type = ArrTypes.NULLABLE_INT_BOOL  # Arrow columns are nullable by construction
    return Column(np.ascontiguousarray(data), validity, c_type if c_type is not None else ctype_of(np_dt), arr_type, n)


def column_to_pandas(c: Column, stream: int = 0):
    import pandas as pd

    vals = c.values_numpy(stream)
    if c.c_type == CTypes.DATETIME:
        vals = vals.view("datetime64[ns]")
    elif c.c_type == CTypes.TIMEDELTA:
        vals = vals.view("timedelta64[ns]")
    elif c.c_type == CTypes.DATE:
        vals = vals.astype("int64").view("datetime64[D]")
    mask = c.valid_mask_numpy(stream)
    if vals.dtype.kind in "Mm" and mask is not None and not mask.all():
        vals = vals.copy()
        vals[~mask] = np.datetime64("NaT") if vals.dtype.kind == "M" else np.timedelta64("NaT")
    if c.arr_type == ArrTypes.NULLABLE_INT_BOOL and c.c_type == CTypes.BOOL:
        m = ~mask if mask is not None else np.zeros(len(vals), dtype=bool)
        return pd.array(pd.arrays.BooleanArray(vals.astype(bool), m), dtype="boolean")
    if c.arr_type == ArrTypes.NULLABLE_INT_BOOL and vals.dtype.kind in "iuf":
        name = {"i": "Int", "u": "UInt", "f": "Float"}[vals.dtype.kind] + str(vals.dtype.itemsize * 8)
        m = ~mask if mask is not None else np.zeros(len(vals), dtype=bool)
        if vals.dtype.kind == "f":
            return pd.array(pd.arrays.FloatingArray(vals.copy(), m), dtype=name)
        return pd.array(pd.arrays.IntegerArray(vals.copy(), m), dtype=name)
    return vals


class CTable:
    """cffi b200_table built from a Table; keeps every referenced buffer alive."""

    def __init__(self, table: Table):
        self.table = table
        n = table.n_cols
        self.cols = ffi.new("b200_column[]", max(n, 1))
        for i, c in enumerate(table.columns):
            self.cols[i].data = ffi.cast("void*", c.data_ptr())
            self.cols[i].validity = ffi.cast("uint8_t*", c.validity_ptr())
            self.cols[i].length = c.length
            self.cols[i].c_type = c.c_type
            self.cols[i].arr_type = c.arr_type
        self.ctab = ffi.new("b200_table*")
        self.ctab.n_rows = table.n_rows
        self.ctab.n_cols = n
        self.ctab.device = table.device
        self.ctab.cols = self.cols

    @property
    def ptr(self):
        return self.ctab


def table_from_ctable(ctab, n_cols: int, names: Sequence[str], owner: Any) -> Table:
    """Wrap the device columns a produce/probe call returned (library-owned memory) as a Table."""
    cols = []
    dev = ctab.device
    for i in range(n_cols):
        cc = ctab.cols[i]
        dt = np_dtype_of(cc.c_type)
        data = DeviceArray(int(ffi.cast("uintptr_t", cc.data)), cc.length, dt, dev, owner)
        validity = None
        if cc.validity != ffi.NULL:
            validity = DeviceArray(int(ffi.cast("uintptr_t", cc.validity)), (cc.length + 7) // 8, np.uint8, dev, owner)
        cols.append(Column(data, validity, cc.c_type, cc.arr_type, cc.length))
    return Table(cols, list(names))


def to_device(table: Table, device: int) -> Table:
    """Host batch -> device batch (torch tensors); device batches pass through."""
    import torch

    if table.device >= 0:
        return table
    dev = torch.device("cuda", device)
    cols = []
    for c in table.columns:
        d = torch.from_numpy(np.ascontiguousarray(c.data)).to(dev, non_blocking=False)
        v = None
        if c.validity is not None:
            vb = np.zeros((len(c.validity) + 7) // 8 * 8 + 8, dtype=np.uint8)
            vb[: len(c.validity)] = c.validity
            v = torch.from_numpy(vb).to(dev)
        cols.append(Column(d, v, c.c_type, c.arr_type, c.length))
    return Table(cols, list(table.names))
