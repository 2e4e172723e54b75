"""shuffle_table — the row -> rank hash shuffle (mirror of bodo.libs.array.shuffle_table,
bodo/libs/array.py:2670-2698 -> shuffle_table_py_entrypt, bodo/libs/_shuffle.cpp:1593-1655).

    out = shuffle_table(table, n_keys)     # every row lands on rank hash_to_rank(hash(key)) — same placement as the reference

Device path: one radix-partition pass (b200_shuffle_partition, csrc/shuffle.cu) groups the rows of all columns by
destination, then ONE all-to-all-v per buffer moves them (torch.distributed -> ncclSend/ncclRecv groups over NVLink;
the reference issues one MPI alltoallv per column buffer, _shuffle.cpp:661-875).  Counts are exchanged first
(mpi_comm_info's MPI_Alltoall, _shuffle.cpp:210-213).

The exchange logic (`exchange_partitioned` / `exchange_table`) is backend-agnostic torch.distributed code (the gloo tests
drive it on CPU with their own partition and bitmap-merge stand-ins); the partition step and the bitmap merge of
`shuffle_table` itself exist only as CUDA kernels (no CPU fallback in this package).
"""

from __future__ import annotations

from typing import Callable, Sequence

import numpy as np

from . import _lib
from ._lib import ffi
from .table import ArrTypes, Column, CTable, Table


def partition_device(table: Table, n_keys: int, n_pes: int, stream: int = 0, want_perm: bool = False, by_class: bool = False):
    """Run the CUDA radix partition. Returns (partitioned Table of torch tensors, send_counts[, perm tensor]).

    by_class=False places rows as the reference's shuffle_table does (b200_shuffle_partition, 4- and 8-byte keys).  by_class=True
    sends every key class to one rank (b200_shuffle_partition_classes): NA and a float NaN are one class, -0.0 equals 0.0, and
    every fixed-width key type is accepted, 1- and 2-byte integers and bool included."""
    import torch

    L = _lib.lib()
    _lib.require_gpu()
    dev_i = table.device
    if dev_i < 0:
        raise _lib.B200Error("shuffle_table: the table must be device resident (stage host batches with torch first)")
    dev = torch.device("cuda", dev_i)
    n = table.n_rows
    out_cols = []
    for c in table.columns:
        npdt = np.dtype(_np_dtype(c))
        data = torch.empty(n, dtype=getattr(torch, str(npdt)), device=dev)
        validity = None
        if c.validity is not None:
            validity = torch.zeros((n + 7) // 8 + n_pes + 8, dtype=torch.uint8, device=dev)
        out_cols.append(Column(data, validity, c.c_type, c.arr_type, n))
    out = Table(out_cols, list(table.names))
    cin, cout = CTable(table), CTable(out)
    counts = ffi.new("int64_t[]", n_pes)
    if by_class:
        perm = torch.empty(n, dtype=torch.int64, device=dev) if want_perm else None
        _lib.check(L.b200_shuffle_partition_classes(cin.ptr, n_keys, n_pes, cout.ptr, counts,
                                                    ffi.cast("int64_t*", perm.data_ptr()) if want_perm else ffi.NULL,
                                                    ffi.cast("void*", stream)), "shuffle partition by key class")
        return (out, [int(counts[i]) for i in range(n_pes)]) + ((perm,) if want_perm else ())
    if want_perm:
        perm = torch.empty(n, dtype=torch.int64, device=dev)
        _lib.check(L.b200_shuffle_partition_perm(cin.ptr, n_keys, n_pes, cout.ptr, counts, ffi.cast("int64_t*", perm.data_ptr()),
                                                 ffi.cast("void*", stream)), "shuffle partition")
        return out, [int(counts[i]) for i in range(n_pes)], perm
    _lib.check(L.b200_shuffle_partition(cin.ptr, n_keys, n_pes, cout.ptr, counts, ffi.cast("void*", stream)), "shuffle partition")
    return out, [int(counts[i]) for i in range(n_pes)]


def hash_keys_table(table: Table, n_keys: int = 1, n_pes: int = 1, stream: int = 0):
    """hash_keys_table(table, n_keys, SEED_HASH_PARTITION) on the device (b200_hash_keys_table): returns (row hashes as an
    int64-viewable uint32 tensor, destination ranks) for a device-resident table whose first n_keys columns are the keys."""
    import torch

    L = _lib.lib()
    _lib.require_gpu()
    dev = torch.device("cuda", table.device)
    n = table.n_rows
    hashes = torch.empty(n, dtype=torch.int32, device=dev)  # uint32 bit patterns
    dest = torch.empty(n, dtype=torch.int32, device=dev)
    ct = CTable(table)
    _lib.check(L.b200_hash_keys_table(ct.ptr, n_keys, n_pes, ffi.cast("int32_t*", dest.data_ptr()), ffi.cast("uint32_t*", hashes.data_ptr()),
                                      ffi.cast("void*", stream)), "hash_keys_table")
    return hashes, dest


def _np_dtype(c: Column):
    from .table import np_dtype_of

    return np_dtype_of(c.c_type)


def exchange_partitioned(buffers: Sequence, send_counts: Sequence[int], validity_buffers: Sequence = (), group=None):
    """All-to-all-v of destination-grouped column buffers.

    buffers: torch tensors (any device torch.distributed's backend supports), each with send_counts.sum() rows grouped
    by destination rank.  validity_buffers: per column either None or a uint8 tensor holding the per-destination bitmaps
    back to back (segment d has ceil(send_counts[d]/8) bytes).  Returns (recv_buffers, recv_validity, recv_counts).
    Mirrors mpi_comm_info (counts -> displacements) + bodo_alltoallv (bodo/libs/_distributed.h:1285-1385).
    """
    import torch
    import torch.distributed as dist

    n_pes = dist.get_world_size(group)
    assert len(send_counts) == n_pes
    dev = buffers[0].device if buffers else torch.device("cpu")
    sc = torch.tensor(list(send_counts), dtype=torch.int64, device=dev)
    rc = torch.empty_like(sc)
    dist.all_to_all_single(rc, sc, group=group)
    recv_counts = [int(x) for x in rc.cpu().tolist()]
    n_send, n_recv = int(sum(send_counts)), int(sum(recv_counts))
    recv_buffers = []
    for b in buffers:
        r = torch.empty((n_recv,) + tuple(b.shape[1:]), dtype=b.dtype, device=b.device)
        dist.all_to_all_single(r, b[:n_send].contiguous(), output_split_sizes=recv_counts, input_split_sizes=list(send_counts), group=group)
        recv_buffers.append(r)
    recv_validity = []
    sbytes = [(c + 7) // 8 for c in send_counts]
    rbytes = [(c + 7) // 8 for c in recv_counts]
    for v in validity_buffers:
        if v is None:
            recv_validity.append(None)
            continue
        r = torch.empty(sum(rbytes), dtype=torch.uint8, device=v.device)
        dist.all_to_all_single(r, v[: sum(sbytes)].contiguous(), output_split_sizes=rbytes, input_split_sizes=sbytes, group=group)
        recv_validity.append(r)
    return recv_buffers, recv_validity, recv_counts


def merge_segment_bitmaps(bitmap, counts: Sequence[int]):
    """Concatenate per-source byte-padded bitmaps (one per sending rank) into one contiguous Arrow bitmap on the device
    (b200_merge_segment_bitmaps, csrc/shuffle.cu)."""
    import torch

    if not bitmap.is_cuda:
        raise _lib.B200Error("merge_segment_bitmaps: device tensors only (this package has no CPU path)")
    n = int(sum(counts))
    out = torch.zeros(((n + 31) // 32 + 2) * 4, dtype=torch.uint8, device=bitmap.device)
    if n == 0:  # a rank that receives no row gets an empty segment buffer, whose null pointer the entry point refuses
        return out
    cnt = ffi.new("int64_t[]", [int(c) for c in counts])
    _lib.check(_lib.lib().b200_merge_segment_bitmaps(ffi.cast("uint8_t*", bitmap.data_ptr()), cnt, len(counts),
                                                     ffi.cast("uint8_t*", out.data_ptr()), bitmap.device.index,
                                                     ffi.cast("void*", torch.cuda.current_stream(bitmap.device).cuda_stream)),
               "merge segment bitmaps")
    return out


def with_schema_validity(table: Table) -> Table:
    """Give every NULLABLE column a validity bitmap (all ones when the local data has no nulls).  Whether a bitmap
    travels must follow from the SCHEMA, not from the local data: Arrow drops the bitmap of a chunk without nulls, and
    ranks that disagreed on the number of collectives would hang or pair the wrong buffers."""
    import torch

    cols = []
    for c in table.columns:
        if c.arr_type == ArrTypes.NULLABLE_INT_BOOL and c.validity is None:
            nbytes = (c.length + 7) // 8 + 8
            if hasattr(c.data, "is_cuda"):
                v = torch.full((nbytes,), 255, dtype=torch.uint8, device=c.data.device)
            else:
                v = np.full(nbytes, 255, dtype=np.uint8)
            c = Column(c.data, v, c.c_type, c.arr_type, c.length)
        cols.append(c)
    return Table(cols, list(table.names))


def exchange_table(part: Table, send_counts: Sequence[int], group=None, merge_bitmaps: Callable = merge_segment_bitmaps) -> Table:
    """All-to-all-v of a destination-grouped table (output of the partition step) and reassembly of the received
    columns; `merge_bitmaps(recv_bitmap_segments, recv_counts)` turns the per-source bitmap segments into one bitmap."""
    bufs = [c.data for c in part.columns]
    vbufs = [c.validity for c in part.columns]
    rbufs, rvalid, recv_counts = exchange_partitioned(bufs, send_counts, vbufs, group=group)
    cols = []
    n_recv = sum(recv_counts)
    for c, rb, rv in zip(part.columns, rbufs, rvalid):
        v = merge_bitmaps(rv, recv_counts) if rv is not None else None
        cols.append(Column(rb, v, c.c_type, c.arr_type if v is None else ArrTypes.NULLABLE_INT_BOOL, n_recv))
    return Table(cols, list(part.names))


def shuffle_table(table: Table, n_keys: int = 1, parallel: bool = True, keep_comm_info: int = 0, *, group=None, stream: int = 0) -> Table:
    """Mirror of bodo.libs.array.shuffle_table(table, n_keys, _is_parallel, keep_comm_info).

    Keys are the first n_keys columns (the reference's convention).  Returns this rank's rows after the shuffle
    (order: by source rank, input order within a source — the same as MPI alltoallv of the stable send arrays).
    """
    import torch
    import torch.distributed as dist

    if not parallel or not dist.is_initialized() or dist.get_world_size(group) == 1:
        return table
    n_pes = dist.get_world_size(group)
    part, send_counts = partition_device(with_schema_validity(table), n_keys, n_pes, stream)
    torch.cuda.current_stream().synchronize()
    return exchange_table(part, send_counts, group)
