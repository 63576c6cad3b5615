"""Python plumbing above the C ABI: device memory and streams come from PyTorch, every compute call
goes through libytgpu.so (include/ytgpu.h).  No CPU fallback — without a CUDA device GpuContext
raises.

Buffers may be numpy arrays (HOST memory flavour of the ABI: the library stages H2D/D2H itself) or
CUDA torch tensors (DEVICE flavour: zero-copy).
"""
from __future__ import annotations

import ctypes as C
import weakref

import numpy as np

from . import capi
from .rowset import VALUE_DTYPE, EValueType, Rowset

try:  # torch is plumbing only
    import torch
except Exception:  # pragma: no cover
    torch = None


def _is_tensor(x) -> bool:
    return torch is not None and isinstance(x, torch.Tensor)


def _ptr_mem(x):
    """-> (pointer, mem) for a numpy array (host) or a CUDA tensor (device)."""
    if x is None:
        return None, capi.MEM_HOST
    if _is_tensor(x):
        if not x.is_cuda:
            raise ValueError("torch tensors passed to ytgpu must live on a CUDA device")
        if not x.is_contiguous():
            raise ValueError("tensor must be contiguous")
        return x.data_ptr(), capi.MEM_DEVICE
    a = x
    if not a.flags["C_CONTIGUOUS"]:
        raise ValueError("array must be C-contiguous")
    return a.ctypes.data, capi.MEM_HOST


def _string_column(heap, starts, lengths, nulls=None) -> capi.StringColumn:
    """ytgpu_string_column over a heap of bytes, 8-byte starts, 4-byte lengths and a 1-byte null map (or None), all numpy
    arrays or all CUDA tensors."""
    def check(x, what, size):
        if _is_tensor(x):
            ok = x.dim() == 1 and x.element_size() == size and not x.dtype.is_floating_point and x.dtype != torch.bool
        else:
            ok = isinstance(x, np.ndarray) and x.ndim == 1 and x.dtype.itemsize == size and x.dtype.kind in "iu"
        if not ok:
            raise ValueError(f"string column {what} must be a 1-D array of {size}-byte integers")
        return _ptr_mem(x)
    hp, mem = check(heap, "heap", 1)
    parts = [check(starts, "starts", 8), check(lengths, "lengths", 4)] + ([check(nulls, "nulls", 1)] if nulls is not None else [])
    if any(m != mem for _, m in parts):
        raise ValueError("heap, starts, lengths and nulls of a string column must all be host arrays or all device tensors")
    n = len(starts)
    if len(lengths) != n or (nulls is not None and len(nulls) != n):
        raise ValueError("starts, lengths and nulls of a string column differ in length")
    return capi.StringColumn(hp, len(heap), parts[0][0], parts[1][0], parts[2][0] if nulls is not None else None, n, mem, 0)


def _string_columns(columns):
    """A ytgpu_string_column array over (heap, starts, lengths, nulls or None) tuples."""
    return (capi.StringColumn * len(columns))(*[_string_column(*c) for c in columns])


class GpuContext:
    """One per device/stream; wraps ytgpu_context (explicit, no thread-local state).

    use_torch_stream=False gives the context a private NON-BLOCKING stream: device inputs produced on another stream
    (torch's H2D copies included) must be complete before a call — synchronize that stream first."""

    def __init__(self, device: int = 0, use_torch_stream: bool = True):
        self.lib = capi.load()
        if torch is None or not torch.cuda.is_available():
            raise RuntimeError("ytsaurus_b200 needs a CUDA device: there is no CPU fallback for the hot path")
        self.device = device
        stream = None
        if use_torch_stream:
            with torch.cuda.device(device):
                stream = torch.cuda.current_stream(device).cuda_stream
                if stream == 0:
                    stream = 1  # cudaStreamLegacy: torch's default stream (NULL would mean "private stream")
        h = C.c_void_p()
        err = capi.Error()
        capi.check(self.lib.ytgpu_context_create(device, C.c_void_p(stream), C.byref(h), C.byref(err)), err)
        self.handle = h

    def close(self):
        if getattr(self, "handle", None):
            for table in list(getattr(self, "_join_tables", ())):  # a join table is destroyed before its context
                table.close()
            for table in list(getattr(self, "_groupby_tables", ())):
                table.close()
            self.lib.ytgpu_context_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- accounting ----
    def synchronize(self):
        err = capi.Error()
        capi.check(self.lib.ytgpu_context_synchronize(self.handle, C.byref(err)), err)

    def launch_count(self) -> int:
        return int(self.lib.ytgpu_context_launch_count(self.handle))

    def enable_timers(self, on: bool = True):
        self.lib.ytgpu_context_enable_timers(self.handle, int(on))

    def reset_timers(self):
        self.lib.ytgpu_context_reset_timers(self.handle)

    def kernel_ms(self, which: int):
        n = C.c_uint64(0)
        ms = self.lib.ytgpu_context_kernel_ms(self.handle, which, C.byref(n))
        return float(ms), int(n.value)

    def set_option(self, name: str, value: int):
        err = capi.Error()
        capi.check(self.lib.ytgpu_context_set_option(self.handle, name.encode(), int(value), C.byref(err)), err)

    def get_option(self, name: str) -> int:
        err = capi.Error()
        out = C.c_int64(0)
        capi.check(self.lib.ytgpu_context_get_option(self.handle, name.encode(), C.byref(out), C.byref(err)), err)
        return out.value

    def last_sort_passes(self) -> int:
        return int(self.lib.ytgpu_context_last_sort_passes(self.handle))

    # ---- helpers ----
    def _rowset_view(self, values, heap):
        vp, mem = _ptr_mem(values)
        if _is_tensor(values):
            if values.dtype != torch.uint8 or values.dim() != 2 or values.shape[1] % 16:
                raise ValueError("device rowsets are uint8 tensors of shape [rows, 16*value_count]")
            n, c = values.shape[0], values.shape[1] // 16
            hp, hmem = _ptr_mem(heap)
            if hmem != mem:
                raise ValueError("values and heap must share a memory space")
            hbytes = heap.numel()
        else:
            if values.dtype != VALUE_DTYPE:
                raise ValueError("host rowsets use ytsaurus_b200.rowset.VALUE_DTYPE")
            n, c = values.shape
            heap = np.ascontiguousarray(heap, dtype=np.uint8)
            hp, hbytes = heap.ctypes.data, heap.size
        view = capi.RowsetView(vp, n, c, 0, hp, hbytes, mem)
        view._keep = (values, heap)
        return view, mem, n, c

    def _out(self, shape, dtype, mem):
        if mem == capi.MEM_DEVICE:
            tdt = {np.uint32: torch.int32, np.int32: torch.int32, np.uint64: torch.int64, np.int64: torch.int64, np.uint8: torch.uint8}[dtype]
            return torch.empty(shape, dtype=tdt, device=f"cuda:{self.device}")
        return np.empty(shape, dtype=dtype)

    # ---- sort (TSortingReader / TPartitionSortReader) ----
    def sort_rowset(self, values, heap, key_columns, want_values: bool = False):
        """-> permutation (u32) [, values gathered in sorted order]."""
        view, mem, n, c = self._rowset_view(values, heap)
        spec = capi.make_sort_spec(key_columns)
        perm = self._out((n,), np.uint32, mem)
        outv = None
        if want_values:
            outv = torch.empty_like(values) if mem == capi.MEM_DEVICE else np.empty_like(values)
        err = capi.Error()
        capi.check(self.lib.ytgpu_sort_rowset(self.handle, C.byref(view), C.byref(spec), _ptr_mem(perm)[0],
                                              _ptr_mem(outv)[0] if want_values else None, mem, C.byref(err)), err)
        return (perm, outv) if want_values else perm

    def sort_fixed_rows(self, rows, row_bytes: int, key_columns, want_rows: bool = True, want_perm: bool = False,
                        out_rows=None):
        """rows: uint8 numpy array / CUDA tensor of n*row_bytes bytes."""
        rp, mem = _ptr_mem(rows)
        nbytes = rows.numel() if _is_tensor(rows) else rows.size
        n = nbytes // row_bytes
        view = capi.FixedRowsView(rp, n, row_bytes, mem)
        spec = capi.make_sort_spec(key_columns)
        if want_rows and out_rows is None:
            out_rows = torch.empty_like(rows) if mem == capi.MEM_DEVICE else np.empty_like(rows)
        perm = self._out((n,), np.uint32, mem) if want_perm else None
        err = capi.Error()
        capi.check(self.lib.ytgpu_sort_fixed_rows(self.handle, C.byref(view), C.byref(spec),
                                                  _ptr_mem(out_rows)[0] if want_rows else None,
                                                  _ptr_mem(perm)[0] if want_perm else None, mem, C.byref(err)), err)
        return out_rows, perm

    def merge_sorted_runs(self, values, heap, key_columns, run_offsets):
        view, mem, n, c = self._rowset_view(values, heap)
        spec = capi.make_sort_spec(key_columns)
        ro = np.ascontiguousarray(run_offsets, dtype=np.uint64)
        perm = self._out((n,), np.uint32, mem)
        err = capi.Error()
        capi.check(self.lib.ytgpu_merge_sorted_runs(self.handle, C.byref(view), C.byref(spec), ro.ctypes.data,
                                                    len(ro) - 1, _ptr_mem(perm)[0], mem, C.byref(err)), err)
        return perm

    def join_sorted_runs(self, values, heap, key_columns, join_key_column_count, run_offsets):
        """TSortedJoiningReader: run 0 = primary stream, the others foreign -> indices of the emitted rows in order."""
        view, mem, n, c = self._rowset_view(values, heap)
        spec = capi.make_sort_spec(key_columns)
        ro = np.ascontiguousarray(run_offsets, dtype=np.uint64)
        perm = self._out((max(n, 1),), np.uint32, mem)
        count = C.c_uint64(0)
        err = capi.Error()
        capi.check(self.lib.ytgpu_join_sorted_runs(self.handle, C.byref(view), C.byref(spec), C.c_uint32(join_key_column_count),
                                                   ro.ctypes.data, C.c_uint32(len(ro) - 1), _ptr_mem(perm)[0],
                                                   C.byref(count), mem, C.byref(err)), err)
        return perm[:count.value]

    # ---- partitioners (IPartitioner) ----
    def _partition_spec(self, kind, partition_count, key_columns=None, bounds: Rowset | None = None,
                        bound_prefix_length=None, bound_inclusive=None, key_column_count=0, salt=0, column_id=0):
        spec = capi.PartitionSpec()
        spec.kind = kind
        spec.partition_count = partition_count
        keep = []
        if key_columns is not None:
            ks = capi.make_sort_spec(key_columns)
            spec.key = ks
            keep.append(ks)
        if bounds is not None:
            bv = np.ascontiguousarray(bounds.values, dtype=VALUE_DTYPE)
            bh = np.ascontiguousarray(bounds.heap, dtype=np.uint8)
            bl = np.ascontiguousarray(bound_prefix_length, dtype=np.uint32)
            bi = np.ascontiguousarray(bound_inclusive, dtype=np.uint8)
            spec.bounds = bv.ctypes.data
            spec.bounds_heap = bh.ctypes.data
            spec.bounds_heap_bytes = bh.size
            spec.bound_value_count = bv.shape[1] if bv.ndim == 2 else 0
            spec.bound_prefix_length = bl.ctypes.data
            spec.bound_inclusive = bi.ctypes.data
            keep += [bv, bh, bl, bi]
        spec.key_column_count = key_column_count
        spec.salt = salt
        spec.partition_column_id = column_id
        spec._keep = keep
        return spec

    def partition_rowset(self, values, heap, spec, want_histogram: bool = True):
        view, mem, n, c = self._rowset_view(values, heap)
        idx = self._out((n,), np.int32, mem)
        hist = self._out((spec.partition_count,), np.uint64, mem) if want_histogram else None
        err = capi.Error()
        capi.check(self.lib.ytgpu_partition_rowset(self.handle, C.byref(view), C.byref(spec), _ptr_mem(idx)[0],
                                                   _ptr_mem(hist)[0] if want_histogram else None, mem,
                                                   C.byref(err)), err)
        return idx, hist

    def partition_rowset_slabs(self, values, heap, spec):
        """-> (partition index, histogram, values grouped by partition (stable), input row of every slab row)."""
        view, mem, n, c = self._rowset_view(values, heap)
        idx = self._out((n,), np.int32, mem)
        hist = self._out((spec.partition_count,), np.uint64, mem)
        if mem == capi.MEM_DEVICE:
            slab = torch.empty_like(values)
        else:
            slab = np.zeros_like(values)
        perm = self._out((n,), np.uint32, mem)
        err = capi.Error()
        capi.check(self.lib.ytgpu_partition_rowset_slabs(self.handle, C.byref(view), C.byref(spec), _ptr_mem(idx)[0], _ptr_mem(hist)[0],
                                                         _ptr_mem(slab)[0], _ptr_mem(perm)[0], mem, C.byref(err)), err)
        return idx, hist, slab, perm

    def partition_fixed_rows(self, rows, row_bytes, spec, want_index=True, want_slabs=True, out_slabs=None):
        rp, mem = _ptr_mem(rows)
        nbytes = rows.numel() if _is_tensor(rows) else rows.size
        n = nbytes // row_bytes
        view = capi.FixedRowsView(rp, n, row_bytes, mem)
        idx = self._out((n,), np.int32, mem) if want_index else None
        hist = self._out((spec.partition_count,), np.uint64, mem)
        if want_slabs and out_slabs is None:
            out_slabs = torch.empty_like(rows) if mem == capi.MEM_DEVICE else np.empty_like(rows)
        err = capi.Error()
        capi.check(self.lib.ytgpu_partition_fixed_rows(self.handle, C.byref(view), C.byref(spec),
                                                       _ptr_mem(idx)[0] if want_index else None, _ptr_mem(hist)[0],
                                                       _ptr_mem(out_slabs)[0] if want_slabs else None, mem,
                                                       C.byref(err)), err)
        return idx, hist, out_slabs

    # ---- NVLink peer memory (in-box shuffle) ----
    def peer_buffer_create(self, nbytes: int):
        """-> (device pointer, 64-byte IPC handle as bytes)."""
        p = C.c_void_p()
        handle = (C.c_uint8 * 64)()
        err = capi.Error()
        capi.check(self.lib.ytgpu_peer_buffer_create(self.handle, nbytes, C.byref(p), handle, C.byref(err)), err)
        return p.value, bytes(handle)

    def peer_buffer_destroy(self, ptr: int):
        err = capi.Error()
        capi.check(self.lib.ytgpu_peer_buffer_destroy(self.handle, C.c_void_p(ptr), C.byref(err)), err)

    def peer_buffer_open(self, handle: bytes) -> int:
        p = C.c_void_p()
        buf = (C.c_uint8 * 64).from_buffer_copy(handle)
        err = capi.Error()
        capi.check(self.lib.ytgpu_peer_buffer_open(self.handle, buf, C.byref(p), C.byref(err)), err)
        return p.value

    def peer_buffer_close(self, ptr: int):
        err = capi.Error()
        capi.check(self.lib.ytgpu_peer_buffer_close(self.handle, C.c_void_p(ptr), C.byref(err)), err)

    def scatter_rows_to_peers(self, rows, row_bytes: int, partition_index, partition_rows, dest_ptrs):
        """rows / partition_index: CUDA tensors; partition_rows: rows per partition (host ints);
        dest_ptrs: device pointer (int) where each partition's slab starts (local or peer-mapped)."""
        rp, mem = _ptr_mem(rows)
        if mem != capi.MEM_DEVICE:
            raise ValueError("peer scatter needs device-resident rows")
        n = rows.numel() // row_bytes
        view = capi.FixedRowsView(rp, n, row_bytes, mem)
        P = len(dest_ptrs)
        pr = (C.c_uint64 * P)(*[int(x) for x in partition_rows])
        dp = (C.c_void_p * P)(*[int(x) for x in dest_ptrs])
        err = capi.Error()
        capi.check(self.lib.ytgpu_scatter_rows_to_peers(self.handle, C.byref(view), _ptr_mem(partition_index)[0], P, pr, dp,
                                                        C.byref(err)), err)

    # ---- in-box distributed sort behind the C ABI (ytgpu_shuffle_*) ----
    def shuffle_create(self, world: int, rank: int, capacity_rows: int, row_bytes: int):
        """-> (opaque shuffle handle, 64-byte IPC handle of this rank's receive buffer)."""
        h = C.c_void_p()
        handle = (C.c_uint8 * 64)()
        err = capi.Error()
        capi.check(self.lib.ytgpu_shuffle_create(self.handle, world, rank, capacity_rows, row_bytes, C.byref(h), handle,
                                                 C.byref(err)), err)
        return h, bytes(handle)

    def shuffle_connect(self, shuffle, handles: bytes):
        buf = (C.c_uint8 * len(handles)).from_buffer_copy(handles)
        err = capi.Error()
        capi.check(self.lib.ytgpu_shuffle_connect(shuffle, buf, C.byref(err)), err)

    def shuffle_sort(self, shuffle, rows, row_bytes: int, key_columns, out_rows):
        """Collective.  rows / out_rows: CUDA uint8 tensors.  -> (rows of this rank's key range, capi.ShuffleStats)."""
        rp, mem = _ptr_mem(rows)
        if mem != capi.MEM_DEVICE:
            raise ValueError("the in-box shuffle sorts device-resident rows")
        n = rows.numel() // row_bytes
        view = capi.FixedRowsView(rp, n, row_bytes, mem)
        spec = capi.make_sort_spec(key_columns)
        got = C.c_uint64(0)
        stats = capi.ShuffleStats()
        err = capi.Error()
        capi.check(self.lib.ytgpu_shuffle_sort(shuffle, C.byref(view), C.byref(spec), _ptr_mem(out_rows)[0],
                                               out_rows.numel() // row_bytes, C.byref(got), C.byref(stats), C.byref(err)), err)
        return int(got.value), stats

    def shuffle_destroy(self, shuffle):
        err = capi.Error()
        capi.check(self.lib.ytgpu_shuffle_destroy(shuffle, C.byref(err)), err)

    # ---- segmented SUM / COUNT over sorted rows (the aggregate stage after a sort) ----
    def reduce_sorted_fixed_rows(self, rows, row_bytes: int, key_offset: int, value_offset: int, value_type: int, out_keys, out_sums,
                                 out_counts) -> int:
        """rows: sorted fixed-width rows (CUDA uint8 tensor); out_*: CUDA int64 tensors of equal capacity.  -> group count."""
        rp, mem = _ptr_mem(rows)
        if mem != capi.MEM_DEVICE:
            raise ValueError("the sorted reduce reads device-resident rows")
        view = capi.FixedRowsView(rp, rows.numel() // row_bytes, row_bytes, mem)
        got = C.c_uint64(0)
        err = capi.Error()
        capi.check(self.lib.ytgpu_reduce_sorted_fixed_rows(self.handle, C.byref(view), key_offset, value_offset, value_type,
                                                           _ptr_mem(out_keys)[0], _ptr_mem(out_sums)[0], _ptr_mem(out_counts)[0],
                                                           out_keys.numel(), C.byref(got), C.byref(err)), err)
        return int(got.value)

    def farm_fingerprints(self, values, heap, key_column_count: int):
        view, mem, n, c = self._rowset_view(values, heap)
        out = self._out((n,), np.uint64, mem)
        err = capi.Error()
        capi.check(self.lib.ytgpu_farm_fingerprint_rowset(self.handle, C.byref(view), key_column_count,
                                                          _ptr_mem(out)[0], mem, C.byref(err)), err)
        return out

    # ---- horizontal block codec (THorizontalBlockReader / Writer) ----
    def decode_horizontal_block(self, block, row_count: int, value_count: int):
        """block: uint8 numpy array or CUDA tensor.  -> (values [rows, value_count], per-row value counts);
        string values point into `block` (use it as the rowset's heap)."""
        bp, mem = _ptr_mem(block)
        nbytes = block.numel() if _is_tensor(block) else block.size
        if mem == capi.MEM_DEVICE:
            out = torch.empty((row_count, value_count * 16), dtype=torch.uint8, device=f"cuda:{self.device}")
        else:
            out = np.zeros((row_count, value_count), dtype=VALUE_DTYPE)
        counts = self._out((row_count,), np.uint32, mem)
        err = capi.Error()
        capi.check(self.lib.ytgpu_decode_horizontal_block(self.handle, bp, nbytes, row_count, value_count,
                                                          _ptr_mem(out)[0], _ptr_mem(counts)[0], mem, C.byref(err)), err)
        return out, counts

    def encode_horizontal_block(self, values, heap, row_value_counts=None):
        """-> block bytes (numpy uint8 / CUDA uint8 tensor)."""
        view, mem, n, c = self._rowset_view(values, heap)
        need = C.c_uint64(0)
        err = capi.Error()
        rc = _ptr_mem(row_value_counts)[0] if row_value_counts is not None else None
        code = self.lib.ytgpu_encode_horizontal_block(self.handle, C.byref(view), rc, None, 0, C.byref(need), mem, C.byref(err))
        if n == 0:
            return self._out((0,), np.uint8, mem)
        if code != capi.ERR_INVALID_ARGUMENT or need.value == 0:
            capi.check(code, err)
        out = self._out((need.value,), np.uint8, mem)
        capi.check(self.lib.ytgpu_encode_horizontal_block(self.handle, C.byref(view), rc, _ptr_mem(out)[0], need.value,
                                                          C.byref(need), mem, C.byref(err)), err)
        return out

    # ---- YQL block aggregators over Arrow blocks (IBlockAggregatorCombineAll) ----
    def block_agg_state(self, value_type: int, nullable: bool = True) -> capi.BlockAggState:
        state = capi.BlockAggState()
        self.lib.ytgpu_block_agg_state_init(C.byref(state), value_type, int(bool(nullable)))
        return state

    def block_combine_all(self, state: capi.BlockAggState, values, validity=None, offset: int = 0, length=None,
                          nullable: bool = True, filter=None):
        """AddMany of sum/avg/min/max/count/count_all over one Arrow array (values: 64-bit buffer NOT offset-adjusted,
        validity: LSB bitmap, 1 = valid).  Folds the batch into `state` and returns it."""
        vp, mem = _ptr_mem(values)
        total = values.numel() if _is_tensor(values) else values.size
        if length is None:
            length = total - offset
        for other in (validity, filter):
            if other is not None and _ptr_mem(other)[1] != mem:
                raise ValueError("values, validity and filter must share a memory space")
        arr = capi.ArrowArray(vp, _ptr_mem(validity)[0], offset, length, state.value_type, int(bool(nullable)), 0, mem)
        err = capi.Error()
        capi.check(self.lib.ytgpu_block_combine_all(self.handle, C.byref(arr), _ptr_mem(filter)[0], C.byref(state),
                                                    C.byref(err)), err)
        return state

    # ---- columnar write side (column converter + unversioned integer column writer) ----
    def convert_integer_column(self, values, heap, column_index: int, value_type: int):
        """rows -> (64-bit words, null bitmap bytes, base value) as TIntegerColumnConverter<T>::Convert emits them."""
        view, mem, n, c = self._rowset_view(values, heap)
        words = self._out((n,), np.uint64, mem)
        bitmap = self._out((8 * ((n + 63) // 64),), np.uint8, mem)
        base = C.c_uint64(0)
        err = capi.Error()
        capi.check(self.lib.ytgpu_convert_integer_column(self.handle, C.byref(view), column_index, value_type,
                                                         _ptr_mem(words)[0], _ptr_mem(bitmap)[0], C.byref(base), mem,
                                                         C.byref(err)), err)
        return words, bitmap, base.value

    def encode_integer_column(self, values, nulls=None, signed: bool = False, max_segment_values: int = 128 * 1024,
                              chunk_row_offset: int = 0):
        """values: uint64/int64 numpy array or int64 CUDA tensor; nulls: uint8 bytemap (1 = null) or None.
        -> (segment data bytes, numpy array of capi.INTEGER_SEGMENT_DTYPE descriptors)."""
        vp, mem = _ptr_mem(values)
        n = values.numel() if _is_tensor(values) else values.size
        np_, nmem = _ptr_mem(nulls)
        if nulls is not None and nmem != mem:
            raise ValueError("values and nulls must share a memory space")
        seg_cap = max(1, (n + max_segment_values - 1) // max_segment_values)
        segs = np.zeros(seg_cap, dtype=capi.INTEGER_SEGMENT_DTYPE)
        need, nseg = C.c_uint64(0), C.c_uint32(0)
        err = capi.Error()
        args = (self.handle, vp, np_, n, int(bool(signed)), max_segment_values, chunk_row_offset, mem)
        if n == 0:
            capi.check(self.lib.ytgpu_encode_integer_column(*args, None, 0, C.byref(need), segs.ctypes.data, seg_cap,
                                                            C.byref(nseg), C.byref(err)), err)
            return self._out((0,), np.uint8, mem), segs[:0]
        # One call: the writer picks the smallest layout by its own estimate and DirectDense is always a candidate, so
        # a segment never needs more than DirectDense's words plus the three vector headers.
        cap = 8 * n + 8 * ((n + 63) // 64 + 8 * seg_cap) + 64
        out = self._out((cap,), np.uint8, mem)
        capi.check(self.lib.ytgpu_encode_integer_column(*args, _ptr_mem(out)[0], cap, C.byref(need), segs.ctypes.data,
                                                        seg_cap, C.byref(nseg), C.byref(err)), err)
        return out[:need.value], segs[:nseg.value]

    def encode_plain_column(self, values, nulls=None, boolean: bool = False, max_segment_values: int = 128 * 1024,
                            chunk_row_offset: int = 0):
        """The double (values: 64-bit patterns) / boolean (values: one byte per row) column writers
        -> (segment data bytes, numpy array of capi.PLAIN_SEGMENT_DTYPE descriptors)."""
        vp, mem = _ptr_mem(values)
        n = values.numel() if _is_tensor(values) else values.size
        np_, nmem = _ptr_mem(nulls)
        if nulls is not None and nmem != mem:
            raise ValueError("values and nulls must share a memory space")
        seg_cap = max(1, (n + max_segment_values - 1) // max_segment_values)
        segs = np.zeros(seg_cap, dtype=capi.PLAIN_SEGMENT_DTYPE)
        need, nseg = C.c_uint64(0), C.c_uint32(0)
        err = capi.Error()
        fn = self.lib.ytgpu_encode_boolean_column if boolean else self.lib.ytgpu_encode_double_column
        cap = (8 if not boolean else 0) * n + 16 * ((n + 63) // 64 + seg_cap) + 8 * seg_cap + 64
        out = self._out((cap,), np.uint8, mem)
        capi.check(fn(self.handle, vp, np_, n, max_segment_values, chunk_row_offset, mem, _ptr_mem(out)[0], cap, C.byref(need),
                      segs.ctypes.data, seg_cap, C.byref(nseg), C.byref(err)), err)
        return out[:need.value], segs[:nseg.value]

    def encode_string_column(self, heap, starts, lengths, nulls=None, max_segment_values: int = 128 * 1024,
                             max_buffer_bytes: int = 0, chunk_row_offset: int = 0):
        """The string column writer: value i = heap[starts[i] : starts[i] + lengths[i]] (uint8 heap, uint64 starts, uint32
        lengths; numpy arrays or CUDA tensors — int64 / int32 tensors stand in for the unsigned types)
        -> (segment data bytes, numpy array of capi.STRING_SEGMENT_DTYPE descriptors)."""
        hp, mem = _ptr_mem(heap)
        sp, lp = _ptr_mem(starts)[0], _ptr_mem(lengths)[0]
        np_ = _ptr_mem(nulls)[0]
        n = starts.numel() if _is_tensor(starts) else starts.size
        hbytes = heap.numel() if _is_tensor(heap) else heap.size
        total = int(lengths.sum()) if n else 0
        buf = max_buffer_bytes or (32 << 20)
        seg_cap = max(1, (n + max_segment_values - 1) // max_segment_values + total // (buf + 1) + 2)
        segs = np.zeros(seg_cap, dtype=capi.STRING_SEGMENT_DTYPE)
        need, nseg = C.c_uint64(0), C.c_uint32(0)
        err = capi.Error()
        cap = total + 16 * n + 128 * seg_cap + 64
        out = self._out((cap,), np.uint8, mem)
        capi.check(self.lib.ytgpu_encode_string_column(self.handle, hp, hbytes, sp, lp, np_, n, max_segment_values, max_buffer_bytes,
                                                       chunk_row_offset, mem, _ptr_mem(out)[0], cap, C.byref(need), segs.ctypes.data,
                                                       seg_cap, C.byref(nseg), C.byref(err)), err)
        return out[:need.value], segs[:nseg.value]

    def decode_string_segment(self, data, segment):
        """data: the column data returned by encode_string_column (numpy / CUDA uint8), segment: one descriptor
        -> (starts u32 relative to the segment's first byte, lengths u32, null bytemap)."""
        a = int(segment["data_offset"])
        blob = data[a:a + int(segment["data_bytes"])]
        bp, mem = _ptr_mem(blob)
        rows = int(segment["row_count"])
        seg = np.ascontiguousarray(np.asarray(segment).reshape(1))
        starts = self._out((rows,), np.uint32, mem)
        lengths = self._out((rows,), np.uint32, mem)
        nulls = self._out((rows,), np.uint8, mem)
        err = capi.Error()
        capi.check(self.lib.ytgpu_decode_string_segment(self.handle, seg.ctypes.data, bp, _ptr_mem(starts)[0], _ptr_mem(lengths)[0],
                                                        _ptr_mem(nulls)[0], mem, C.byref(err)), err)
        return starts, lengths, nulls

    def string_value_ids(self, heap, starts, lengths, nulls=None):
        """-> (ids u64: index of the first row holding the same string, null bytemap): string GROUP BY keys."""
        hp, mem = _ptr_mem(heap)
        n = starts.numel() if _is_tensor(starts) else starts.size
        hbytes = heap.numel() if _is_tensor(heap) else heap.size
        ids = self._out((n,), np.uint64, mem)
        onull = self._out((n,), np.uint8, mem)
        err = capi.Error()
        capi.check(self.lib.ytgpu_string_value_ids(self.handle, hp, hbytes, _ptr_mem(starts)[0], _ptr_mem(lengths)[0], _ptr_mem(nulls)[0], n,
                                                   _ptr_mem(ids)[0], _ptr_mem(onull)[0], mem, C.byref(err)), err)
        return ids, onull

    def extract_column(self, values, heap, column: int, value_type: int):
        """rows -> one flat column: (payload u64, lengths u32, null bytemap)."""
        view, mem, n, c = self._rowset_view(values, heap)
        payload = self._out((n,), np.uint64, mem)
        lengths = self._out((n,), np.uint32, mem)
        nulls = self._out((n,), np.uint8, mem)
        err = capi.Error()
        capi.check(self.lib.ytgpu_extract_column(self.handle, C.byref(view), column, value_type, _ptr_mem(payload)[0], _ptr_mem(lengths)[0],
                                                 _ptr_mem(nulls)[0], mem, C.byref(err)), err)
        return payload, lengths, nulls

    # ---- columnar ----
    def decode_column(self, col: "Column", want_nulls: bool = True):
        view = col.view()
        mem = view.mem
        n = col.value_count
        out = self._out((n,), np.uint64, mem)
        nulls = self._out((n,), np.uint8, mem) if want_nulls else None
        err = capi.Error()
        capi.check(self.lib.ytgpu_decode_column(self.handle, C.byref(view), _ptr_mem(out)[0],
                                                _ptr_mem(nulls)[0] if want_nulls else None, mem, C.byref(err)), err)
        return out, nulls

    def decode_column_typed(self, col: "Column", element_bytes: int, want_nulls: bool = True):
        """The decode into a ClickHouse ColumnVector<T>: values narrowed to element_bytes (floats widened to doubles)."""
        view = col.view()
        mem = view.mem
        n = col.value_count
        if mem == capi.MEM_DEVICE:
            out = torch.empty(n * element_bytes, dtype=torch.uint8, device=f"cuda:{self.device}")
        else:
            out = np.empty(n, dtype={1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[element_bytes])
        nulls = self._out((n,), np.uint8, mem) if want_nulls else None
        err = capi.Error()
        capi.check(self.lib.ytgpu_decode_column_typed(self.handle, C.byref(view), element_bytes, _ptr_mem(out)[0],
                                                      _ptr_mem(nulls)[0] if want_nulls else None, mem, C.byref(err)), err)
        return out, nulls

    def decode_string_offsets(self, encoded, avg_length, start, end):
        ep, mem = _ptr_mem(encoded)
        out = self._out((end - start + 1,), np.uint32, mem)
        err = capi.Error()
        capi.check(self.lib.ytgpu_decode_string_offsets(self.handle, ep, avg_length, start, end, _ptr_mem(out)[0],
                                                        mem, C.byref(err)), err)
        return out

    def decode_string_pointers_and_lengths(self, encoded, avg_length):
        """-> (start offsets u32, lengths i32) of every value of a string segment (DecodeStringPointersAndLengths)."""
        ep, mem = _ptr_mem(encoded)
        n = encoded.numel() if _is_tensor(encoded) else encoded.size
        st = self._out((n,), np.uint32, mem)
        ln = self._out((n,), np.int32, mem)
        err = capi.Error()
        capi.check(self.lib.ytgpu_decode_string_pointers_and_lengths(self.handle, ep, avg_length, n, _ptr_mem(st)[0], _ptr_mem(ln)[0],
                                                                     mem, C.byref(err)), err)
        return st, ln

    # ---- YT string column -> ClickHouse ColumnString (ConvertStringLikeYTColumnToCHColumn) ----
    def convert_string_column_to_ch(self, offsets, avg_length, chars, dict_idx, rle, start, count, filter_hint=None, size_query=False):
        """-> (chars uint8[], offsets uint64[count]).  size_query: ask for the exact chars size first (two calls); otherwise the
        buffer is sized with the reference's estimate and the call is repeated only when that was too small."""
        op, mem = _ptr_mem(offsets)
        size = lambda a: 0 if a is None else (a.numel() if _is_tensor(a) else a.size)
        for other in (chars, dict_idx, rle, filter_hint):
            if other is not None and _ptr_mem(other)[1] != mem:
                raise ValueError("all buffers of a string column must share a memory space")
        view = capi.StringColumnView(op, size(offsets), int(avg_length), mem, _ptr_mem(chars)[0], size(chars), _ptr_mem(dict_idx)[0],
                                     size(dict_idx), _ptr_mem(rle)[0], size(rle), int(start), int(count))
        need = C.c_uint64(0)
        err = capi.Error()
        out_offsets = self._out((max(count, 0),), np.uint64, mem)
        if size_query:
            capi.check(self.lib.ytgpu_convert_string_column_to_ch(self.handle, C.byref(view), _ptr_mem(filter_hint)[0], None, 0, None,
                                                                  C.byref(need), mem, C.byref(err)), err)
            capacity = need.value
        else:  # the reference's own first guess (columnar_conversion.cpp:497-503): (avg + 1) * rows * 2 + 1 KB
            capacity = (int(avg_length) + 1) * max(count, 0) * 2 + 1024
        out_chars = self._out((capacity,), np.uint8, mem)
        code = self.lib.ytgpu_convert_string_column_to_ch(self.handle, C.byref(view), _ptr_mem(filter_hint)[0], _ptr_mem(out_chars)[0],
                                                          capacity, _ptr_mem(out_offsets)[0], C.byref(need), mem, C.byref(err))
        if code != capi.OK and need.value > capacity:  # the guess was too small: the call reported the exact size
            capacity = need.value
            out_chars = self._out((capacity,), np.uint8, mem)
            code = self.lib.ytgpu_convert_string_column_to_ch(self.handle, C.byref(view), _ptr_mem(filter_hint)[0], _ptr_mem(out_chars)[0],
                                                              capacity, _ptr_mem(out_offsets)[0], C.byref(need), mem, C.byref(err))
        capi.check(code, err)
        return out_chars[:need.value], out_offsets

    # ---- ClickHouse column -> unversioned values (TCHToYTConverter, simple types) ----
    def convert_ch_column_to_values(self, ch_type, data, row_count, offsets=None, null_map=None, time_adjustment=0):
        """-> values[row_count] (VALUE_DTYPE on the host, uint8[row_count, 16] on the device); strings point into `data`."""
        dp, mem = _ptr_mem(data)
        for other in (offsets, null_map):
            if other is not None and _ptr_mem(other)[1] != mem:
                raise ValueError("all buffers of a ClickHouse column must share a memory space")
        chars = 0
        if offsets is not None:
            chars = data.numel() if _is_tensor(data) else data.size
        col = capi.ChColumn(int(ch_type), mem, dp, _ptr_mem(offsets)[0], chars, _ptr_mem(null_map)[0], int(time_adjustment), row_count)
        if mem == capi.MEM_DEVICE:
            out = torch.empty((row_count, 16), dtype=torch.uint8, device=f"cuda:{self.device}")
        else:
            out = np.zeros(row_count, dtype=VALUE_DTYPE)
        err = capi.Error()
        capi.check(self.lib.ytgpu_convert_ch_column_to_values(self.handle, C.byref(col), _ptr_mem(out)[0], mem, C.byref(err)), err)
        return out

    # ---- null / dictionary-index helpers of the column readers (client/table_client/columnar.h) ----
    @staticmethod
    def _flag_source(kind, data, data_count, rle):
        dp, mem = _ptr_mem(data)
        rp, rmem = _ptr_mem(rle)
        if rle is not None and rmem != mem:
            raise ValueError("flag source data and rle indexes must live in the same memory space")
        n_rle = 0 if rle is None else (rle.numel() if _is_tensor(rle) else rle.size)
        return capi.FlagSource(kind, 0, dp, data_count, rp, n_rle), mem

    def build_bitmap_from_flags(self, kind, data, data_count, rle, start, end, negate):
        """Validity bitmaps / bitmap range copies -> uint8[GetBitmapByteSize(end - start)]."""
        src, mem = self._flag_source(kind, data, data_count, rle)
        out = self._out((max(end - start + 7, 0) // 8,), np.uint8, mem)
        err = capi.Error()
        capi.check(self.lib.ytgpu_build_bitmap_from_flags(self.handle, C.byref(src), start, end, int(negate), _ptr_mem(out)[0], mem,
                                                          C.byref(err)), err)
        return out

    def build_bytemap_from_flags(self, kind, data, data_count, rle, start, end, negate=False):
        """Null bytemaps -> uint8[end - start] of 0 / 1."""
        src, mem = self._flag_source(kind, data, data_count, rle)
        out = self._out((max(end - start, 0),), np.uint8, mem)
        err = capi.Error()
        capi.check(self.lib.ytgpu_build_bytemap_from_flags(self.handle, C.byref(src), start, end, int(negate), _ptr_mem(out)[0], mem,
                                                           C.byref(err)), err)
        return out

    def count_flags(self, kind, data, data_count, rle, start, end) -> int:
        src, mem = self._flag_source(kind, data, data_count, rle)
        out = C.c_int64(0)
        err = capi.Error()
        capi.check(self.lib.ytgpu_count_flags(self.handle, C.byref(src), start, end, C.byref(out), mem, C.byref(err)), err)
        return out.value

    def build_dictionary_indexes(self, dict_idx, rle, start, end):
        """idx - 1 per row (null -> 0xFFFFFFFF); dict_idx None: the run number of every row (iota)."""
        dp, mem = _ptr_mem(dict_idx)
        rp, rmem = _ptr_mem(rle)
        if dict_idx is None:
            mem = rmem
        n_dict = 0 if dict_idx is None else (dict_idx.numel() if _is_tensor(dict_idx) else dict_idx.size)
        n_rle = 0 if rle is None else (rle.numel() if _is_tensor(rle) else rle.size)
        out = self._out((max(end - start, 0),), np.uint32, mem)
        err = capi.Error()
        capi.check(self.lib.ytgpu_build_dictionary_indexes(self.handle, dp, n_dict, rp, n_rle, start, end, _ptr_mem(out)[0], mem,
                                                           C.byref(err)), err)
        return out

    def count_total_string_length(self, dict_idx, rle, lengths, start, end) -> int:
        dp, mem = _ptr_mem(dict_idx)
        n_rle = rle.numel() if _is_tensor(rle) else rle.size
        n_str = lengths.numel() if _is_tensor(lengths) else lengths.size
        out = C.c_int64(0)
        err = capi.Error()
        capi.check(self.lib.ytgpu_count_total_string_length(self.handle, dp, _ptr_mem(rle)[0], n_rle, _ptr_mem(lengths)[0], n_str,
                                                            start, end, C.byref(out), mem, C.byref(err)), err)
        return out.value

    def translate_rle_indexes(self, rle, indexes, end_flavour=False):
        rp, mem = _ptr_mem(rle)
        n_rle = rle.numel() if _is_tensor(rle) else rle.size
        n = indexes.numel() if _is_tensor(indexes) else indexes.size
        out = self._out((n,), np.int64, mem)
        err = capi.Error()
        capi.check(self.lib.ytgpu_translate_rle_indexes(self.handle, rp, n_rle, _ptr_mem(indexes)[0], n, int(end_flavour),
                                                        _ptr_mem(out)[0], mem, C.byref(err)), err)
        return out

    def scan_filter_groupby(self, key_col: "Column", val_col: "Column", predicate=None, group_count_hint: int = 0,
                            capacity: int | None = None, want_first_rows: bool = False, want_min_max: bool = False):
        """-> dict(keys, key_null, sum (u64 bit patterns), sum_null, count[, first_row][, min, max]), ordered by (key_null, key)."""
        kv, vv = key_col.view(), val_col.view()
        mem = kv.mem
        if capacity is None:
            capacity = min(key_col.value_count, group_count_hint * 2 if group_count_hint else key_col.value_count) + 2
        keys = self._out((capacity,), np.uint64, mem)
        sums = self._out((capacity,), np.uint64, mem)
        counts = self._out((capacity,), np.uint64, mem)
        kn = self._out((capacity,), np.uint8, mem)
        sn = self._out((capacity,), np.uint8, mem)
        first = self._out((capacity,), np.uint64, mem) if want_first_rows else None
        mins = self._out((capacity,), np.uint64, mem) if want_min_max else None
        maxs = self._out((capacity,), np.uint64, mem) if want_min_max else None
        res = capi.GroupByResult(0, _ptr_mem(keys)[0], _ptr_mem(kn)[0], _ptr_mem(sums)[0], _ptr_mem(sn)[0],
                                 _ptr_mem(counts)[0], capacity, _ptr_mem(first)[0] if want_first_rows else None,
                                 _ptr_mem(mins)[0] if want_min_max else None, _ptr_mem(maxs)[0] if want_min_max else None)
        pred = None
        if predicate is not None:
            op, const = predicate
            pred = capi.Predicate(op, 0, const & 0xFFFFFFFFFFFFFFFF)
        err = capi.Error()
        capi.check(self.lib.ytgpu_scan_filter_groupby(self.handle, C.byref(kv), C.byref(vv),
                                                      C.byref(pred) if pred is not None else None,
                                                      group_count_hint, C.byref(res), mem, C.byref(err)), err)
        g = int(res.group_count)
        res_d = dict(keys=keys[:g], key_null=kn[:g], sum=sums[:g], sum_null=sn[:g], count=counts[:g])
        if want_first_rows:
            res_d["first_row"] = first[:g]
        if want_min_max:
            res_d["min"], res_d["max"] = mins[:g], maxs[:g]
        return res_d


    def scan_filter_groupby_multi(self, key_cols, value_cols, aggregates, predicate=None, predicate_column: int = -1,
                                  group_count_hint: int = 0, capacity: int | None = None, string_columns=()):
        """GROUP BY key tuple with a list of aggregates [(op, column[, by_column])] ->
        dict(keys=[...], key_null=[...], values=[...], value_null=[...], count, first_row), first-seen order.
        string_columns: (heap, starts, lengths, nulls or None) per column; aggregate column len(value_cols) + i is string
        column i, and a string-valued result is the index of the row that holds it."""
        kviews = [c.view() for c in key_cols]
        vviews = [c.view() for c in value_cols]
        mem = kviews[0].mem
        sarr = (capi.StringColumn * max(len(string_columns), 1))()
        for i, column in enumerate(string_columns):
            sarr[i] = _string_column(*column)
        n = key_cols[0].value_count
        if capacity is None:
            capacity = max(n, 1)
        karr = (capi.ColumnView * len(kviews))(*kviews)
        varr = (capi.ColumnView * max(len(vviews), 1))(*vviews)
        aggs = (capi.Aggregate * max(len(aggregates), 1))()
        for i, a in enumerate(aggregates):
            aggs[i].op, aggs[i].column = a[0], a[1]
            aggs[i].by_column = a[2] if len(a) > 2 else -1
        keys = [self._out((capacity,), np.uint64, mem) for _ in kviews]
        kn = [self._out((capacity,), np.uint8, mem) for _ in kviews]
        vals = [self._out((capacity,), np.uint64, mem) for _ in aggregates]
        vn = [self._out((capacity,), np.uint8, mem) for _ in aggregates]
        counts = self._out((capacity,), np.uint64, mem)
        first = self._out((capacity,), np.uint64, mem)

        def ptrs(arrs):
            return (C.c_void_p * max(len(arrs), 1))(*[_ptr_mem(a)[0] for a in arrs])
        pk, pkn, pv, pvn = ptrs(keys), ptrs(kn), ptrs(vals), ptrs(vn)
        res = capi.GroupByMultiResult(0, capacity, pk, pkn, pv, pvn, _ptr_mem(counts)[0], _ptr_mem(first)[0])
        pred = None
        if predicate is not None:
            op, const = predicate
            pred = capi.Predicate(op, 0, const & 0xFFFFFFFFFFFFFFFF)
        err = capi.Error()
        args = [self.handle, C.cast(karr, C.c_void_p), len(kviews), C.cast(varr, C.c_void_p), len(vviews), C.cast(aggs, C.c_void_p),
                len(aggregates), C.cast(C.pointer(pred), C.c_void_p) if pred is not None else None, predicate_column,
                group_count_hint, C.byref(res), mem]
        if string_columns:
            code = self.lib.ytgpu_scan_filter_groupby_multi_strings(*args, C.cast(sarr, C.c_void_p), len(string_columns), C.byref(err))
        else:
            code = self.lib.ytgpu_scan_filter_groupby_multi(*args, C.byref(err))
        capi.check(code, err)
        g = int(res.group_count)
        return dict(keys=[k[:g] for k in keys], key_null=[k[:g] for k in kn], values=[v[:g] for v in vals],
                    value_null=[v[:g] for v in vn], count=counts[:g], first_row=first[:g])

    def hash_join(self, primary_keys, foreign_keys, kind: int = capi.JOIN_INNER, count_only: bool = False,
                  capacity: int | None = None, out_mem: int | None = None):
        """Hash JOIN of key tuples (ytgpu_hash_join): primary_keys and foreign_keys are lists of Column, key k of one type on
        both sides.  -> (primary rows, foreign rows): the pairs in ascending (primary, foreign) order, a LEFT join's unmatched
        primary row paired with capi.JOIN_NO_ROW, as uint32 arrays (int32 tensors in DEVICE memory); with count_only, the
        pair count.  The outputs are in out_mem (default: the primary keys' memory).  Without a capacity a count query sizes
        them first; a capacity below the count raises YtGpuError with .pair_count set."""
        pviews = [c.view() for c in primary_keys]
        fviews = [c.view() for c in foreign_keys]
        if out_mem is None:
            out_mem = pviews[0].mem if pviews else capi.MEM_HOST
        parr = (capi.ColumnView * max(len(pviews), 1))(*pviews)
        farr = (capi.ColumnView * max(len(fviews), 1))(*fviews)
        count = C.c_uint64(0)
        err = capi.Error()

        def call(prim=None, fore=None, cap=0):
            code = self.lib.ytgpu_hash_join(self.handle, C.cast(parr, C.c_void_p), C.cast(farr, C.c_void_p), len(pviews), kind,
                                            _ptr_mem(prim)[0], _ptr_mem(fore)[0], cap, C.byref(count), out_mem, C.byref(err))
            if code != capi.OK:
                e = capi.YtGpuError(code, err.message.decode(errors="replace"), err.cuda_error)
                e.pair_count = int(count.value)  # the needed capacity when that was too small
                raise e
        if count_only or capacity is None:
            call()
            if count_only:
                return int(count.value)
            capacity = int(count.value)
        prim = self._out((max(capacity, 1),), np.uint32, out_mem)
        fore = self._out((max(capacity, 1),), np.uint32, out_mem)
        call(prim, fore, capacity)
        pairs = int(count.value)
        return prim[:pairs], fore[:pairs]

    def join_table(self, foreign_keys, nulls: int = capi.JOIN_NULLS_EQUAL, string_keys=()) -> "JoinTable":
        """ytgpu_join_table_build: a join table over foreign_keys (a list of Column), built once and probed any number of
        times (JoinTable.probe).  nulls: capi.JOIN_NULLS_EQUAL (NULL equals NULL, as hash_join) or
        capi.JOIN_NULLS_NEVER_MATCH (a tuple with a NULL component matches nothing).  string_keys: string key columns as
        (heap, starts, lengths, nulls or None) tuples, after the numeric keys in the key tuple (ytgpu_join_table_build_strings);
        foreign_keys may then be empty.  The table owns a copy of the keys: the columns may be freed or overwritten once
        this returns."""
        return JoinTable(self, foreign_keys, nulls, string_keys)

    def groupby_table(self, key_types, string_key_count, value_types, aggregates, hint: int = 0,
                      string_value_count: int = 0) -> "GroupByTable":
        """ytgpu_groupby_table_create_strings: a GROUP BY table updated block by block (GroupByTable.update) whose result
        (GroupByTable.result) is the one-shot scan_filter_groupby_multi over all the blocks' rows.  key_types: the numeric
        keys' EValueTypes, followed in the key tuple by string_key_count string keys; value_types: the value columns every
        update passes, followed by string_value_count string value columns; aggregates [(op, column[, by_column])] over
        them (column len(value_types) + i is string value i)."""
        return GroupByTable(self, key_types, string_key_count, value_types, aggregates, hint, string_value_count)

    def gather_column(self, column: "Column", rows):
        """ytgpu_gather_column: `column` decoded at rows (uint32; capi.JOIN_NO_ROW gives NULL) -> dict(values, null_bitmap,
        null_count, column) in the rows' memory flavour, laid out as evaluate_expression's result: `column` is a Column over
        them (without the bitmap when no row is NULL)."""
        view = column.view()
        rp, mem = _ptr_mem(rows)
        count = rows.numel() if _is_tensor(rows) else rows.size
        values = self._out((count,), np.uint64, mem)
        null_bitmap = self._out(((count + 63) // 64 * 8,), np.uint8, mem)
        nulls = C.c_uint64(0)
        err = capi.Error()
        capi.check(self.lib.ytgpu_gather_column(self.handle, C.byref(view), rp, count, _ptr_mem(values)[0], _ptr_mem(null_bitmap)[0],
                                                C.byref(nulls), mem, C.byref(err)), err)
        out = Column(column.value_type, values=values, value_count=count, null_bitmap=null_bitmap if nulls.value else None)
        return dict(values=values, null_bitmap=null_bitmap, null_count=int(nulls.value), column=out)

    def gather_string_column(self, heap, starts, lengths, nulls, rows):
        """ytgpu_gather_string_column: the string column (heap, starts, lengths, nulls or None) at rows -> (heap, starts,
        lengths, null_bytemap), the gathered arrays in the rows' memory flavour and the heap itself, not copied."""
        scol = _string_column(heap, starts, lengths, nulls)
        rp, mem = _ptr_mem(rows)
        count = rows.numel() if _is_tensor(rows) else rows.size
        ostarts = self._out((count,), np.uint64, mem)
        olengths = self._out((count,), np.uint32, mem)
        onulls = self._out((count,), np.uint8, mem)
        err = capi.Error()
        capi.check(self.lib.ytgpu_gather_string_column(self.handle, C.byref(scol), rp, count, _ptr_mem(ostarts)[0], _ptr_mem(olengths)[0],
                                                       _ptr_mem(onulls)[0], mem, C.byref(err)), err)
        return heap, ostarts, olengths, onulls

    def order_rows(self, columns, string_columns=(), items=(), rows=None, offset: int = 0, limit: int | None = None,
                   count_only: bool = False, out_mem: int | None = None, row_count: int | None = None):
        """ORDER BY ... OFFSET ... LIMIT (ytgpu_order_rows).  columns: Column objects; string_columns: (heap, starts, lengths,
        nulls or None) per column; items: (column, is_string, descending) per ORDER BY item, column indexing columns or
        string_columns.  rows (uint32; None: every row of the item columns) are the rows to order.  -> the row indexes of
        sorted positions [offset, offset + limit) as uint32 (int32 tensors in DEVICE memory); with count_only, their number.
        The output is in the rows' memory; without rows in out_mem (default: the first item column's).  row_count overrides
        the number of rows passed to the call."""
        views = [c.view() for c in columns]
        sarr = (capi.StringColumn * max(len(string_columns), 1))()
        for i, column in enumerate(string_columns):
            sarr[i] = _string_column(*column)
        iarr = (capi.OrderItem * max(len(items), 1))()
        for i, (column, is_string, descending) in enumerate(items):
            iarr[i] = capi.OrderItem(column, int(bool(is_string)), int(bool(descending)), 0)
        first = items[0] if items else None
        column_mem, column_rows = capi.MEM_HOST, 0
        if first is not None and first[1] and first[0] < len(string_columns):
            column_mem, column_rows = sarr[first[0]].mem, int(sarr[first[0]].row_count)
        elif first is not None and not first[1] and first[0] < len(views):
            column_mem, column_rows = views[first[0]].mem, int(views[first[0]].value_count)
        if rows is not None:
            rp, rows_mem = _ptr_mem(rows)
            n = rows.numel() if _is_tensor(rows) else rows.size
        else:
            rp, rows_mem, n = None, column_mem, column_rows
        if row_count is not None:
            n = row_count
        if rows is not None or out_mem is None:
            out_mem = rows_mem
        if limit is None:
            limit = n
        count = C.c_uint64(0)
        err = capi.Error()
        window = min(limit, n - min(offset, n))
        out = None if count_only else self._out((max(window, 1),), np.uint32, out_mem)
        arr = (capi.ColumnView * max(len(views), 1))(*views)
        capi.check(self.lib.ytgpu_order_rows(self.handle, C.cast(arr, C.c_void_p), len(views), C.cast(sarr, C.c_void_p),
                                             len(string_columns), iarr, len(items), rp, n, offset, limit,
                                             _ptr_mem(out)[0] if out is not None else None, C.byref(count), out_mem, C.byref(err)), err)
        if count_only:
            return int(count.value)
        return out[:int(count.value)]

    @staticmethod
    def _program_columns(caller, columns, string_columns):
        """Column arrays of an evaluator call -> (ColumnView array, views, StringColumn array, mem and n of column 0)."""
        views = [c.view() for c in columns]
        sarr = (capi.StringColumn * max(len(string_columns), 1))()
        for i, column in enumerate(string_columns):
            sarr[i] = _string_column(*column)
        if views:
            mem, n = views[0].mem, int(views[0].value_count)
        elif string_columns:
            mem, n = sarr[0].mem, int(sarr[0].row_count)
        else:
            raise ValueError(f"{caller} needs at least one column")
        return (capi.ColumnView * max(len(views), 1))(*views), views, sarr, mem, n

    def evaluate_filter(self, columns, string_columns=(), program=(), list_values=(), string_constants=b"",
                        want_bitmap: bool = True, want_bytemap: bool = True, want_rows: bool = True,
                        rows_capacity: int | None = None):
        """WHERE expression (ytgpu_evaluate_filter) -> dict(bitmap, bytemap, rows, count).
        columns: Column objects; string_columns: (heap, starts, lengths, nulls or None) per column, node column
        len(columns) + i naming string column i.  program: postfix nodes, each a capi.FilterNode or a tuple
        (op, cmp, column, column2, constant, length); a LIKE node's column2 is its escape byte (-1: none).  list_values: IN entries (uint64 bit patterns; for a string column
        (offset << 32) | length into string_constants).  The outputs are in the inputs' memory flavour: bitmap
        8 * ceil(n / 64) bytes, bytemap n bytes, rows uint32 (int32 on the device) trimmed to the count; an output not
        wanted is None."""
        carr, views, sarr, mem, n = self._program_columns("evaluate_filter", columns, string_columns)
        nodes = (capi.FilterNode * max(len(program), 1))()
        for i, node in enumerate(program):
            if isinstance(node, capi.FilterNode):
                nodes[i] = node
            else:
                op, cmp, column, column2, constant, length = (tuple(node) + (0,) * 6)[:6]
                nodes[i] = capi.FilterNode(op, cmp, column, column2, int(constant) & 0xFFFFFFFFFFFFFFFF, length, 0)
        lv = np.ascontiguousarray(np.asarray(list_values, dtype=np.uint64).reshape(-1))
        sc = np.frombuffer(bytes(string_constants), dtype=np.uint8) if len(string_constants) else np.zeros(0, np.uint8)
        words = (n + 63) // 64
        bitmap = self._out((words * 8,), np.uint8, mem) if want_bitmap else None
        bytemap = self._out((n,), np.uint8, mem) if want_bytemap else None
        if rows_capacity is None:
            rows_capacity = n
        rows = self._out((max(rows_capacity, 1),), np.uint32, mem) if want_rows else None
        selected = C.c_uint64(0)
        err = capi.Error()
        code = self.lib.ytgpu_evaluate_filter(self.handle, C.cast(carr, C.c_void_p), len(views), C.cast(sarr, C.c_void_p),
                                              len(string_columns), C.cast(nodes, C.c_void_p), len(program),
                                              lv.ctypes.data if lv.size else None, lv.size, sc.ctypes.data if sc.size else None,
                                              sc.size, _ptr_mem(bitmap)[0], _ptr_mem(bytemap)[0], _ptr_mem(rows)[0], rows_capacity,
                                              C.byref(selected), mem, C.byref(err))
        count = int(selected.value)
        if code != capi.OK:
            e = capi.YtGpuError(code, err.message.decode(errors="replace"), err.cuda_error)
            e.selected = count  # the needed rows_capacity when that was too small
            raise e
        return dict(bitmap=bitmap, bytemap=bytemap, rows=rows[:count] if rows is not None else None, count=count)

    def evaluate_expression(self, columns, program, selection=None, string_columns=(), string_constants=b""):
        """Computed column (ytgpu_evaluate_expression) -> dict(values, null_bitmap, null_count, value_type, column).
        columns: Column objects; program: postfix nodes, each a capi.ExprNode or a tuple (op, column, type, constant).
        selection: nullable bitmap in ytgpu_evaluate_filter's layout (its "bitmap" output).  The outputs are in the inputs'
        memory flavour: values n uint64 (int64 on the device), null_bitmap 8 * ceil(n / 64) bytes; `column` is a Column
        over them (without the bitmap when no row is NULL), ready for scan_filter_groupby_multi / evaluate_filter.
        string_columns: (heap, starts, lengths, nulls or None) per column, node column len(columns) + i naming string column
        i; a STRING constant is (offset << 32) | length into string_constants (capi.ExprConstants builds it, IN lists and
        patterns and FORMAT_TIMESTAMP formats included).  With either, a string op, FORMAT_TIMESTAMP or an IN / STARTS_WITH / CONTAINS / LIKE in the program, or a STRING
        constant in a program with a conditional op, the call is ytgpu_evaluate_expression_strings, made twice: a type and size query, then the call that fills the outputs
        of that type, so a STRING result runs its size pass twice (a caller that knows the heap size calls the library once).
        A STRING result comes back as heap / starts / lengths / null_bytemap (values, null_bitmap and column None), ready
        for evaluate_filter's string_columns and string_value_ids."""
        carr, views, sarr, mem, n = self._program_columns("evaluate_expression", columns, string_columns)
        nodes = (capi.ExprNode * max(len(program), 1))()
        for i, node in enumerate(program):
            if isinstance(node, capi.ExprNode):
                nodes[i] = node
            else:
                op, column, vtype, constant = (tuple(node) + (0,) * 4)[:4]
                nodes[i].op, nodes[i].column, nodes[i].type = op, column, vtype
                nodes[i].constant = int(constant) & 0xFFFFFFFFFFFFFFFF
        words = (n + 63) // 64
        vtype, nulls = C.c_uint8(0), C.c_uint64(0)
        err = capi.Error()
        # the string entry point for string columns, constants bytes, string ops or predicates; a program with a conditional
        # op also for a STRING
        # constant (`x = ''`, `if(c, '', '')` name no bytes).  Programs of the earlier ops route as they always have.
        ops = [nodes[i].op for i in range(len(program))]
        conditional = any(op >= capi.EXPR_COMPARE for op in ops)
        string_constants = bytes(string_constants)
        strings = (bool(string_columns) or len(string_constants) > 0 or
                   any(op in capi.EXPR_STRING_OPS or op in capi.EXPR_PREDICATE_OPS or op == capi.EXPR_FORMAT_TIMESTAMP for op in ops) or
                   (conditional and any(nodes[i].op == capi.EXPR_CONSTANT and nodes[i].type == int(EValueType.String)
                                        for i in range(len(program)))))
        if not strings:
            values = self._out((n,), np.uint64, mem)
            null_bitmap = self._out((words * 8,), np.uint8, mem)
            capi.check(self.lib.ytgpu_evaluate_expression(self.handle, C.cast(carr, C.c_void_p), len(views), C.cast(nodes, C.c_void_p),
                                                          len(program), _ptr_mem(selection)[0], _ptr_mem(values)[0],
                                                          _ptr_mem(null_bitmap)[0], C.byref(vtype), C.byref(nulls), mem, C.byref(err)), err)
            column = Column(int(vtype.value), values=values, value_count=n,
                            null_bitmap=null_bitmap if nulls.value else None)
            return dict(values=values, null_bitmap=null_bitmap, null_count=int(nulls.value), value_type=int(vtype.value), column=column)
        sc = np.frombuffer(bytes(string_constants), dtype=np.uint8) if len(string_constants) else np.zeros(0, np.uint8)
        heap_bytes = C.c_uint64(0)

        def call(values=None, null_bitmap=None, heap=None, capacity=0, starts=None, lengths=None, null_bytemap=None):
            capi.check(self.lib.ytgpu_evaluate_expression_strings(
                self.handle, C.cast(carr, C.c_void_p), len(views), C.cast(sarr, C.c_void_p), len(string_columns),
                sc.ctypes.data if sc.size else None, sc.size, C.cast(nodes, C.c_void_p), len(program), _ptr_mem(selection)[0],
                _ptr_mem(values)[0], _ptr_mem(null_bitmap)[0], _ptr_mem(heap)[0], capacity, _ptr_mem(starts)[0],
                _ptr_mem(lengths)[0], _ptr_mem(null_bytemap)[0], C.byref(heap_bytes), C.byref(vtype), C.byref(nulls), mem,
                C.byref(err)), err)
        # a type and size query first (no launch for a numeric result, the size pass and scan for a STRING one), then the
        # call that fills the outputs of that type: a STRING result pays the size pass twice
        call()
        if int(vtype.value) != int(EValueType.String):
            values = self._out((n,), np.uint64, mem)
            null_bitmap = self._out((words * 8,), np.uint8, mem)
            if n:
                call(values, null_bitmap)
            column = Column(int(vtype.value), values=values, value_count=n,
                            null_bitmap=null_bitmap if nulls.value else None)
            return dict(values=values, null_bitmap=null_bitmap, null_count=int(nulls.value), value_type=int(vtype.value), column=column)
        size = int(heap_bytes.value)
        heap = self._out((max(size, 1),), np.uint8, mem)
        starts = self._out((n,), np.uint64, mem)
        lengths = self._out((n,), np.uint32, mem)
        null_bytemap = self._out((n,), np.uint8, mem)
        if n:
            call(heap=heap, capacity=size, starts=starts, lengths=lengths, null_bytemap=null_bytemap)
        return dict(values=None, null_bitmap=None, null_count=int(nulls.value), value_type=int(vtype.value), column=None,
                    heap=heap[:size], starts=starts, lengths=lengths, null_bytemap=null_bytemap)


class JoinTable:
    """A built join table (ytgpu_join_table); see GpuContext.join_table.  close() or a with block destroys it."""

    def __init__(self, ctx: GpuContext, foreign_keys, nulls: int, string_keys=()):
        self.ctx, self.handle = ctx, None
        views = [c.view() for c in foreign_keys]
        arr = (capi.ColumnView * max(len(views), 1))(*views)
        h = C.c_void_p()
        err = capi.Error()
        if string_keys:
            sarr = _string_columns(string_keys)
            capi.check(ctx.lib.ytgpu_join_table_build_strings(ctx.handle, C.cast(arr, C.c_void_p), len(views), C.cast(sarr, C.c_void_p),
                                                              len(string_keys), nulls, C.byref(h), C.byref(err)), err)
        else:
            capi.check(ctx.lib.ytgpu_join_table_build(ctx.handle, C.cast(arr, C.c_void_p), len(views), nulls, C.byref(h), C.byref(err)), err)
        self.handle = h
        if not hasattr(ctx, "_join_tables"):
            ctx._join_tables = weakref.WeakSet()
        ctx._join_tables.add(self)

    def probe(self, primary_keys, kind: int = capi.JOIN_INNER, count_only: bool = False, capacity: int | None = None,
              out_mem: int | None = None, string_keys=()):
        """ytgpu_join_table_probe with primary_keys (a list of Column), and string_keys as GpuContext.join_table takes them
        (ytgpu_join_table_probe_strings).  INNER / LEFT -> (primary rows, foreign rows) as GpuContext.hash_join returns
        them; SEMI / ANTI -> the ascending primary rows (uint32; int32 tensors in DEVICE memory); with count_only, the
        count.  The outputs are in out_mem (default: the primary keys' memory).  Without a capacity, SEMI / ANTI size the
        output for every primary row and INNER / LEFT run a count query first; a capacity below the count raises
        YtGpuError with .pair_count set."""
        if self.handle is None:
            raise ValueError("the join table is closed")
        views = [c.view() for c in primary_keys]
        sarr = _string_columns(string_keys) if string_keys else None
        if out_mem is None:
            out_mem = views[0].mem if views else (sarr[0].mem if string_keys else capi.MEM_HOST)
        arr = (capi.ColumnView * max(len(views), 1))(*views)
        rows_only = kind in (capi.JOIN_SEMI, capi.JOIN_ANTI)
        count = C.c_uint64(0)
        err = capi.Error()

        def call(prim=None, fore=None, cap=0):
            if string_keys:
                code = self.ctx.lib.ytgpu_join_table_probe_strings(self.ctx.handle, self.handle, C.cast(arr, C.c_void_p), len(views),
                                                                   C.cast(sarr, C.c_void_p), len(string_keys), kind, _ptr_mem(prim)[0],
                                                                   _ptr_mem(fore)[0], cap, C.byref(count), out_mem, C.byref(err))
            else:
                code = self.ctx.lib.ytgpu_join_table_probe(self.ctx.handle, self.handle, C.cast(arr, C.c_void_p), len(views), kind,
                                                           _ptr_mem(prim)[0], _ptr_mem(fore)[0], cap, C.byref(count), out_mem, C.byref(err))
            if code != capi.OK:
                e = capi.YtGpuError(code, err.message.decode(errors="replace"), err.cuda_error)
                e.pair_count = int(count.value)
                raise e
        if count_only:
            call()
            return int(count.value)
        if capacity is None:
            if rows_only:
                capacity = views[0].value_count if views else (sarr[0].row_count if string_keys else 0)
            else:
                call()
                capacity = int(count.value)
        prim = self.ctx._out((max(capacity, 1),), np.uint32, out_mem)
        if rows_only:
            call(prim, None, capacity)
            return prim[:int(count.value)]
        fore = self.ctx._out((max(capacity, 1),), np.uint32, out_mem)
        call(prim, fore, capacity)
        pairs = int(count.value)
        return prim[:pairs], fore[:pairs]

    def close(self):
        if self.handle is not None:
            if getattr(self.ctx, "handle", None):
                err = capi.Error()
                capi.check(self.ctx.lib.ytgpu_join_table_destroy(self.handle, C.byref(err)), err)
            self.handle = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class GroupByTable:
    """A GROUP BY table (ytgpu_groupby_table); see GpuContext.groupby_table.  close() or a with block destroys it."""

    def __init__(self, ctx: GpuContext, key_types, string_key_count: int, value_types, aggregates, hint: int = 0,
                 string_value_count: int = 0):
        self.ctx, self.handle = ctx, None
        self.numeric, self.strings, self.aggregate_count = len(key_types), string_key_count, len(aggregates)
        # string-valued aggregates: MIN / MAX / FIRST of a string, ARGMIN / ARGMAX whose column is a string
        self.value_strings = sum(1 for a in aggregates if a[1] >= len(value_types) and a[0] != capi.AGG_COUNT)
        kt = (C.c_uint8 * max(len(key_types), 1))(*[int(t) for t in key_types])
        vt = (C.c_uint8 * max(len(value_types), 1))(*[int(t) for t in value_types])
        aggs = (capi.Aggregate * max(len(aggregates), 1))()
        for i, a in enumerate(aggregates):
            aggs[i].op, aggs[i].column = a[0], a[1]
            aggs[i].by_column = a[2] if len(a) > 2 else -1
        h = C.c_void_p()
        err = capi.Error()
        capi.check(ctx.lib.ytgpu_groupby_table_create_strings(ctx.handle, C.cast(kt, C.c_void_p), len(key_types), string_key_count,
                                                              C.cast(vt, C.c_void_p), len(value_types), string_value_count,
                                                              C.cast(aggs, C.c_void_p), len(aggregates), hint, C.byref(h), C.byref(err)), err)
        self.handle = h
        if not hasattr(ctx, "_groupby_tables"):
            ctx._groupby_tables = weakref.WeakSet()
        ctx._groupby_tables.add(self)

    def update(self, key_cols, value_cols, string_keys=(), predicate=None, predicate_column: int = -1, string_values=()):
        """ytgpu_groupby_table_update_strings with key_cols and value_cols (lists of Column) and string_keys and
        string_values as (heap, starts, lengths, nulls or None) tuples; predicate (op, constant) over
        value_cols[predicate_column]."""
        if self.handle is None:
            raise ValueError("the GROUP BY table is closed")
        kviews = [c.view() for c in key_cols]
        vviews = [c.view() for c in value_cols]
        karr = (capi.ColumnView * max(len(kviews), 1))(*kviews)
        varr = (capi.ColumnView * max(len(vviews), 1))(*vviews)
        sarr = _string_columns(string_keys) if string_keys else None
        varr_s = _string_columns(string_values) if string_values else None
        pred = None
        if predicate is not None:
            op, const = predicate
            pred = capi.Predicate(op, 0, const & 0xFFFFFFFFFFFFFFFF)
        err = capi.Error()
        capi.check(self.ctx.lib.ytgpu_groupby_table_update_strings(
            self.ctx.handle, self.handle, C.cast(karr, C.c_void_p), len(kviews), C.cast(sarr, C.c_void_p) if sarr is not None else None,
            len(string_keys), C.cast(varr, C.c_void_p), len(vviews), C.cast(varr_s, C.c_void_p) if varr_s is not None else None,
            len(string_values), C.cast(C.pointer(pred), C.c_void_p) if pred is not None else None, predicate_column, C.byref(err)), err)

    def _call_result(self, res, skeys, svals, out_mem):
        err = capi.Error()
        sarr = (capi.GroupByStringKeys * max(self.strings, 1))(*skeys)
        varr = (capi.GroupByStringKeys * max(self.value_strings, 1))(*svals)
        code = self.ctx.lib.ytgpu_groupby_table_result_strings(self.ctx.handle, self.handle, C.byref(res), C.cast(sarr, C.c_void_p),
                                                               self.strings, C.cast(varr, C.c_void_p), self.value_strings, out_mem,
                                                               C.byref(err))
        return code, err, [int(sarr[s].heap_bytes) for s in range(self.strings)] + [int(varr[s].heap_bytes) for s in range(self.value_strings)]

    def result(self, count_only: bool = False, out_mem: int = capi.MEM_HOST, capacity: int | None = None, heap_capacity=None):
        """ytgpu_groupby_table_result_strings -> dict(keys=[...], key_null=[...], values=[...], value_null=[...], count,
        first_row, string_keys=[(heap, starts, lengths, nulls)], string_values=[(heap, starts, lengths, nulls)]) in
        first-seen order, in out_mem; with count_only, the group count.  string_values: one per string-valued aggregate,
        in aggregate order.  heap_capacity: one per string key, then one per string value.  Without capacities a count
        query sizes the outputs first; a capacity below the need raises YtGpuError with .group_count and .heap_bytes
        (keys, then values) set."""
        if self.handle is None:
            raise ValueError("the GROUP BY table is closed")
        zero = [capi.GroupByStringKeys() for _ in range(self.strings + self.value_strings)]
        empty = (C.c_void_p * 1)()
        if count_only or capacity is None or heap_capacity is None:
            res = capi.GroupByMultiResult(0, 0, empty, empty, empty, empty, None, None)
            code, err, heap_bytes = self._call_result(res, zero[:self.strings], zero[self.strings:], out_mem)
            if code not in (capi.OK, capi.ERR_INVALID_ARGUMENT) or (code != capi.OK and res.group_count == 0):
                capi.check(code, err)
            if count_only:
                return int(res.group_count)
            capacity = int(res.group_count) if capacity is None else capacity
            heap_capacity = heap_bytes if heap_capacity is None else heap_capacity
        out = self.ctx._out
        cap = max(capacity, 1)
        keys = [out((cap,), np.uint64, out_mem) for _ in range(self.numeric)]
        kn = [out((cap,), np.uint8, out_mem) for _ in range(self.numeric)]
        vals = [out((cap,), np.uint64, out_mem) for _ in range(self.aggregate_count)]
        vn = [out((cap,), np.uint8, out_mem) for _ in range(self.aggregate_count)]
        counts = out((cap,), np.uint64, out_mem)
        first = out((cap,), np.uint64, out_mem)
        sout = [(out((max(hc, 1),), np.uint8, out_mem), out((cap,), np.uint64, out_mem), out((cap,), np.uint32, out_mem),
                 out((cap,), np.uint8, out_mem)) for hc in heap_capacity]

        def ptrs(arrs):
            return (C.c_void_p * max(len(arrs), 1))(*[_ptr_mem(a)[0] for a in arrs])
        pk, pkn, pv, pvn = ptrs(keys), ptrs(kn), ptrs(vals), ptrs(vn)
        res = capi.GroupByMultiResult(0, capacity, pk, pkn, pv, pvn, _ptr_mem(counts)[0], _ptr_mem(first)[0])
        skeys = [capi.GroupByStringKeys(_ptr_mem(h)[0], hc, 0, _ptr_mem(st)[0], _ptr_mem(ln)[0], _ptr_mem(nl)[0])
                 for (h, st, ln, nl), hc in zip(sout, heap_capacity)]
        code, err, heap_bytes = self._call_result(res, skeys[:self.strings], skeys[self.strings:], out_mem)
        if code != capi.OK:
            e = capi.YtGpuError(code, err.message.decode(errors="replace"), err.cuda_error)
            e.group_count, e.heap_bytes = int(res.group_count), heap_bytes
            raise e
        g = int(res.group_count)
        strings = [(h[:hb], st[:g], ln[:g], nl[:g]) for (h, st, ln, nl), hb in zip(sout, heap_bytes)]
        return dict(keys=[k[:g] for k in keys], key_null=[k[:g] for k in kn], values=[v[:g] for v in vals],
                    value_null=[v[:g] for v in vn], count=counts[:g], first_row=first[:g], string_keys=strings[:self.strings],
                    string_values=strings[self.strings:])

    def close(self):
        if self.handle is not None:
            if getattr(self.ctx, "handle", None):
                err = capi.Error()
                capi.check(self.ctx.lib.ytgpu_groupby_table_destroy(self.handle, C.byref(err)), err)
            self.handle = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Column:
    """Host- or device-side description of IUnversionedColumnarRowBatch::TColumn (row_batch.h:49-191)."""

    def __init__(self, value_type, values=None, bit_width=64, start_index=0, value_count=None, base_value=0,
                 zigzag=False, null_bitmap=None, dictionary_indexes=None, rle_indexes=None, arrow_validity=False):
        self.value_type = value_type
        self.arrow_validity = arrow_validity  # null_bitmap holds Arrow validity bits (1 = valid)
        self.values = values
        self.bit_width = bit_width
        self.start_index = start_index
        self.base_value = base_value
        self.zigzag = zigzag
        self.null_bitmap = null_bitmap
        self.dictionary_indexes = dictionary_indexes
        self.rle_indexes = rle_indexes
        if value_count is None:
            if rle_indexes is not None:
                raise ValueError("value_count is required for RLE columns")
            src = dictionary_indexes if dictionary_indexes is not None else values
            value_count = (src.numel() if _is_tensor(src) else len(src)) - start_index
        self.value_count = int(value_count)

    def _len(self, x):
        return 0 if x is None else (x.numel() if _is_tensor(x) else x.size)

    def view(self) -> capi.ColumnView:
        vp, mem = _ptr_mem(self.values)
        if self.values is None:
            for other in (self.null_bitmap, self.dictionary_indexes, self.rle_indexes):
                if other is not None:
                    mem = _ptr_mem(other)[1]
        v = capi.ColumnView()
        v.start_index = self.start_index
        v.value_count = self.value_count
        v.value_type = self.value_type
        v.has_values = int(self.values is not None)
        v.zigzag = int(bool(self.zigzag))
        v.bit_width = self.bit_width
        v.reserved = 1 if self.arrow_validity else 0  # YTGPU_COLUMN_ARROW_VALIDITY
        v.base_value = self.base_value & 0xFFFFFFFFFFFFFFFF
        v.values = vp
        v.values_count = self._len(self.values) * (8 if self.bit_width == 1 else 1)  # a TBitmap holds 8 values per byte
        v.null_bitmap = _ptr_mem(self.null_bitmap)[0]
        v.dictionary_indexes = _ptr_mem(self.dictionary_indexes)[0]
        v.dictionary_index_count = self._len(self.dictionary_indexes)
        v.rle_indexes = _ptr_mem(self.rle_indexes)[0]
        v.rle_count = self._len(self.rle_indexes)
        v.mem = mem
        v._keep = (self.values, self.null_bitmap, self.dictionary_indexes, self.rle_indexes)
        return v
