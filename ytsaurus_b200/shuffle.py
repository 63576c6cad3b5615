"""In-box multi-GPU sort: range partition -> all-to-all over NVLink -> local sort.

The reference materialises its shuffle through intermediate chunks: Partition jobs tag blocks with a
partition index (yt/yt/ytlib/table_client/schemaless_chunk_writer.cpp:1604-1667), Sort jobs fetch the
blocks of their partition over RPC (partition_chunk_reader.cpp:82-86), pivots come from sampled keys
(yt/yt/server/controller_agent/helpers.cpp:263-425).  Inside one 8-GPU box the same structure is one
collective: every rank range-partitions its rows with the ordered partitioner (bit-identical partition
indices), the per-destination slabs travel in one NCCL all_to_all_single, and each rank sorts what it
received.  Rank r ends up with key range r, so the concatenation over ranks is globally sorted.

torch.distributed is plumbing (rendezvous, NCCL); every compute step is a libytgpu.so call made
through the `ops` object (GpuContext in production; tests inject a checker-backed double to exercise
the host logic under gloo on CPU).
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch
import torch.distributed as dist

from . import capi
from .partition_keys import PartitionKey, build_partition_keys_from_sorted_samples
from .rowset import EValueType, Rowset, VALUE_DTYPE

SAMPLES_PER_PARTITION = 1000  # TSortOperationSpecBase::SamplesPerPartition (ytlib/scheduler/config.h:2134-2300)


@dataclass
class ShuffleStats:
    rows_in: int
    rows_out: int
    sent: list
    received: list


def pivot_bounds_from_rows(pivot_rows: np.ndarray, key_columns) -> tuple[Rowset, list, list]:
    """pivot_rows: [P-1, row_bytes] uint8 (host).  -> (bounds rowset incl. the universal bound 0,
    prefix lengths, inclusiveness) — inclusive lower bounds, as CreatePartitioner builds them
    (yt/yt/ytlib/job_proxy/helpers.cpp:113-147)."""
    k = len(key_columns)
    p1 = pivot_rows.shape[0]
    vals = np.zeros((p1 + 1, k), dtype=VALUE_DTYPE)
    heap = bytearray()
    for b in range(p1):
        for c, col in enumerate(key_columns):
            off, width, typ = col[0], col[1], col[2]
            v = vals[b + 1, c]
            v["id"] = c
            v["type"] = typ
            if typ == EValueType.String:
                v["length"] = width
                v["data"] = len(heap)
                heap += pivot_rows[b, off:off + width].tobytes()
            elif typ == EValueType.Boolean:
                v["data"] = int(pivot_rows[b, off] != 0)
            else:
                v["data"] = int(pivot_rows[b, off:off + 8].copy().view(np.uint64)[0])
    bounds = Rowset(vals, np.frombuffer(bytes(heap) or b"\0", dtype=np.uint8).copy())
    return bounds, [0] + [k] * p1, [1] * (p1 + 1)


class PeerMemoryUnavailable(RuntimeError):
    """CUDA IPC peer mappings could not be established on some rank (raised on every rank together)."""


class ShuffleSorter:
    """Distributed sort of fixed-width rows across the ranks of a process group."""

    def __init__(self, ops, group=None):
        self.ops = ops
        self.group = group
        self.world = dist.get_world_size(group)
        self.rank = dist.get_rank(group)

    # -- host logic -------------------------------------------------------------------------
    def _sample(self, rows2d: torch.Tensor) -> torch.Tensor:
        n = rows2d.shape[0]
        want = SAMPLES_PER_PARTITION * self.world
        take = min(n, want)
        if take == 0:
            return rows2d[:0]
        idx = (torch.arange(take, dtype=torch.int64, device=rows2d.device) * (n - 1)) // max(take - 1, 1)
        return rows2d.index_select(0, idx)

    def _gather_samples(self, sample: torch.Tensor, row_bytes: int) -> torch.Tensor:
        want = SAMPLES_PER_PARTITION * self.world
        padded = torch.zeros((want, row_bytes), dtype=torch.uint8, device=sample.device)
        padded[: sample.shape[0]] = sample
        counts = torch.tensor([sample.shape[0]], dtype=torch.int64, device=sample.device)
        all_counts = [torch.zeros_like(counts) for _ in range(self.world)]
        all_samples = [torch.zeros_like(padded) for _ in range(self.world)]
        dist.all_gather(all_counts, counts, group=self.group)
        dist.all_gather(all_samples, padded, group=self.group)
        parts = [s[: int(c.item())] for s, c in zip(all_samples, all_counts)]
        return torch.cat(parts, dim=0)

    def _exchange(self, slabs2d: torch.Tensor, send_counts: torch.Tensor):
        """all-to-all-v of row slabs; returns (received rows [m, row_bytes], recv_counts)."""
        recv_counts = torch.zeros_like(send_counts)
        dist.all_to_all_single(recv_counts, send_counts, group=self.group)
        send = [int(x) for x in send_counts.cpu().tolist()]
        recv = [int(x) for x in recv_counts.cpu().tolist()]
        out = torch.empty((sum(recv), slabs2d.shape[1]), dtype=torch.uint8, device=slabs2d.device)
        dist.all_to_all_single(out, slabs2d, output_split_sizes=recv, input_split_sizes=send, group=self.group)
        return out, send, recv

    def _plan_partitions(self, rows2d: torch.Tensor, row_bytes: int, key_columns):
        """Sample -> sort the samples with the same kernels -> BuildPartitionKeysFromSamples (partition_keys.py).
        Every rank computes the identical spec.  -> (partition spec or None when there are no rows anywhere,
        maniac flags per partition)."""
        P = self.world
        samples = self._gather_samples(self._sample(rows2d), row_bytes)
        if samples.shape[0] == 0:
            return None, [False] * P
        sorted_samples, _ = self.ops.sort_fixed_rows(samples.reshape(-1), row_bytes, key_columns)
        ss = sorted_samples.view(-1, row_bytes).cpu().numpy()
        m = ss.shape[0]
        cols = [(c[0], c[1] if c[2] == EValueType.String else (1 if c[2] == EValueType.Boolean else 8)) for c in key_columns]

        def same_key(a: int, b: int) -> bool:
            return all(bytes(ss[a, off:off + w]) == bytes(ss[b, off:off + w]) for off, w in cols)

        keys = build_partition_keys_from_sorted_samples(m, same_key, np.ones(m, dtype=np.int64), np.zeros(m, dtype=bool), P)
        while len(keys) < P - 1:  # fewer distinct pivots than ranks: duplicate bounds are legal, those ranks get nothing
            keys.append(PartitionKey(keys[-1].sample, keys[-1].inclusive) if keys else PartitionKey(0, True))
        pivot_rows = ss[[k.sample for k in keys]] if keys else ss[:0]
        bounds, blen, _ = pivot_bounds_from_rows(pivot_rows, key_columns)
        binc = [1] + [int(k.inclusive) for k in keys]
        maniac = [False] + [k.maniac for k in keys]
        spec = self.ops._partition_spec(capi.PARTITION_ORDERED, P, key_columns=key_columns, bounds=bounds,
                                        bound_prefix_length=blen, bound_inclusive=binc)
        return spec, maniac

    def _local_sort(self, received: torch.Tensor, row_bytes: int, key_columns, maniac: bool):
        if maniac:  # a maniac partition holds a single key: already in (source rank, position) order
            return received.clone()
        out, _ = self.ops.sort_fixed_rows(received, row_bytes, key_columns)
        return out

    # -- the sort ---------------------------------------------------------------------------
    def sort(self, rows: torch.Tensor, row_bytes: int, key_columns):
        """rows: uint8 tensor (n*row_bytes) on this rank's device.  key_columns: fixed-row key columns
        (offset, width, type, descending, required).  -> (sorted rows of this rank's key range, stats)."""
        rows2d = rows.view(-1, row_bytes)
        n = rows2d.shape[0]
        # 1. sample -> identical pivots on every rank
        spec, maniac = self._plan_partitions(rows2d, row_bytes, key_columns)
        if spec is None:
            return rows.clone(), ShuffleStats(n, n, [n], [n])
        # 2. partition into per-destination slabs (stable)
        _, hist, slabs = self.ops.partition_fixed_rows(rows, row_bytes, spec, want_index=False, want_slabs=True)
        send_counts = hist if isinstance(hist, torch.Tensor) else torch.from_numpy(hist.astype(np.int64))
        send_counts = send_counts.to(torch.int64).to(rows.device)
        # 3. exchange over NVLink
        received, send, recv = self._exchange(slabs.view(-1, row_bytes), send_counts)
        # 4. local sort of this rank's key range
        out = self._local_sort(received.reshape(-1), row_bytes, key_columns, maniac[self.rank])
        return out, ShuffleStats(n, received.shape[0], send, recv)


class _DevicePointerArray:
    """Zero-copy torch view of device memory owned by libytgpu (a peer receive buffer)."""

    def __init__(self, ptr: int, nbytes: int):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (ptr, False), "version": 2}


class PeerShuffleSorter(ShuffleSorter):
    """Same sort, but rows never pass through NCCL: the partition step's slab scatter writes every
    destination's rows straight into that GPU's receive buffer over NVLink (CUDA IPC peer mappings,
    ytgpu_scatter_rows_to_peers).  torch.distributed only carries the 64-byte IPC handles (once) and the
    g x g row-count matrix plus two barriers per sort."""

    def __init__(self, ops, capacity_rows: int, row_bytes: int, group=None):
        super().__init__(ops, group)
        self.row_bytes = row_bytes
        self.capacity_rows = capacity_rows
        nbytes = capacity_rows * row_bytes
        dev = torch.device("cuda", ops.device)
        # Every step below is followed by an agreement round: if any rank cannot create or map a buffer,
        # ALL ranks raise PeerMemoryUnavailable together (callers then switch to the NCCL path in step).
        self.local_ptr, handle, problem = None, bytes(64), ""
        try:
            self.local_ptr, handle = ops.peer_buffer_create(nbytes)
        except Exception as e:  # noqa: BLE001
            problem = f"create: {e}"
        self._agree(problem, dev)
        self.local = torch.as_tensor(_DevicePointerArray(self.local_ptr, nbytes), device=dev)
        mine = torch.tensor(list(handle), dtype=torch.uint8, device=dev)
        handles = [torch.zeros_like(mine) for _ in range(self.world)]
        dist.all_gather(handles, mine, group=self.group)
        self.peer_ptrs = []
        try:
            for r, h in enumerate(handles):
                self.peer_ptrs.append(self.local_ptr if r == self.rank else ops.peer_buffer_open(bytes(h.cpu().tolist())))
        except Exception as e:  # noqa: BLE001
            problem = f"open: {e}"
        self._agree(problem, dev)

    def _agree(self, problem: str, dev):
        bad = torch.tensor([1 if problem else 0], dtype=torch.int32, device=dev)
        dist.all_reduce(bad, op=dist.ReduceOp.MAX, group=self.group)
        if int(bad.item()):
            raise PeerMemoryUnavailable(problem or "another rank could not set up its peer buffers")

    def close(self):
        torch.cuda.synchronize()
        dist.barrier(group=self.group)
        for r, p in enumerate(self.peer_ptrs):
            if r != self.rank:
                self.ops.peer_buffer_close(p)
        self.peer_ptrs = []
        self.local = None
        self.ops.peer_buffer_destroy(self.local_ptr)

    def sort(self, rows: torch.Tensor, row_bytes: int, key_columns):
        assert row_bytes == self.row_bytes
        rows2d = rows.view(-1, row_bytes)
        n = rows2d.shape[0]
        P = self.world
        spec, maniac = self._plan_partitions(rows2d, row_bytes, key_columns)
        if spec is None:
            return rows.clone(), ShuffleStats(n, n, [n], [n])
        # partition index + histogram only (no local slab copy)
        idx, hist, _ = self.ops.partition_fixed_rows(rows, row_bytes, spec, want_index=True, want_slabs=False)
        mine = hist.to(torch.int64)
        counts = [torch.zeros_like(mine) for _ in range(P)]
        dist.all_gather(counts, mine, group=self.group)           # counts[src][dst]
        H = torch.stack(counts).cpu().tolist()
        recv = [H[s][self.rank] for s in range(P)]
        total_in = sum(recv)
        for d in range(P):
            if sum(H[s][d] for s in range(P)) > self.capacity_rows:
                raise RuntimeError(f"rank {d} would receive more rows than its receive buffer holds "
                                   f"({self.capacity_rows}): raise capacity_rows")
        # my slab for destination d starts after the slabs of lower-ranked sources
        dest = [self.peer_ptrs[d] + sum(H[s][d] for s in range(self.rank)) * row_bytes for d in range(P)]
        dist.barrier(group=self.group)  # every rank is done reading its receive buffer from the previous sort
        self.ops.scatter_rows_to_peers(rows, row_bytes, idx, H[self.rank], dest)
        torch.cuda.synchronize()
        dist.barrier(group=self.group)  # all slabs have landed
        received = self.local[: total_in * row_bytes]
        out = self._local_sort(received, row_bytes, key_columns, maniac[self.rank])
        return out, ShuffleStats(n, total_in, H[self.rank], recv)


class NativeShuffleSorter:
    """The in-box distributed sort behind the C ABI (ytgpu_shuffle_*, csrc/shuffle.cu): sampling, pivot selection,
    partitioning, the count exchange, the barriers and the row scatter are kernels that talk through peer-mapped
    device memory; this class only gathers the 64-byte IPC handles once (torch.distributed is the plumbing a job
    proxy replaces with its own RPC) and forwards sort() to ytgpu_shuffle_sort."""

    def __init__(self, ops, capacity_rows: int, row_bytes: int, group=None):
        self.ops = ops
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.row_bytes = row_bytes
        self.capacity_rows = capacity_rows
        self.dev = getattr(ops, "torch_device", None) or torch.device("cuda", ops.device)  # tests inject a CPU double
        self.handle, problem, ipc = None, "", bytes(64)
        try:
            self.handle, ipc = ops.shuffle_create(self.world, self.rank, capacity_rows, row_bytes)
        except Exception as e:  # noqa: BLE001
            problem = f"create: {e}"
        self._agree(problem)
        if self.world > 1:
            mine = torch.tensor(list(ipc), dtype=torch.uint8, device=self.dev)
            handles = [torch.zeros_like(mine) for _ in range(self.world)]
            dist.all_gather(handles, mine, group=self.group)
            try:
                ops.shuffle_connect(self.handle, b"".join(bytes(h.cpu().tolist()) for h in handles))
            except Exception as e:  # noqa: BLE001
                problem = f"connect: {e}"
            self._agree(problem)
        self._out = None

    def _agree(self, problem: str):
        """All ranks raise PeerMemoryUnavailable together when any of them failed (callers then switch paths in step)."""
        if self.world == 1:
            if problem:
                raise PeerMemoryUnavailable(problem)
            return
        bad = torch.tensor([1 if problem else 0], dtype=torch.int32, device=self.dev)
        dist.all_reduce(bad, op=dist.ReduceOp.MAX, group=self.group)
        if int(bad.item()):
            raise PeerMemoryUnavailable(problem or "another rank could not set up its peer buffers")

    def sort(self, rows: torch.Tensor, row_bytes: int, key_columns, out: torch.Tensor | None = None):
        """Collective.  -> (sorted rows of this rank's key range (a view of `out` / an internal buffer), ShuffleStats)."""
        assert row_bytes == self.row_bytes
        if out is None:
            if self._out is None:
                self._out = torch.empty(self.capacity_rows * row_bytes, dtype=torch.uint8, device=self.dev)
            out = self._out
        m, st = self.ops.shuffle_sort(self.handle, rows, row_bytes, key_columns, out)
        stats = ShuffleStats(int(st.rows_in), int(st.rows_out), [int(st.sent[q]) for q in range(self.world)],
                             [int(st.received[q]) for q in range(self.world)])
        return out[: m * row_bytes], stats

    def close(self):
        if self.handle is not None:
            if self.dev.type == "cuda":
                torch.cuda.synchronize()
            if self.world > 1:
                dist.barrier(group=self.group)
            self.ops.shuffle_destroy(self.handle)
            self.handle = None
            self._out = None


def distributed_groupby(ops, key_col, val_col, predicate=None, group_count_hint: int = 0, group=None):
    """SELECT key, SUM(val), COUNT(*) GROUP BY key over row shards held by the ranks of `group`.

    The shape the reference uses for distributed aggregation (CHYT secondary queries: partial aggregate per
    instance + merge on the initiator; YT QL Intermediate -> Aggregated stream tags,
    library/query/engine/cg_routines/registry.cpp:1783-1834): every rank aggregates its shard with the fused
    scan->filter->group-by kernel, the partial (key, sum, count) states are hash-partitioned by key over the ranks
    (all_to_all_single), and each rank merges the states of its keys with the same kernel (SUM of sums, SUM of
    counts).  Integer results are exact; rank r returns the groups with key % world == r (NULL key: rank 0),
    ordered by key."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    part = ops.scan_filter_groupby(key_col, val_col, predicate, group_count_hint=group_count_hint)
    if world == 1:
        return part
    from .runtime import Column
    dev = part["keys"].device
    g = part["keys"].numel()
    keys = part["keys"].to(torch.int64)
    dest = torch.where(part["key_null"].bool(), torch.zeros_like(keys), torch.remainder(keys, world))  # int64 % world >= 0
    order = torch.argsort(dest, stable=True)
    counts = torch.bincount(dest, minlength=world).to(torch.int64)
    recv_counts = torch.zeros_like(counts)
    dist.all_to_all_single(recv_counts, counts, group=group)
    send, recv = counts.cpu().tolist(), recv_counts.cpu().tolist()

    def exchange(t):
        t = t.index_select(0, order).contiguous()
        out = torch.empty((sum(recv),), dtype=t.dtype, device=dev)
        dist.all_to_all_single(out, t, output_split_sizes=recv, input_split_sizes=send, group=group)
        return out

    rk, rs, rc = exchange(keys), exchange(part["sum"].to(torch.int64)), exchange(part["count"].to(torch.int64))
    rkn, rsn = exchange(part["key_null"]), exchange(part["sum_null"])
    m = rk.numel()
    if m == 0:
        return {k: v[:0] for k, v in part.items()}
    # bitmaps for the merge: NULL keys and "no non-null value seen" partial sums
    def bitmap(flags):
        f = flags.to(torch.uint8).cpu().numpy()
        return torch.from_numpy(np.packbits(f, bitorder="little")).to(dev)

    kcol = Column(EValueType.Uint64, values=rk, null_bitmap=bitmap(rkn) if bool(rkn.any()) else None)
    vtype = val_col.value_type
    scol = Column(vtype, values=rs, null_bitmap=bitmap(rsn) if bool(rsn.any()) else None)
    ccol = Column(EValueType.Uint64, values=rc)
    hint = m  # the received partial states are an upper bound on this rank's groups
    sums = ops.scan_filter_groupby(kcol, scol, None, group_count_hint=hint, capacity=m + 2)
    cnts = ops.scan_filter_groupby(kcol, ccol, None, group_count_hint=hint, capacity=m + 2)
    return dict(keys=sums["keys"], key_null=sums["key_null"], sum=sums["sum"], sum_null=sums["sum_null"],
                count=cnts["sum"])
