"""ytgpu_scatter_rows_to_peers on one GPU, across partition counts, row widths, row counts and index shapes.

The scatter writes every row to the slab of its partition, the rows of one partition in input order.  Its destinations
are plain device pointers, so one GPU runs every path of it with each partition pointed at a local buffer:
  - up to 32 partitions, the streaming kernel: 64-byte rows through the warp transpose, which stores each round of 32
    rows in destination order, every other width through the per-row copy loop; tiles of 1024 rows, rounds of 32,
    partition-bit ballots that change width between 16/17 and 31/32 partitions;
  - 33 to 4096 partitions, the many-partition path: a radix sort of the index, then a gather that finds each row's
    partition by binary search over the slab starts.  YTGPU_SCATTER_STREAM=0 forces it at any count, but the library
    reads that variable once per process, so those cases run in a child process that imports this module.

The reference for partition p's slab is the input rows whose index is p, in input order.  Every destination byte is a
sentinel before the call; after it, the slabs must hold exactly the reference rows and every byte around them must
still be the sentinel.  A rejected call must leave every destination byte untouched and the context usable.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from ytsaurus_b200 import capi

SENTINEL = 0xA5
GUARD = 64  # sentinel bytes before and after each destination buffer; a multiple of 16 keeps the slabs aligned
STREAM_PARTS = [1, 2, 3, 16, 17, 31, 32]
MANY_PARTS = [33, 257, 3071, 3072, 4096]  # from 3072 on, slab starts and pointers together would pass 48 KiB of shared memory
ROW_WIDTHS = [16, 32, 48, 64, 80, 128, 256]  # 64: the warp transpose; every other width: the per-row copy loop
ROW_COUNTS = [0, 1, 31, 32, 33, 1023, 1024, 1025, 4095, 4097, 150_001]
LAYOUTS = ["tensors", "contiguous", "peer"]
# all_*: one partition holds every row, so on the many-partition path the index sort skips every digit and returns the
# identity permutation; sorted: the digit passes run and produce the identity
SHAPES = ["uniform", "all_first", "all_last", "all_middle", "empty_ends_and_middle", "sorted", "runs_31_32_33", "skew_99"]


# ---- references (host only) ----
def make_index(shape, n, parts, rng):
    """Partition index (int32) of n rows over `parts` partitions."""
    mid = parts // 2
    if shape == "uniform":
        idx = rng.integers(0, parts, n)
    elif shape == "all_first":
        idx = np.zeros(n)
    elif shape == "all_last":
        idx = np.full(n, parts - 1)
    elif shape == "all_middle":
        idx = np.full(n, mid)
    elif shape == "empty_ends_and_middle":  # needs parts >= 4
        live = np.setdiff1d(np.arange(parts), [0, mid, parts - 1])
        idx = live[rng.integers(0, len(live), n)]
    elif shape == "sorted":
        idx = np.sort(rng.integers(0, parts, n))
    elif shape == "runs_31_32_33":  # runs of equal indices around the 32-row round of the streaming kernel
        lengths = np.resize([31, 32, 33], n // 31 + 1)
        idx = np.repeat(rng.integers(0, parts, len(lengths)), lengths)[:n]
    elif shape == "skew_99":
        idx = rng.integers(0, parts, n)
        idx[rng.random(n) < 0.99] = mid
    else:
        raise ValueError(shape)
    return idx.astype(np.int32)


def expected_slabs(rows, idx, parts):
    """Slab of every partition: the rows whose index is p, in input order -> list of `parts` [rows_p, row_bytes] arrays."""
    order = np.argsort(idx, kind="stable")
    counts = np.bincount(idx, minlength=parts)
    return np.split(rows[order], np.cumsum(counts)[:-1])


def expected_buffer(layout, slabs):
    """Every destination byte after a correct scatter into a _Slabs of `layout`, buffers in order."""
    g = np.full(GUARD, SENTINEL, dtype=np.uint8)
    if layout == "tensors":
        return np.concatenate([x for s in slabs for x in (g, s.reshape(-1), g)])
    return np.concatenate([g, *[s.reshape(-1) for s in slabs], g])


def _first_difference(got, want):
    bad = np.flatnonzero(got != want)
    return f"{bad.size} bytes differ, first at byte {bad[0]}" if bad.size else "equal"


# ---- device plumbing ----
class _Slabs:
    """Destination slabs of counts[p] rows each, every byte a sentinel.  Layouts:
    tensors    - one tensor per partition, GUARD sentinel bytes before and after its slab;
    contiguous - one tensor, slabs back to back at multiples of the row width (as PeerShuffleSorter lays out a receive
                 buffer), GUARD bytes before the first and after the last;
    peer       - the contiguous layout in a buffer from ytgpu_peer_buffer_create."""

    def __init__(self, ctx, layout, counts, row_bytes):
        import torch
        from ytsaurus_b200.shuffle import _DevicePointerArray
        self.ctx, self.peer_ptr = ctx, None
        counts = [int(c) for c in counts]
        if layout == "tensors":
            self.bufs = [torch.full((2 * GUARD + c * row_bytes,), SENTINEL, dtype=torch.uint8, device="cuda") for c in counts]
            self.ptrs = [b.data_ptr() + GUARD for b in self.bufs]
            return
        nbytes = 2 * GUARD + sum(counts) * row_bytes
        if layout == "peer":
            self.peer_ptr, _ = ctx.peer_buffer_create(nbytes)
            buf = torch.as_tensor(_DevicePointerArray(self.peer_ptr, nbytes), device="cuda")
            buf.fill_(SENTINEL)
        else:
            buf = torch.full((nbytes,), SENTINEL, dtype=torch.uint8, device="cuda")
        self.bufs = [buf]
        starts = np.concatenate([[0], np.cumsum(counts, dtype=np.int64)])
        self.ptrs = [buf.data_ptr() + GUARD + int(s) * row_bytes for s in starts[:-1]]

    def host_bytes(self):
        import torch
        return (torch.cat(self.bufs) if len(self.bufs) > 1 else self.bufs[0]).cpu().numpy()

    def close(self):
        self.bufs = []
        if self.peer_ptr is not None:
            self.ctx.peer_buffer_destroy(self.peer_ptr)
            self.peer_ptr = None


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).reshape(-1)).cuda()


def _random_rows(rng, n, row_bytes):
    return rng.integers(0, 256, (n, row_bytes), dtype=np.uint8)


def scatter_and_check(ctx, rows, idx, parts, layout):
    """Scatter host rows [n, row_bytes] by idx into `layout` and compare every destination byte with the reference."""
    row_bytes = rows.shape[1]
    counts = np.bincount(idx, minlength=parts)
    dest = _Slabs(ctx, layout, counts, row_bytes)
    try:
        ctx.scatter_rows_to_peers(_dev(rows), row_bytes, _dev(idx), counts.tolist(), dest.ptrs)
        got = dest.host_bytes()
    finally:
        dest.close()
    want = expected_buffer(layout, expected_slabs(rows, idx, parts))
    assert got.shape == want.shape and (got == want).all(), (
        f"{len(rows)} rows x {row_bytes} B, {parts} partitions, {layout}: {_first_difference(got, want)}")


def _expect_rejected(ctx, rows, row_bytes, idx, counts, parts, layout="tensors", dest_offsets=None):
    """The call fails with ERR_INVALID_ARGUMENT and writes no destination byte."""
    dest = _Slabs(ctx, layout, counts, row_bytes)
    try:
        ptrs = list(dest.ptrs)
        for p, off in (dest_offsets or {}).items():
            ptrs[p] += off
        with pytest.raises(capi.YtGpuError) as e:
            ctx.scatter_rows_to_peers(rows, row_bytes, idx, [int(c) for c in counts], ptrs)
        assert e.value.code == capi.ERR_INVALID_ARGUMENT, e.value.message
        got = dest.host_bytes()
    finally:
        dest.close()
    assert (got == SENTINEL).all(), f"{parts} partitions: rejected call wrote {_first_difference(got, SENTINEL)}"
    return e.value.message


def _still_usable(ctx, parts, seed):
    """A well-formed call on the same context right after a rejected one."""
    rng = np.random.default_rng(seed)
    rows = _random_rows(rng, 3000, 48)
    scatter_and_check(ctx, rows, make_index("uniform", 3000, parts, rng), parts, "contiguous")


@pytest.fixture(scope="module")
def ctx():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from ytsaurus_b200 import GpuContext
    c = GpuContext(0)
    yield c
    c.close()


# ---- host-only check of the references ----
def test_references_on_host():
    rng = np.random.default_rng(5)
    for parts in (1, 4, 33):
        for n in (0, 1, 100, 1000):
            rows = _random_rows(rng, n, 16)
            idx = make_index("uniform", n, parts, rng)
            slabs = expected_slabs(rows, idx, parts)
            assert len(slabs) == parts
            for p in range(parts):  # per-row definition: rows of partition p, in input order
                want = [rows[i] for i in range(n) if idx[i] == p]
                assert slabs[p].tobytes() == b"".join(r.tobytes() for r in want)
            for layout in LAYOUTS:
                buf = expected_buffer(layout, slabs)
                guards = 2 * GUARD * (parts if layout == "tensors" else 1)
                assert buf.size == n * 16 + guards and (buf == SENTINEL).sum() >= guards
    n, parts = 10_000, 40
    for shape in SHAPES:
        idx = make_index(shape, n, parts, rng)
        assert idx.dtype == np.int32 and idx.min() >= 0 and idx.max() < parts
        counts = np.bincount(idx, minlength=parts)
        if shape.startswith("all_"):
            assert counts.max() == n
        if shape == "empty_ends_and_middle":
            assert counts[0] == counts[parts // 2] == counts[-1] == 0 and (np.delete(counts, [0, parts // 2, parts - 1]) > 0).all()
        if shape == "sorted":
            assert (np.diff(idx) >= 0).all()
        if shape == "skew_99":
            assert counts[parts // 2] > 0.98 * n
    runs = make_index("runs_31_32_33", 96, 4096, np.random.default_rng(0))
    assert len(runs) == 96 and len(set(runs[:31])) == 1 and len(set(runs[31:63])) == 1 and len(set(runs[63:96])) == 1


# ---- every path, width and row count ----
@pytest.mark.gpu
@pytest.mark.parametrize("row_bytes", ROW_WIDTHS)
@pytest.mark.parametrize("parts", STREAM_PARTS + MANY_PARTS)
def test_scatter_rows(ctx, parts, row_bytes):
    rng = np.random.default_rng(parts * 1000 + row_bytes)
    failures = []  # every row count runs: a failure names all the counts that fail, not only the first
    for i, n in enumerate(ROW_COUNTS):
        rows = _random_rows(rng, n, row_bytes)
        idx = make_index("uniform", n, parts, rng)
        layout = LAYOUTS[(i + parts + row_bytes // 16) % len(LAYOUTS)]
        try:
            scatter_and_check(ctx, rows, idx, parts, layout)
        except (AssertionError, capi.YtGpuError) as e:
            failures.append(f"n={n} {layout}: {e}")
    assert not failures, "\n".join(failures)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("parts", [4, 17, 32, 33, 257, 4096])
def test_scatter_index_shapes(ctx, parts, shape):
    rng = np.random.default_rng(parts * 31 + SHAPES.index(shape))
    for n, layout in ((4097, "tensors"), (150_001, "contiguous")):
        idx = make_index(shape, n, parts, rng)
        for row_bytes in (48, 64):
            rows = _random_rows(rng, n, row_bytes)
            scatter_and_check(ctx, rows, idx, parts, layout)


# ---- the many-partition path at few partitions, in a child process ----
def forced_many_partition_cases():
    """Run in a child process with YTGPU_SCATTER_STREAM=0: the checks above at 1, 4 and 32 partitions, on the path that
    sorts the index."""
    from ytsaurus_b200 import GpuContext
    assert os.environ.get("YTGPU_SCATTER_STREAM") == "0"
    ctx = GpuContext(0)
    rng = np.random.default_rng(17)
    ran = 0
    for parts in (1, 4, 32):
        for row_bytes in (16, 48, 64, 256):
            for n in (0, 1, 33, 1025, 150_001):
                for shape in ("uniform", "all_last", "runs_31_32_33"):
                    rows = _random_rows(rng, n, row_bytes)
                    idx = make_index(shape, n, parts, rng)
                    scatter_and_check(ctx, rows, idx, parts, LAYOUTS[ran % len(LAYOUTS)])
                    ran += 1
        rows = _random_rows(rng, 5000, 64)
        idx = make_index("uniform", 5000, parts, rng)
        counts = np.bincount(idx, minlength=parts)
        for bad_value in (parts, -1):
            bad = idx.copy()
            bad[2500] = bad_value
            _expect_rejected(ctx, _dev(rows), 64, _dev(bad), counts, parts)
            ran += 1
        if parts > 1:
            wrong = counts.copy()
            wrong[0] += 1
            wrong[-1] -= 1
            _expect_rejected(ctx, _dev(rows), 64, _dev(idx), wrong, parts)
            ran += 1
        _still_usable(ctx, parts, parts)
    ctx.close()
    print(f"ok: {ran} forced many-partition scatters")


@pytest.mark.gpu
def test_many_partition_path_at_few_partitions():
    env = dict(os.environ, YTGPU_SCATTER_STREAM="0")
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys; sys.path[:0] = [{os.path.dirname(here)!r}, {here!r}]; "
            "import test_peer_scatter as t; t.forced_many_partition_cases()")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "ok:" in r.stdout, f"exit {r.returncode}\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}"


# ---- large inputs, checked on the device ----
def _scatter_large(ctx, n, parts, row_bytes):
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(n + parts)
    rows = torch.randint(0, 256, (n * row_bytes,), dtype=torch.uint8, device="cuda", generator=g)
    idx = torch.randint(0, parts, (n,), dtype=torch.int32, device="cuda", generator=g)
    counts = torch.bincount(idx, minlength=parts).cpu().tolist()
    dest = _Slabs(ctx, "contiguous", counts, row_bytes)
    try:
        ctx.scatter_rows_to_peers(rows, row_bytes, idx, counts, dest.ptrs)
        got = dest.bufs[0]
        rows2d = rows.view(n, row_bytes)
        want = torch.cat([rows2d[idx == p] for p in range(parts)]).view(-1)  # boolean masks keep input order
        assert bool((got[:GUARD] == SENTINEL).all()) and bool((got[-GUARD:] == SENTINEL).all())
        same = got[GUARD:-GUARD] == want
        assert bool(same.all()), f"{int((~same).sum())} bytes differ, first at slab byte {int((~same).nonzero()[0])}"
    finally:
        dest.close()


@pytest.mark.gpu
def test_scatter_bench_exchange_shape(ctx):
    # the row exchange of the 8-GPU sort: 3*10^7 rows of 64 B over 8 partitions
    _scatter_large(ctx, 30_000_000, 8, 64)


@pytest.mark.gpu
def test_scatter_large_many_partitions(ctx):
    # 10^7 rows: the index sort takes the radix sort's hybrid schedule
    _scatter_large(ctx, 10_000_000, 4096, 64)


# ---- fed by the partition step ----
@pytest.mark.gpu
@pytest.mark.parametrize("parts", [8, 1000])
@pytest.mark.parametrize("kind", ["ordered", "hash"])
def test_scatter_matches_partition_slabs(ctx, kind, parts):
    """ytgpu_partition_fixed_rows' index and histogram fed to the scatter, all slabs in one buffer: both promise stable
    partition order, so the scatter must reproduce the partition step's own slab output byte for byte."""
    from ytsaurus_b200.rowset import EValueType as T
    from ytsaurus_b200.shuffle import pivot_bounds_from_rows
    n = 150_001
    rng = np.random.default_rng(parts + len(kind))
    key_columns = [(8, 8, T.Uint64, 0, 1)]
    for row_bytes in (48, 64):
        rows = _random_rows(rng, n, row_bytes)
        rows[: n // 4, 8:16] = rows[n // 2: n // 2 + n // 4, 8:16]  # duplicate keys
        if kind == "ordered":
            keys = rows[:, 8:16].copy().view(np.uint64).reshape(-1)
            pivots = rows[np.argsort(keys, kind="stable")[np.linspace(0, n - 1, parts + 1).astype(np.int64)[1:-1]]]
            bounds, blen, binc = pivot_bounds_from_rows(pivots, key_columns)
            spec = ctx._partition_spec(capi.PARTITION_ORDERED, parts, key_columns=key_columns, bounds=bounds,
                                       bound_prefix_length=blen, bound_inclusive=binc)
        else:
            spec = ctx._partition_spec(capi.PARTITION_HASH, parts, key_columns=key_columns, key_column_count=1, salt=0x5EED)
        src = _dev(rows)
        idx, hist, slabs = ctx.partition_fixed_rows(src, row_bytes, spec, want_index=True, want_slabs=True)
        counts = hist.cpu().numpy().view(np.uint64).tolist()
        assert sum(counts) == n and sum(c > 0 for c in counts) > parts // 2
        dest = _Slabs(ctx, "contiguous", counts, row_bytes)
        try:
            ctx.scatter_rows_to_peers(src, row_bytes, idx, counts, dest.ptrs)
            got = dest.host_bytes()
        finally:
            dest.close()
        want = np.concatenate([np.full(GUARD, SENTINEL, np.uint8), slabs.cpu().numpy(), np.full(GUARD, SENTINEL, np.uint8)])
        assert (got == want).all(), f"{row_bytes} B: {_first_difference(got, want)}"
        ref = expected_buffer("contiguous", expected_slabs(rows, idx.cpu().numpy(), parts))
        assert (got == ref).all()


# ---- rejected calls ----
@pytest.mark.gpu
@pytest.mark.parametrize("case", ["index_past_end", "index_negative", "counts_disagree"])
@pytest.mark.parametrize("parts", [5, 32, 33, 4096])
def test_scatter_rejects_bad_index(ctx, parts, case):
    """Caller-supplied indices and counts are checked before anything is written, on both paths: an index outside
    [0, parts), or counts that sum to n but disagree with the index, would put rows into the wrong slabs."""
    n = 5000
    rng = np.random.default_rng(parts + len(case))
    rows = _random_rows(rng, n, 64)
    idx = make_index("uniform", n, parts, rng)
    counts = np.bincount(idx, minlength=parts)
    if case == "counts_disagree":
        src = int(np.flatnonzero(counts)[0])
        counts[src] -= 1
        counts[(src + 1) % parts] += 1
    else:
        idx[[0, n // 2, n - 1]] = [parts, 2**31 - 1, parts + 7] if case == "index_past_end" else [-1, -2**31, -parts]
    _expect_rejected(ctx, _dev(rows), 64, _dev(idx), counts, parts)
    _still_usable(ctx, parts, parts)


@pytest.mark.gpu
@pytest.mark.parametrize("parts", [0, 4097])
def test_scatter_rejects_partition_count(ctx, parts):
    n = 100
    rows = _random_rows(np.random.default_rng(3), n, 64)
    idx = np.zeros(n, dtype=np.int32)
    counts = [n] + [0] * (parts - 1) if parts else []
    msg = _expect_rejected(ctx, _dev(rows), 64, _dev(idx), counts, parts, layout="contiguous")
    assert "partition_count" in msg
    _still_usable(ctx, 4, parts)


@pytest.mark.gpu
@pytest.mark.parametrize("row_bytes", [0, 8, 24])
def test_scatter_rejects_row_width(ctx, row_bytes):
    import ctypes as C
    n, parts = 64, 4
    rows = _dev(_random_rows(np.random.default_rng(4), n, 32))
    idx = _dev(np.arange(n, dtype=np.int32) % parts)
    counts = [n // parts] * parts
    dest = _Slabs(ctx, "tensors", counts, 32)
    try:
        view = capi.FixedRowsView(rows.data_ptr(), n, row_bytes, capi.MEM_DEVICE)  # the wrapper divides by row_bytes
        err = capi.Error()
        got = ctx.lib.ytgpu_scatter_rows_to_peers(ctx.handle, C.byref(view), idx.data_ptr(), parts,
                                                  (C.c_uint64 * parts)(*counts), (C.c_void_p * parts)(*dest.ptrs), C.byref(err))
        assert got == capi.ERR_INVALID_ARGUMENT and b"row_bytes" in err.message, err.message
        assert (dest.host_bytes() == SENTINEL).all()
    finally:
        dest.close()
    _still_usable(ctx, parts, row_bytes)


@pytest.mark.gpu
@pytest.mark.parametrize("what", ["rows", "destination"])
@pytest.mark.parametrize("parts", [4, 300])
def test_scatter_rejects_misaligned_pointers(ctx, parts, what):
    """Both paths move rows as 16-byte vectors: a rows pointer or slab start that is not 16-byte aligned (a byte slice
    of a tensor, say) is rejected before any launch."""
    n = 4000
    rng = np.random.default_rng(parts)
    rows = _random_rows(rng, n, 64)
    idx = make_index("uniform", n, parts, rng)
    counts = np.bincount(idx, minlength=parts)
    if what == "rows":
        padded = _dev(np.concatenate([np.zeros(8, np.uint8), rows.reshape(-1)]))
        msg = _expect_rejected(ctx, padded[8:], 64, _dev(idx), counts, parts)
    else:
        msg = _expect_rejected(ctx, _dev(rows), 64, _dev(idx), counts, parts, dest_offsets={parts // 2: 8})
    assert "aligned" in msg
    _still_usable(ctx, parts, parts + 1)

