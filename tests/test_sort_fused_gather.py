"""Fixed-row sorts that take the three-pass packed hybrid schedule (2^20 < n <= 2^27 rows, digits not skewed) move the
rows in the hybrid tail: the block that orders a tile's runs of equal 24-bit prefixes also gathers the rows of the
positions it owns, and writes the permutation only when the caller asks for it.  Rows must come out as
rows[argsort(keys, stable)] byte for byte on every path: rows only and with the permutation, any row width, runs that
cross the tail's 1984-position tiles, mixed long runs re-sorted on the side (their rows gathered again) and the complete
schedule (all rows gathered again)."""
import numpy as np
import pytest

from ytsaurus_b200.rowset import EValueType as T

pytestmark = pytest.mark.gpu

TILE = 1984  # positions per block of the hybrid tail (radix_sort.cu kRunTile)
MIXED_CAP = 16384  # mixed long runs sorted one by one (radix_sort.cu kMixedCap); more take the complete schedule


@pytest.fixture(scope="module")
def ctx():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from ytsaurus_b200 import GpuContext
    c = GpuContext(0)
    yield c
    c.close()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).reshape(-1)).cuda()


def _rows(rng, keys, row_bytes, key_off):
    """Random bytes (rows with equal keys differ) with the key at byte key_off."""
    n = len(keys)
    rows = rng.integers(0, 256, (n, row_bytes), dtype=np.uint8)
    rows[:, key_off:key_off + 8] = keys.view(np.uint8).reshape(n, 8)
    return rows


def _sort(ctx, rows, row_bytes, key_off, want_perm, host=False):
    src = rows.reshape(-1) if host else _dev(rows)
    out, perm = ctx.sort_fixed_rows(src, row_bytes, [(key_off, 8, T.Uint64, 0, 1)], want_rows=True, want_perm=want_perm)
    out = out if host else out.cpu().numpy()
    if perm is not None:
        perm = perm if host else perm.cpu().numpy()
        perm = perm.view(np.uint32)
    return out.reshape(-1, row_bytes), perm


def _check(ctx, rng, keys, passes, want_perm, row_bytes=16, key_off=0, host=False):
    rows = _rows(rng, keys, row_bytes, key_off)
    want = np.argsort(keys, kind="stable").astype(np.uint32)
    out, perm = _sort(ctx, rows, row_bytes, key_off, want_perm, host)
    assert ctx.last_sort_passes() == passes
    assert np.array_equal(out, rows[want])
    if want_perm:
        assert np.array_equal(perm, want)


def _uniform(rng, n):
    return rng.integers(0, 2**64 - 1, n, dtype=np.uint64, endpoint=True)


def _designed(rng, n, runs):
    """Keys whose sorted position p has a 24-bit prefix that grows with p, except inside the listed runs (start, length,
    equal) of sorted positions, which share one prefix; the low 40 bits are random, or one value for an `equal` run.
    The prefixes spread evenly over the 24-bit space, so no sorted digit is skewed.  Returned in a random order."""
    steps = rng.integers(1, max(2, int(2**24 / n * 1.9)), n, dtype=np.uint64)
    steps[0] = 0
    low = rng.integers(0, 2**40, n, dtype=np.uint64)
    for s, length, equal in runs:
        steps[s + 1: s + length] = 0
        if equal:
            low[s: s + length] = low[s]
    prefix = np.cumsum(steps, dtype=np.uint64)
    assert prefix[-1] < 2**24
    keys = np.empty(n, dtype=np.uint64)
    keys[rng.permutation(n)] = (prefix << np.uint64(40)) | low
    return keys


@pytest.mark.parametrize("want_perm", [False, True])
@pytest.mark.parametrize("n", [2**20 + 1, 3_000_001])
def test_uniform_keys(ctx, n, want_perm):
    rng = np.random.default_rng(n + want_perm)
    _check(ctx, rng, _uniform(rng, n), passes=3, want_perm=want_perm)


@pytest.mark.parametrize("want_perm", [False, True])
@pytest.mark.parametrize("row_bytes", [16, 48, 64, 80, 128])
def test_row_widths_with_the_key_inside_the_row(ctx, row_bytes, want_perm):
    n = 2**21 + 1001  # not a multiple of the tile
    assert n % TILE
    rng = np.random.default_rng(row_bytes * 2 + want_perm)
    _check(ctx, rng, _uniform(rng, n), passes=3, want_perm=want_perm, row_bytes=row_bytes, key_off=row_bytes - 8)


@pytest.mark.parametrize("want_perm", [False, True])
def test_runs_across_tile_boundaries_and_at_both_ends(ctx, want_perm):
    """Short runs (2-32 rows) that cross a tile boundary by 1 to length-1 positions, start on one or end just before one;
    short runs at sorted positions 0 and n-1; long runs (33-3000 rows) of equal and of mixed keys across boundaries."""
    n = 2**21 + 77
    rng = np.random.default_rng(11 + want_perm)
    runs = [(0, 7, False), (n - 9, 9, False)]
    k = 3
    for length in [2, 3, 17, 31, 32]:
        for cut in sorted({1, length // 2, length - 1}):  # positions before the boundary
            runs.append((k * TILE - cut, length, False))
            k += 3
        runs.append((k * TILE, length, False))  # starts on a boundary
        runs.append(((k + 3) * TILE - length, length, False))  # ends just before one
        k += 6
    for length in [33, 40, 100, 3000]:
        for equal in (False, True):
            runs.append((k * TILE - 20, length, equal))
            k += 4
    _check(ctx, rng, _designed(rng, n, runs), passes=3, want_perm=want_perm)


@pytest.mark.parametrize("host", [False, True])
def test_mixed_long_runs_rows_only(ctx, host):
    """Long runs of different keys are sorted on the side after the tail gathered them: their rows are gathered again."""
    n = 2**21 + 3
    rng = np.random.default_rng(5 + host)
    starts = rng.choice(np.arange(1, n // 600), 300, replace=False) * 600
    lengths = rng.integers(33, 400, len(starts))
    _check(ctx, rng, _designed(rng, n, [(int(s), int(m), False) for s, m in zip(starts, lengths)]), passes=3, want_perm=False,
           host=host)


@pytest.mark.parametrize("want_perm", [False, True])
def test_many_mixed_long_runs_take_the_complete_schedule(ctx, want_perm):
    n = 2**21
    rng = np.random.default_rng(7)
    keys = _uniform(rng, n)
    order = rng.permutation(n)
    low = np.uint64((1 << 40) - 1)
    for r in range(MIXED_CAP + 600):
        members = order[r * 34: (r + 1) * 34]
        keys[members] = (keys[members] & low) | (keys[members[0]] & ~low)
    _check(ctx, rng, keys, passes=3 + 8, want_perm=want_perm)


@pytest.mark.parametrize("want_perm", [False, True])
def test_host_input_and_output(ctx, want_perm):
    n = 2**20 + 4097
    rng = np.random.default_rng(9 + want_perm)
    _check(ctx, rng, _uniform(rng, n), passes=3, want_perm=want_perm, row_bytes=64, key_off=8, host=True)


def test_launches_of_a_three_pass_sort(ctx):
    """Key extract, plan, three passes, the gathering tail and the long-run classification: no separate gather kernel.
    The permutation adds one launch (it is written by the tail and copied out)."""
    n = 2**21
    rng = np.random.default_rng(13)
    rows = _rows(rng, _uniform(rng, n), 64, 0)
    src = _dev(rows)
    launches = []
    for want_perm in (False, True):
        before = ctx.launch_count()
        ctx.sort_fixed_rows(src, 64, [(0, 8, T.Uint64, 0, 1)], want_rows=True, want_perm=want_perm)
        launches.append(ctx.launch_count() - before)
        assert ctx.last_sort_passes() == 3
    assert launches == [7, 8]
