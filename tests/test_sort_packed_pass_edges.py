"""Edge shapes of the packed digit pass (one (prefix << 32) | row index word per row, 24 items per thread in tiles of
6144 rows): partial last tiles, digits shared by a whole warp, whole tiles of one key, heavy duplicates, descending and
signed keys, and the plain packed schedule on both sides of the 2^18-row packed threshold.  Ranking inside the warp is
item-major and the look-back adds the counts of earlier tiles, so each shape must keep the stable order: every sort is
compared bit for bit with numpy's stable argsort."""
import numpy as np
import pytest

from ytsaurus_b200.rowset import EValueType as T

pytestmark = pytest.mark.gpu

ROW = 16  # key (8 B) + the row number: rows with equal keys stay distinguishable
TILE = 256 * 24  # rows per packed pass tile (kSortThreads x items per thread)


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
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()


def _check(ctx, keys, typ=T.Uint64, desc=0):
    n = len(keys)
    rows = np.empty((n, ROW), dtype=np.uint8)
    rows[:, :8] = keys.view(np.uint8).reshape(n, 8)
    rows[:, 8:] = np.arange(n, dtype=np.uint64).view(np.uint8).reshape(n, 8)
    order_keys = keys.view(np.int64) if typ == T.Int64 else keys
    want = np.argsort(~order_keys if desc else order_keys, kind="stable").astype(np.uint32)
    out, perm = ctx.sort_fixed_rows(_dev(rows), ROW, [(0, 8, typ, desc, 1)], want_rows=True, want_perm=True)
    assert np.array_equal(perm.cpu().numpy().view(np.uint32), want)
    del perm
    assert np.array_equal(out.cpu().numpy().reshape(-1, ROW), rows[want])
    return ctx.last_sort_passes()


def _uniform(rng, n):
    return rng.integers(0, 2**64 - 1, n, dtype=np.uint64, endpoint=True)


@pytest.mark.parametrize("n", [50 * TILE - 1, 50 * TILE + 1, 171 * TILE - 1, 171 * TILE + 1])
def test_partial_last_tile(ctx, n):
    # 50 tiles: packed, below the three-pass range; 171 tiles: above 2^20 rows, the three-pass hybrid schedule
    rng = np.random.default_rng(n)
    _check(ctx, _uniform(rng, n))


@pytest.mark.parametrize("n", [60 * TILE - 1, 60 * TILE + 1, 200 * TILE])
def test_tiles_of_one_digit(ctx, n):
    """Every other tile holds one key (every item of the tile has one digit in every pass); the others are random.
    Tiles are counted from the start, so the partial last tile is one key too when its index is even."""
    rng = np.random.default_rng(n + 1)
    keys = _uniform(rng, n)
    tile = np.arange(n) // TILE
    one = tile % 2 == 0
    keys[one] = _uniform(rng, tile[-1] + 1)[tile[one]]
    _check(ctx, keys)


@pytest.mark.parametrize("run", [32, 32 * 24])
@pytest.mark.parametrize("n", [80 * TILE + 7, 180 * TILE + 5])
def test_warp_uniform_digits(ctx, run, n):
    """Keys constant over aligned runs of 32 rows (one item across a warp) or of 768 rows (a warp's slice of a tile):
    the digit is uniform across the warp for an item but not across the tile."""
    rng = np.random.default_rng(run * 7 + n)
    keys = _uniform(rng, n // run + 1)[np.arange(n) // run]
    _check(ctx, keys)


@pytest.mark.parametrize("n", [300_001, 2_000_003])
def test_heavy_duplicates(ctx, n):
    rng = np.random.default_rng(n)
    pool = _uniform(rng, 5)
    keys = pool[rng.choice(5, n, p=[0.6, 0.25, 0.1, 0.04, 0.01])]
    _check(ctx, keys)


@pytest.mark.parametrize("n", [400_003, 1_500_001])
def test_descending(ctx, n):
    rng = np.random.default_rng(n)
    keys = _uniform(rng, n)
    keys[rng.integers(0, n, n // 4)] = keys[0]  # ties must keep their input order under DESC too
    _check(ctx, keys, desc=1)


@pytest.mark.parametrize("n", [400_003, 1_500_001])
def test_int64(ctx, n):
    rng = np.random.default_rng(n)
    keys = rng.integers(-2**40, 2**40, n, dtype=np.int64).view(np.uint64)
    _check(ctx, keys, typ=T.Int64)


@pytest.mark.parametrize("n", [2**18 - 1, 2**18, 50 * TILE + 1])
def test_plain_packed_schedule(ctx, n):
    """Four active digits: the plain schedule, one pass per digit, packed from 2^18 rows on and pair format below."""
    rng = np.random.default_rng(n)
    keys = rng.integers(0, 2**32, n, dtype=np.uint64) << np.uint64(16)
    assert _check(ctx, keys) == 4
