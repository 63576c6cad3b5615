"""Packed hybrid sorts of 2^20 < n <= 2^27 rows whose sorted digits are not skewed run three digit passes instead of
four: the passes order the rows by the top three bytes of the 32-bit prefix only, and the hybrid tail orders each run of
equal 24-bit prefixes by the whole prefix, and by the full key where prefixes tie.  Every shape must give the stable
order, and the schedule that ran is checked through the pass count."""
import numpy as np
import pytest

from ytsaurus_b200.rowset import EValueType as T

pytestmark = pytest.mark.gpu

ROW = 16  # key (8 B) + 8 payload bytes: the payload tells rows with equal keys apart
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
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()


def _rows(rng, keys):
    n = len(keys)
    rows = np.empty((n, ROW), dtype=np.uint8)
    rows[:, :8] = keys.view(np.uint8).reshape(n, 8)
    rows[:, 8:] = np.arange(n, dtype=np.uint64).view(np.uint8).reshape(n, 8)
    return rows


def _check(ctx, rng, keys, passes, want=None, typ=T.Uint64, desc=0):
    rows = _rows(rng, keys)
    if want is None:
        order_keys = keys.view(np.int64) if typ == T.Int64 else keys
        want = np.argsort(~order_keys if desc else order_keys, kind="stable")
    want = want.astype(np.uint32)
    out, perm = ctx.sort_fixed_rows(_dev(rows), ROW, [(0, 8, typ, desc, 1)], want_rows=True, want_perm=True)
    assert ctx.last_sort_passes() == passes
    got = perm.cpu().numpy().view(np.uint32)
    assert np.array_equal(got, want)
    del perm
    assert np.array_equal(out.cpu().numpy().reshape(-1, ROW), rows[want])


def _uniform(rng, n):
    return rng.integers(0, 2**64 - 1, n, dtype=np.uint64, endpoint=True)


def _set_top(keys, members, bits, value):
    """keys[members] get the top `bits` bits of `value`; their other bits stay."""
    low = np.uint64((1 << (64 - bits)) - 1)
    keys[members] = (keys[members] & low) | (np.uint64(value) & ~low)


@pytest.mark.parametrize("n", [2**20, 2**20 + 1, 3_000_000])
def test_uniform_keys(ctx, n):
    # 2^20 rows: three hybrid passes of three scheduled digits; from 2^20 + 1 rows on, three of four
    rng = np.random.default_rng(n)
    _check(ctx, rng, _uniform(rng, n), passes=3)


@pytest.mark.parametrize("n", [2**27 - 1, 2**27 + 1])
def test_uniform_keys_at_the_row_limit(ctx, n):
    """Up to 2^27 rows three passes, above four.  The keys are distinct: an ascending set spread over ~98 % of the key
    space, handed out in a random order, so the stable order is that shuffle (a numpy sort of 2^27 keys is slow)."""
    rng = np.random.default_rng(n)
    steps = rng.integers(1, int(2**64 / n * 1.96), n, dtype=np.uint64)
    ascending = np.cumsum(steps, dtype=np.uint64)
    assert ascending[-1] > ascending[0]  # no wrap-around
    shuffle = rng.permutation(n)
    keys = np.empty(n, dtype=np.uint64)
    keys[shuffle] = ascending
    _check(ctx, rng, keys, passes=3 if n <= 2**27 else 4, want=shuffle)


@pytest.mark.parametrize("shape", ["byte4", "byte3_and_below", "equal", "all_three"])
def test_runs_of_equal_top_bytes(ctx, shape):
    """Groups of 2-31 rows share their top 24 bits and differ only in byte 4 (the byte the tail sorts), share their top
    32 bits and differ only in bytes 3-0 (equal prefixes: the full keys decide), or are the same key (stability)."""
    n = 2_500_000
    rng = np.random.default_rng(len(shape))
    keys = _uniform(rng, n)
    order = rng.permutation(n)
    kinds = ["byte4", "byte3_and_below", "equal"] if shape == "all_three" else [shape]
    pos = 0
    for g in range(60_000):
        m = int(rng.integers(2, 32))
        members = order[pos: pos + m]
        pos += m
        kind = kinds[g % len(kinds)]
        leader = keys[members[0]]
        if kind == "equal":
            keys[members] = leader
        else:
            _set_top(keys, members, 24 if kind == "byte4" else 32, leader)
    _check(ctx, rng, keys, passes=3)


@pytest.mark.parametrize("length", [32, 33])
@pytest.mark.parametrize("content", ["mixed", "equal"])
def test_run_of_32_and_33_rows(ctx, length, content):
    """A run of 32 equal 24-bit prefixes is the longest the tail sorts itself; 33 rows are a long run: equal keys stay as
    they are, mixed keys are sorted on the side.  The runs are placed across tile boundaries as well."""
    n = 2**21 + 17
    rng = np.random.default_rng(length * 2 + (content == "equal"))
    keys = _uniform(rng, n)
    for r in range(40):
        members = np.sort(rng.choice(n, length, replace=False)) if r % 2 else rng.integers(0, n - length) + np.arange(length)
        if content == "equal":
            keys[members] = keys[members[0]]
        else:
            _set_top(keys, members, 24, keys[members[0]])
    _check(ctx, rng, keys, passes=3)


def test_many_mixed_long_runs_take_the_complete_schedule(ctx):
    n = 2**21
    rng = np.random.default_rng(7)
    keys = _uniform(rng, n)
    order = rng.permutation(n)
    runs = MIXED_CAP + 600
    for r in range(runs):
        members = order[r * 34: (r + 1) * 34]
        _set_top(keys, members, 24, keys[members[0]])
    _check(ctx, rng, keys, passes=3 + 8)  # three hybrid passes, then the complete LSD schedule over all 8 digits


@pytest.mark.parametrize("shape", ["one_hot_value", "top_byte"])
def test_skewed_digit_keeps_four_passes(ctx, shape):
    """One value on 12 % of the rows (hashed Zipf keys) skews every digit; 3 % of the rows on one top byte (four times
    its uniform share, > 2 n / 256) skews one.  Either keeps the fourth pass."""
    n = 2**21
    rng = np.random.default_rng(len(shape))
    keys = _uniform(rng, n)
    hot = rng.random(n) < (0.12 if shape == "one_hot_value" else 0.03)
    if shape == "one_hot_value":
        keys[hot] = np.uint64(0x9E3779B97F4A7C15)
    else:
        _set_top(keys, np.flatnonzero(hot), 8, 0xA5 << 56)
    _check(ctx, rng, keys, passes=4)


@pytest.mark.parametrize("constant_digit", [4, 5])
def test_non_adjacent_active_digits(ctx, constant_digit):
    """Digit 4 constant: the prefix is digits 3, 5, 6, 7 and the tail sorts digit 3; digit 5 constant: digits 3, 4, 6, 7."""
    n = 2**21 + 5
    rng = np.random.default_rng(constant_digit)
    keys = _uniform(rng, n)
    shift = np.uint64(8 * constant_digit)
    keys = (keys & ~(np.uint64(0xFF) << shift)) | (np.uint64(0x3C) << shift)
    _check(ctx, rng, keys, passes=3)


@pytest.mark.parametrize("typ,desc", [(T.Uint64, 1), (T.Int64, 0), (T.Int64, 1)])
def test_descending_and_int64_keys(ctx, typ, desc):
    n = 2**21 + 3
    rng = np.random.default_rng(int(typ) * 2 + desc)
    keys = _uniform(rng, n)
    dup = rng.integers(0, n, n // 10)  # a tenth of the rows repeat another row's key
    keys[dup] = keys[rng.integers(0, n, len(dup))]
    _check(ctx, rng, keys, passes=3, typ=typ, desc=desc)


def test_presorted_keys(ctx):
    n = 2**21
    rng = np.random.default_rng(3)
    _check(ctx, rng, np.sort(_uniform(rng, n)), passes=3)
