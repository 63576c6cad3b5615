"""Rowset sort, merge and join by keys whose fixed-width normalised form exceeds 256 bytes: the refinement rounds over
the width-free key words (csrc/long_keys.cu) against the oracle comparator, bit for bit, in the HOST and DEVICE memory
flavours.  `last_sort_refine_rounds` tells which path ran: >= 1 for the refinement sort, 0 for normalised keys."""
import numpy as np
import pytest

import oracle
from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import EValueType as T, Sentinel, U64, VALUE_DTYPE, make_rowset

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from ytsaurus_b200 import GpuContext
    c = GpuContext(0)
    yield c
    c.close()


def _dev(rs):
    import torch
    return (torch.from_numpy(rs.values.view(np.uint8).reshape(rs.row_count, -1).copy()).cuda(),
            torch.from_numpy(rs.heap.copy()).cuda())


def check_sort(ctx, rows, cols, ncols=None, long_path=True):
    """Sorts in both flavours, with and without values, and compares with the oracle's stable sort."""
    rs = make_rowset(rows, ncols=ncols or len(cols))
    k = len(cols)
    assert [c["index"] for c in cols] == list(range(k))
    want, _ = oracle.sort_rows(rs.values, rs.heap, k, [c.get("descending", 0) for c in cols], oracle.SORT_STABLE)
    want_vals = rs.values[want.astype(np.int64)]
    dv, dh = _dev(rs)
    for device in (False, True):
        for want_values in (False, True):
            v, h = (dv, dh) if device else (rs.values, rs.heap)
            out = ctx.sort_rowset(v, h, cols, want_values=want_values)
            perm, outv = out if want_values else (out, None)
            if device:
                perm = perm.cpu().numpy().view(np.uint32)
                if want_values:
                    outv = outv.cpu().numpy().reshape(-1).view(VALUE_DTYPE).reshape(rs.values.shape)
            assert (perm == want).all(), (device, want_values)
            if want_values:
                assert outv.tobytes() == want_vals.tobytes()
            rounds = ctx.get_option("last_sort_refine_rounds")
            assert (rounds >= 1) if long_path else (rounds == 0)
    return rounds


def _rand_bytes(rng, n, alphabet=None):
    if alphabet is None:
        return rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    return bytes(rng.choice(np.frombuffer(alphabet, dtype=np.uint8), n))


def long_strings(rng, n):
    """Lengths 0..2000, shared 300- and 1000-byte prefixes, embedded zeros, exact duplicates."""
    p300, p1000 = _rand_bytes(rng, 300), _rand_bytes(rng, 1000)
    out = []
    for i in range(n):
        kind = int(rng.integers(0, 5))
        if kind == 0:
            s = _rand_bytes(rng, int(rng.integers(0, 2001)))
        elif kind == 1:
            s = p300 + _rand_bytes(rng, int(rng.integers(0, 40)), b"ab\x00")
        elif kind == 2:
            s = p1000 + _rand_bytes(rng, int(rng.integers(0, 40)), b"ab\x00")
        elif kind == 3 and out:
            s = out[int(rng.integers(0, len(out)))]
        else:
            s = p1000[: int(rng.integers(250, 1000))]
        out.append(s)
    out.append(b"x" * 300)  # the key does not fit the fixed-width form whatever was drawn
    return out


@pytest.mark.parametrize("desc", [0, 1])
def test_one_long_string_column(ctx, desc):
    rng = np.random.default_rng(1 + desc)
    rows = [[s, i] for i, s in enumerate(long_strings(rng, 3000))]
    check_sort(ctx, rows, [dict(index=0, type=T.String, descending=desc)], ncols=2)
    check_sort(ctx, rows, [dict(index=0, type=T.String, descending=desc, required=1)], ncols=2)


@pytest.mark.parametrize("desc", [0, 1])
def test_staircase(ctx, desc):
    """"a", "aa", "aaa", ...: every split loses one row, the worst case for the rounds."""
    rng = np.random.default_rng(3)
    ks = rng.permutation(2000)
    rows = [[b"a" * int(k), int(k)] for k in ks]
    check_sort(ctx, rows, [dict(index=0, type=T.String, descending=desc)], ncols=2)


def test_long_string_then_int64(ctx):
    rng = np.random.default_rng(4)
    ss = long_strings(rng, 2000)
    rows = [[s, int(rng.integers(-3, 3))] for s in ss]
    check_sort(ctx, rows, [dict(index=0, type=T.String), dict(index=1, type=T.Int64)])


def test_int64_desc_then_long_string(ctx):
    rng = np.random.default_rng(5)
    ss = long_strings(rng, 2000)
    rows = [[int(rng.integers(-2, 2)), s] for s in ss]
    check_sort(ctx, rows, [dict(index=0, type=T.Int64, descending=1, required=1), dict(index=1, type=T.String)])


@pytest.mark.parametrize("desc", [0, 1])
def test_any_scalar_column_with_long_strings(ctx, desc):
    rng = np.random.default_rng(6 + desc)
    scalars = [None, 0, -1, 1, U64(0), U64(2**64 - 1), float("nan"), -0.0, 0.0, float("-inf"), 1.5, True, False,
               Sentinel(T.Min), Sentinel(T.Max), b"", b"\x00", b"ab"]
    ss = long_strings(rng, 1000)
    rows = [[scalars[int(rng.integers(0, len(scalars)))] if rng.random() < 0.5 else ss[i], i] for i in range(len(ss))]
    rows.append([b"y" * 700, -1])
    check_sort(ctx, rows, [dict(index=0, type=0, descending=desc)], ncols=2)


def test_many_rows(ctx):
    """>= 2^18 rows: the radix sort inside the rounds takes its packed and hybrid paths."""
    rng = np.random.default_rng(7)
    n = (1 << 18) + 1000
    hosts = [b"https://host%03d.example.org/" % i + _rand_bytes(rng, int(rng.integers(0, 12)), b"abc") for i in range(256)]
    tails = rng.integers(0, 400, n)
    rows = []
    for i in range(n):
        if i and rng.random() < 0.1:
            rows.append([rows[int(rng.integers(0, i))][0], i])
        else:
            rows.append([hosts[int(rng.integers(0, 256))] + _rand_bytes(rng, int(tails[i]), b"abcdefghijklmnop"), i])
    rows.append([b"z" * 300, n])
    check_sort(ctx, rows, [dict(index=0, type=T.String)], ncols=2)


def test_all_rows_equal(ctx):
    rows = [[b"q" * 1000, i] for i in range(5000)]
    assert check_sort(ctx, rows, [dict(index=0, type=T.String)], ncols=2) == 1


def test_short_keys_keep_the_normalised_path(ctx):
    rng = np.random.default_rng(8)
    rows = [[_rand_bytes(rng, int(rng.integers(0, 200))), i] for i in range(3000)]
    check_sort(ctx, rows, [dict(index=0, type=T.String)], ncols=2, long_path=False)


def test_declared_width_shorter_than_a_string(ctx):
    rows = [[b"a" * 100], [b"b" * 400], [b"c" * 20]]
    rs = make_rowset(rows)
    with pytest.raises(capi.YtGpuError) as e:
        ctx.sort_rowset(rs.values, rs.heap, [dict(index=0, type=T.String, width=300)])
    assert e.value.code == capi.ERR_SCHEMA_VIOLATION and "longer than the declared" in e.value.message
    # a declared width that holds every string sorts
    perm = ctx.sort_rowset(rs.values, rs.heap, [dict(index=0, type=T.String, width=400)])
    assert perm.tolist() == [0, 1, 2] and ctx.get_option("last_sort_refine_rounds") >= 1


def test_any_value_is_still_rejected(ctx):
    rs = make_rowset([[b"x" * 300], [b"y"]])
    rs.values["type"][1, 0] = T.Any
    with pytest.raises(capi.YtGpuError) as e:
        ctx.sort_rowset(rs.values, rs.heap, [dict(index=0, type=0)])
    assert e.value.code == capi.ERR_UNSUPPORTED


def _sorted_runs(rng, run_count, per_run):
    runs = []
    for r in range(run_count):
        ss = long_strings(rng, int(rng.integers(0, per_run)))
        runs.append(sorted(ss))
    return runs


@pytest.mark.parametrize("device", [False, True])
def test_merge_sorted_runs(ctx, device):
    rng = np.random.default_rng(9)
    runs = _sorted_runs(rng, 5, 800)
    flat = [[s, r] for r, run in enumerate(runs) for s in run]
    rs = make_rowset(flat)
    off = np.cumsum([0] + [len(r) for r in runs])
    want = oracle.merge_sorted(rs.values, rs.heap, 1, None, off)
    v, h = _dev(rs) if device else (rs.values, rs.heap)
    got = ctx.merge_sorted_runs(v, h, [dict(index=0, type=T.String)], off)
    if device:
        got = got.cpu().numpy().view(np.uint32)
    assert (got == want).all()
    assert ctx.get_option("last_merge_used_merge_path") == 0
    assert ctx.get_option("last_sort_refine_rounds") >= 1


@pytest.mark.parametrize("device", [False, True])
def test_join_sorted_runs(ctx, device):
    rng = np.random.default_rng(10)
    base = long_strings(rng, 300)
    streams = [sorted(base[i] for i in rng.integers(0, len(base), int(rng.integers(100, 600)))) for _ in range(4)]
    flat = [[s, i, t] for t, st in enumerate(streams) for i, s in enumerate(st)]
    rs = make_rowset(flat)
    off = np.cumsum([0] + [len(s) for s in streams])
    tags = list(range(len(streams)))
    want = oracle.join_sorted(rs.values, rs.heap, 1, None, off, tags)
    v, h = _dev(rs) if device else (rs.values, rs.heap)
    got = ctx.join_sorted_runs(v, h, [dict(index=0, type=T.String), dict(index=2, type=T.Int64, required=1)], 1, off)
    if device:
        got = got.cpu().numpy().view(np.uint32)
    assert got.tolist() == want.tolist()
    assert ctx.get_option("last_sort_refine_rounds") >= 1
