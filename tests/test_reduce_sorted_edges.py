"""Segmented SUM / COUNT over sorted rows (ytgpu_reduce_sorted_fixed_rows) at the edges of its layout.

The kernel reads one 8-byte key and one 8-byte value per row, gives each thread 8 rows and each tile 2048, and finds
the number of groups before a tile by decoupled look-back over the tiles.  These tests vary what that arithmetic
depends on: the row width and where the key and value sit in the row, groups that start on thread and tile boundaries,
tiles without a group head, thousands of tiles, keys next to the kernel's default of 0, wrapping integer sums, double
zeros, infinities and NaNs, and the output capacity.

The reference is plain numpy over the runs of equal neighbouring keys (the header promises that only neighbour
equality is used, so it never sorts): integer sums wrap mod 2^64 like the kernel's, double sums are math.fsum.  Keys,
counts and integer sums must match bit for bit.  Integer-valued doubles whose sums stay below 2^53 are exact in any
order and must match bit for bit; other doubles must be within (count - 1) * 2^-53 * sum|x| of the exact sum, a bound
that holds for any summation order (the kernel's atomics make the order arbitrary)."""
import ctypes as C
import math

import numpy as np
import pytest

from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import EValueType as T

TILE = 2048  # 256 threads x 8 rows
U = 2.0 ** -53
TYPES = (capi.TYPE_INT64, capi.TYPE_UINT64, capi.TYPE_DOUBLE)


# ---------------------------------------------------------------- reference

def reference(keys, vals, value_type):
    """-> (keys, counts, sums) of the runs of equal neighbouring keys, in row order.  keys, vals: uint64 words.
    Integer sums are uint64 words (wrapping mod 2^64); double sums are math.fsum of each run, as Python floats."""
    n = len(keys)
    heads = np.r_[True, keys[1:] != keys[:-1]] if n else np.zeros(0, bool)
    starts = np.flatnonzero(heads)
    counts = np.diff(np.r_[starts, n]).astype(np.uint64)
    if value_type == capi.TYPE_DOUBLE:
        x = vals.view(np.float64)
        sums = [math.fsum(x[s:s + c]) for s, c in zip(starts.tolist(), counts.tolist())]
    else:
        sums = np.add.reduceat(vals.astype(np.uint64), starts) if n else np.zeros(0, np.uint64)
    return keys[starts], counts, sums


def double_sum_error(got, xs):
    """got - sum(xs), computed exactly and rounded once."""
    return math.fsum([got] + (-np.asarray(xs, dtype=np.float64)).tolist())


def double_sum_ok(got, xs):
    """|got - sum(xs)| <= (len(xs) - 1) * 2^-53 * sum|xs|: the error bound of any order of recursive summation."""
    xs = np.asarray(xs, dtype=np.float64)
    return abs(double_sum_error(got, xs)) <= max(len(xs) - 1, 0) * U * math.fsum(np.abs(xs).tolist())


def test_reference_runs_of_equal_neighbours():
    keys = np.array([5, 5, 0, 0, 0, 5, 2**64 - 1, 2**64 - 1, 2**63, 0], dtype=np.uint64)
    vals = np.array([2**63, 2**63, 1, 2, 3, 7, 2**64 - 1, 2, 0, 9], dtype=np.uint64)
    k, c, s = reference(keys, vals, capi.TYPE_UINT64)
    # the two runs of 5 and the two runs of 0 stay separate groups: the input is not sorted
    assert k.tolist() == [5, 0, 5, 2**64 - 1, 2**63, 0]
    assert c.tolist() == [2, 3, 1, 2, 1, 1]
    assert s.tolist() == [0, 6, 7, 1, 0, 9]  # 2^63 + 2^63 and (2^64 - 1) + 2 wrap
    k, c, s = reference(np.array([7], np.uint64), np.array([3], np.uint64), capi.TYPE_INT64)
    assert (k.tolist(), c.tolist(), s.tolist()) == ([7], [1], [3])


def test_reference_double_sums_and_bound():
    keys = np.array([1, 1, 1, 2, 2, 3], dtype=np.uint64)
    x = np.array([1e16, 1.0, -1e16, -0.0, -0.0, 0.1], dtype=np.float64)
    _, c, s = reference(keys, x.view(np.uint64), capi.TYPE_DOUBLE)
    assert c.tolist() == [3, 2, 1] and s[0] == 1.0 and s[2] == 0.1
    # sequential (1 + 2^-53) + 2^-53 rounds to 1.0, 2^-52 from the exact sum: inside the bound of 2 * 2^-53 * sum|x|
    xs = [1.0, U, U]
    assert double_sum_ok(1.0, xs) and double_sum_ok(1.0 + 2 * U, xs)
    assert not double_sum_ok(1.0 + 8 * U, xs)
    # one value: the sum must be the value itself
    assert double_sum_ok(0.1, [0.1]) and not double_sum_ok(math.nextafter(0.1, 1), [0.1])


# ---------------------------------------------------------------- GPU helpers

@pytest.fixture(scope="module")
def ctx():
    from ytsaurus_b200 import GpuContext
    c = GpuContext(0)
    yield c
    c.close()


def _rows(rng, keys, vals, row_bytes, key_off, val_off):
    """Device rows of `row_bytes` with random filler, the value word at val_off and the key word at key_off (written
    last: when the offsets are equal the value is the key).  -> (rows tensor, the value words as stored)."""
    import torch
    words = rng.integers(-2**63, 2**63 - 1, (len(keys), row_bytes // 8), dtype=np.int64, endpoint=True)
    words[:, val_off // 8] = vals.view(np.int64)
    words[:, key_off // 8] = keys.view(np.int64)
    return torch.from_numpy(words).cuda().view(torch.uint8).reshape(-1), words[:, val_off // 8].view(np.uint64).copy()


def _raw(ctx, rows_ptr, n, row_bytes, key_off, val_off, vtype, outs, capacity):
    """The C call itself, which reports the group count also when it fails: -> (return code, *out_group_count)."""
    view = capi.FixedRowsView(rows_ptr, n, row_bytes, capi.MEM_DEVICE)
    got = C.c_uint64(0)
    err = capi.Error()
    code = ctx.lib.ytgpu_reduce_sorted_fixed_rows(ctx.handle, C.byref(view), key_off, val_off, vtype, *outs, capacity,
                                                  C.byref(got), C.byref(err))
    return code, int(got.value)


def _run(ctx, rows, row_bytes, key_off, val_off, vtype, capacity):
    import torch
    ok, os_, oc = (torch.full((capacity,), -1, dtype=torch.int64, device="cuda") for _ in range(3))
    g = ctx.reduce_sorted_fixed_rows(rows, row_bytes, key_off, val_off, vtype, ok, os_, oc)
    return g, (ok[:g].cpu().numpy().view(np.uint64), oc[:g].cpu().numpy().view(np.uint64), os_[:g].cpu().numpy().view(np.uint64))


def _check(ctx, rng, keys, vals, vtype, row_bytes=16, key_off=0, val_off=8, capacity=None, exact_double=False, info=""):
    """Runs the kernel over keys / vals laid out as described and compares with the reference.  capacity defaults to
    the exact number of groups."""
    rows, stored = _rows(rng, keys, vals, row_bytes, key_off, val_off)
    wk, wc, ws = reference(keys, stored, vtype)
    g, (gk, gc, gs) = _run(ctx, rows, row_bytes, key_off, val_off, vtype, len(wk) if capacity is None else capacity)
    assert g == len(wk), info
    assert np.array_equal(gk, wk), info
    assert np.array_equal(gc, wc), info
    if vtype != capi.TYPE_DOUBLE:
        assert np.array_equal(gs, ws), info
        return
    got = gs.view(np.float64)
    x = stored.view(np.float64)
    if exact_double:
        starts = np.r_[0, np.cumsum(wc)[:-1]].astype(np.int64)
        want = np.add.reduceat(x.astype(np.int64), starts).astype(np.float64)
        assert np.abs(x).sum() < 2.0 ** 53, "exact comparison needs integer sums below 2^53"
        assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), info
        return
    bad = [i for i, (s, c) in enumerate(zip(np.r_[0, np.cumsum(wc)[:-1]].astype(np.int64).tolist(), wc.tolist()))
           if not double_sum_ok(float(got[i]), x[s:s + c])]
    assert not bad, (info, bad[:5], [(float(got[i]), ws[i]) for i in bad[:5]])


def _values(rng, n, vtype, exact_double=False):
    """uint64 words: full-range integers (sums wrap past 2^63 and 2^64), or doubles."""
    if vtype == capi.TYPE_INT64:
        return rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64, endpoint=True).view(np.uint64)
    if vtype == capi.TYPE_UINT64:
        return rng.integers(0, 2**64 - 1, n, dtype=np.uint64, endpoint=True)
    if exact_double:
        return rng.integers(-1000, 1000, n).astype(np.float64).view(np.uint64)
    return (rng.standard_normal(n) * 10.0 ** rng.integers(-3, 6, n)).view(np.uint64)


def _keys_from_heads(heads, base=0):
    """Non-decreasing uint64 keys whose group heads are exactly `heads` (heads[0] must be set)."""
    assert heads[0]
    return (np.cumsum(heads, dtype=np.uint64) - np.uint64(1)) * np.uint64(3) + np.uint64(base)


# ---------------------------------------------------------------- GPU cases

def _layouts(row_bytes):
    w = row_bytes // 8
    cand = [(0, w - 1), (w - 1, 0), (0, min(1, w - 1)), (w - 1, max(w - 2, 0)), (w // 2, w // 2), (w - 1, w - 1)]
    return sorted({(8 * k, 8 * v) for k, v in cand})


@pytest.mark.gpu
@pytest.mark.parametrize("row_bytes", [8, 16, 24, 40, 64, 72, 128, 256])
def test_row_layouts(ctx, row_bytes):
    """Key first / last word, value before / after the key, and key and value in one word (then SUM is the sum of
    the keys), over three tiles and a partial one with random group lengths."""
    rng = np.random.default_rng(row_bytes)
    n = 3 * TILE + 5
    heads = rng.random(n) < 0.05
    heads[0] = True
    for key_off, val_off in _layouts(row_bytes):
        for vtype in TYPES:
            if key_off == val_off and vtype == capi.TYPE_DOUBLE:
                # the key is the value: integer-valued doubles, increasing, so the bit patterns are sorted too
                keys = (np.cumsum(heads).astype(np.float64) * 4.0).view(np.uint64)
                _check(ctx, rng, keys, keys, vtype, row_bytes, key_off, val_off, exact_double=True,
                       info=(row_bytes, key_off, val_off, vtype))
                continue
            keys = _keys_from_heads(heads, base=int(rng.integers(0, 2**62)))
            _check(ctx, rng, keys, _values(rng, n, vtype), vtype, row_bytes, key_off, val_off, info=(row_bytes, key_off, val_off, vtype))


def _heads(kind, n, rng):
    r = np.arange(n)
    if kind == "tile_edges":       # a group opens on row 0 and on the last row of every tile
        h = (r % TILE == 0) | (r % TILE == TILE - 1)
    elif kind == "thread_edges":   # a group opens on every thread's first row
        h = r % 8 == 0
    elif kind == "every_row":      # groups == n
        h = np.ones(n, bool)
    else:                          # random short groups
        h = rng.random(n) < 0.3
    h[0] = True
    return h


_EDGE_N = [1, 7, 8, 9, 2047, 2048, 2049, 4095, 4096, 4097, 3000 * TILE - 1, 3000 * TILE + 1]


@pytest.mark.gpu
@pytest.mark.parametrize("n", _EDGE_N)
@pytest.mark.parametrize("kind", ["tile_edges", "thread_edges", "every_row", "random"])
def test_tile_and_thread_edges(ctx, n, kind):
    """Row counts around a thread (8), a tile (2048) and thousands of tiles, with groups opening on tile and thread
    boundaries or on every row; the output capacity is exactly the number of groups."""
    rng = np.random.default_rng(n * 7 + len(kind))
    heads = _heads(kind, n, rng)
    keys = _keys_from_heads(heads)
    for vtype in TYPES:
        exact = vtype == capi.TYPE_DOUBLE and n > 10_000  # fsum per group is too slow for millions of groups
        _check(ctx, rng, keys, _values(rng, n, vtype, exact), vtype, exact_double=exact, info=(n, kind, vtype))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["one_group", "group_per_tile", "long_and_single"])
def test_look_back_depth(ctx, kind):
    """2 * 10^7 rows (9766 tiles): one group over every row, so every tile after the first has no head and flushes
    into the group an earlier tile opened; one group per tile; and groups crossing hundreds of tiles between groups
    of one row."""
    rng = np.random.default_rng(len(kind))
    n = 20_000_000 + 3
    heads = np.zeros(n, bool)
    if kind == "one_group":
        heads[0] = True
    elif kind == "group_per_tile":
        heads[::TILE] = True
    else:
        at = 0
        while at < n:
            heads[at] = True
            if rng.random() < 0.5:
                at += int(rng.integers(100 * TILE, 400 * TILE))
            else:
                at += 1
    keys = _keys_from_heads(heads, base=2**63 - 5)
    _check(ctx, rng, keys, _values(rng, n, capi.TYPE_INT64), capi.TYPE_INT64, info=kind)
    _check(ctx, rng, keys, _values(rng, n, capi.TYPE_DOUBLE, exact_double=True), capi.TYPE_DOUBLE, exact_double=True, info=kind)


_EDGE_KEYS = np.array([0, 1, 2, 2**63, 2**63 + 1, 1 << 62, (1 << 62) | 1, 2**64 - 1, 2**64 - 2, 2**63 - 1, 5], dtype=np.uint64)


@pytest.mark.gpu
def test_key_values(ctx):
    """Key 0 first and around thread boundaries (the kernel's `prev` defaults to 0), key 2^64 - 1, and neighbours that
    differ only in the top or the bottom bit.  The input is not sorted: only neighbour equality may count."""
    rng = np.random.default_rng(5)
    # hand-written: rows 0..7 hold 5, rows 8.. hold 0: row 8 opens a group although 0 is the kernel's default `prev`
    keys = np.array([5] * 8 + [0] * 9 + [2**63] * 7 + [0] + [1] * 8 + [2**64 - 1] * 8 + [2**64 - 2], dtype=np.uint64)
    for vtype in TYPES:
        _check(ctx, rng, keys, _values(rng, len(keys), vtype), vtype, info=("hand", vtype))
    # runs of 1..20 rows of edge keys, consecutive runs possibly equal (then they merge into one group)
    lens = rng.integers(1, 21, 20_000)
    keys = np.repeat(_EDGE_KEYS[rng.integers(0, len(_EDGE_KEYS), len(lens))], lens)
    keys[:3] = 0  # key 0 first
    for vtype in TYPES:
        _check(ctx, rng, keys, _values(rng, len(keys), vtype), vtype, info=("runs", vtype))


@pytest.mark.gpu
def test_integer_sums_wrap(ctx):
    """INT64 / UINT64 groups whose sums pass 2^63 and 2^64, including groups that span a tile boundary."""
    rng = np.random.default_rng(6)
    n = 2 * TILE + 100
    heads = np.zeros(n, bool)
    heads[[0, 10, TILE - 3, TILE + 50, 2 * TILE + 1]] = True
    keys = _keys_from_heads(heads)
    for vtype, big in ((capi.TYPE_INT64, np.int64(2**62 + 12345).view(np.uint64)), (capi.TYPE_UINT64, np.uint64(2**63 + 99))):
        vals = np.full(n, big, dtype=np.uint64)
        vals[rng.integers(0, n, 50)] = np.uint64(2**64 - 1)
        _check(ctx, rng, keys, vals, vtype, info=vtype)


_NZ, _PINF, _NINF = np.uint64(0x8000000000000000), np.uint64(0x7ff0000000000000), np.uint64(0xfff0000000000000)
_QNAN, _NAN_PAYLOAD, _NEG_NAN = np.uint64(0x7ff8000000000000), np.uint64(0x7ff8000000000abc), np.uint64(0xfff8000000000000)


@pytest.mark.gpu
def test_double_special_groups(ctx):
    """Groups of only -0.0, of +inf, of -inf, of both infinities and with NaNs.

    The bits of the -0.0, +inf and -inf groups are pinned (sums start from +0.0, so only -0.0 gives +0.0) and equal
    those of ytgpu_scan_filter_groupby over the same rows.  NaN results are deliberately not pinned to one bit pattern:
    when a group holds NaNs with different bits, which one an addition passes on depends on the order of the operands,
    and the atomics leave that order open; the header promises only "a NaN".  A group whose NaNs all have one bit
    pattern (the canonical NaN), or that makes its NaN from +inf + -inf, must still give the same bits as
    ytgpu_scan_filter_groupby."""
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(7)
    groups = [
        ("-0.0 x1", [_NZ]), ("-0.0 x9", [_NZ] * 9), ("-0.0 over a tile edge", [_NZ] * (TILE + 17)),
        ("+inf", [_PINF] * 3), ("-inf", [_NINF] * 12), ("+inf and 1.0", [_PINF, np.float64(1.0).view(np.uint64)]),
        ("+inf and -inf", [_PINF] * 5 + [_NINF] * 5), ("canonical NaN", [_QNAN] * 4),
        ("NaN payloads", [_NAN_PAYLOAD, np.float64(2.0).view(np.uint64), _NEG_NAN]),
        ("-0.0 then +0.0", [_NZ, np.uint64(0)]), ("+0.0 then -0.0", [np.uint64(0), _NZ]),
    ]
    # a random filler group between special ones, so the special groups start at varied thread offsets
    parts, names = [], []
    for name, vals in groups:
        parts.append(np.array(vals, dtype=np.uint64))
        names.append(name)
        parts.append(rng.integers(-100, 100, int(rng.integers(1, 30))).astype(np.float64).view(np.uint64))
        names.append(None)
    vals = np.concatenate(parts)
    keys = np.repeat(np.arange(len(parts), dtype=np.uint64) * np.uint64(11), [len(p) for p in parts])
    rows, stored = _rows(rng, keys, vals, 24, 16, 0)
    g, (gk, gc, gs) = _run(ctx, rows, 24, 16, 0, capi.TYPE_DOUBLE, len(parts))
    assert g == len(parts) and gc.tolist() == [len(p) for p in parts]
    by = ctx.scan_filter_groupby(Column(T.Uint64, values=keys), Column(T.Double, values=vals), None, group_count_hint=len(parts))
    order = np.argsort(np.asarray(by["keys"]).view(np.uint64))
    hb_sum = np.asarray(by["sum"]).view(np.uint64)[order]
    assert np.array_equal(np.asarray(by["keys"]).view(np.uint64)[order], gk)
    want_bits = {"-0.0 x1": 0, "-0.0 x9": 0, "-0.0 over a tile edge": 0, "+inf": _PINF, "-inf": _NINF,
                 "+inf and 1.0": _PINF, "-0.0 then +0.0": 0, "+0.0 then -0.0": 0}
    for i, name in enumerate(names):
        got = gs[i]
        if name is None:
            assert got == np.float64(math.fsum(parts[i].view(np.float64))).view(np.uint64)
        elif name in want_bits:
            assert int(got) == int(want_bits[name]), (name, hex(int(got)))
            assert got == hb_sum[i], (name, hex(int(got)), hex(int(hb_sum[i])))
        else:
            assert np.isnan(gs[i:i + 1].view(np.float64)[0]), (name, hex(int(got)))
            if name != "NaN payloads":  # which NaN survives several depends on the order of the additions
                assert got == hb_sum[i], (name, hex(int(got)), hex(int(hb_sum[i])))


@pytest.mark.gpu
@pytest.mark.parametrize("groups", [1000, 1_000_000])
@pytest.mark.parametrize("vtype", [capi.TYPE_INT64, capi.TYPE_UINT64])
def test_same_as_scan_filter_groupby(ctx, groups, vtype):
    """The header's promise: the same keys, sums and counts as ytgpu_scan_filter_groupby over the same sorted rows."""
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(groups + vtype)
    pool = np.unique(rng.integers(0, 2**64 - 1, groups + groups // 10 + 10, dtype=np.uint64, endpoint=True))
    ukeys = np.sort(rng.choice(pool, groups, replace=False))
    keys = np.repeat(ukeys, rng.integers(1, 6, groups))
    vals = _values(rng, len(keys), vtype)
    rows, _ = _rows(rng, keys, vals, 16, 8, 0)
    g, (gk, gc, gs) = _run(ctx, rows, 16, 8, 0, vtype, groups)
    vt = T.Int64 if vtype == capi.TYPE_INT64 else T.Uint64
    by = ctx.scan_filter_groupby(Column(T.Uint64, values=keys), Column(vt, values=vals), None, group_count_hint=groups)
    bk = np.asarray(by["keys"]).view(np.uint64)
    order = np.argsort(bk)
    assert g == len(bk) == groups
    assert not np.asarray(by["key_null"]).any() and not np.asarray(by["sum_null"]).any()
    assert np.array_equal(gk, bk[order])
    assert np.array_equal(gs, np.asarray(by["sum"]).view(np.uint64)[order])
    assert np.array_equal(gc, np.asarray(by["count"]).view(np.uint64)[order])


@pytest.mark.gpu
def test_capacity(ctx):
    """capacity == groups succeeds; groups - 1 and 1 fail with INVALID_ARGUMENT and report the true group count; the
    context stays usable."""
    import torch
    rng = np.random.default_rng(8)
    n = 5 * TILE + 3
    heads = rng.random(n) < 0.4
    heads[0] = True
    keys = _keys_from_heads(heads)
    vals = _values(rng, n, capi.TYPE_INT64)
    rows, _ = _rows(rng, keys, vals, 16, 0, 8)
    groups = int(heads.sum())
    for cap in (groups - 1, 1):
        outs = [torch.zeros(cap, dtype=torch.int64, device="cuda") for _ in range(3)]
        code, got = _raw(ctx, rows.data_ptr(), n, 16, 0, 8, capi.TYPE_INT64, [o.data_ptr() for o in outs], cap)
        assert code == capi.ERR_INVALID_ARGUMENT and got == groups, (cap, code, got)
        with pytest.raises(capi.YtGpuError) as e:
            _run(ctx, rows, 16, 0, 8, capi.TYPE_INT64, cap)
        assert e.value.code == capi.ERR_INVALID_ARGUMENT and "capacity" in e.value.message
    _check(ctx, rng, keys, vals, capi.TYPE_INT64, 16, 0, 8, capacity=groups)
    _check(ctx, rng, keys, vals, capi.TYPE_UINT64, 16, 0, 8, capacity=groups + 1)


@pytest.mark.gpu
def test_misaligned_pointers_are_refused(ctx):
    """Rows or outputs that are not 8-byte aligned (for example a uint8 slice rows[3:]) are INVALID_ARGUMENT, refused
    before any launch; the context stays usable."""
    import torch
    rng = np.random.default_rng(9)
    n = 1000
    keys = np.sort(rng.integers(0, 50, n, dtype=np.uint64))
    vals = _values(rng, n, capi.TYPE_INT64)
    rows, _ = _rows(rng, keys, vals, 16, 0, 8)
    buf = torch.zeros(16 * n + 16, dtype=torch.uint8, device="cuda")
    buf[3:3 + 16 * n] = rows
    outs = [torch.zeros(n + 1, dtype=torch.int64, device="cuda") for _ in range(3)]
    ptrs = [o.data_ptr() for o in outs]
    for shift in (1, 3, 4, 7):
        code, _ = _raw(ctx, buf.data_ptr() + shift, n, 16, 0, 8, capi.TYPE_INT64, ptrs, n)
        assert code == capi.ERR_INVALID_ARGUMENT, shift
    for which in range(3):
        bad = list(ptrs)
        bad[which] += 4
        code, _ = _raw(ctx, rows.data_ptr(), n, 16, 0, 8, capi.TYPE_INT64, bad, n)
        assert code == capi.ERR_INVALID_ARGUMENT, which
    with pytest.raises(capi.YtGpuError) as e:
        ctx.reduce_sorted_fixed_rows(buf[3:3 + 16 * n], 16, 0, 8, capi.TYPE_INT64, *outs)
    assert e.value.code == capi.ERR_INVALID_ARGUMENT
    _check(ctx, rng, keys, vals, capi.TYPE_INT64, 16, 0, 8)
