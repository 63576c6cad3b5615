"""TIMESTAMP_FLOOR and FORMAT_TIMESTAMP as expression ops (csrc/expression.cu) against Python's own calendar.

The model is include/ytgpu.h's: seconds since the epoch, UTC, proleptic Gregorian.  Floors are integer arithmetic for the
hour, day and Monday week, and numpy's datetime64[M] / [Y] casts for the month and year; a formatted value is
time.strftime(fmt, time.gmtime(t)) in the C locale, which calls the C library's strftime.  A timestamp outside
[0, 253402300799], or a week floor before 1970-01-05, fails the call with UNSUPPORTED, but only where it is evaluated."""
import calendar
import locale
import os
import time

import numpy as np
import pytest

import oracle
from ytsaurus_b200 import capi
from ytsaurus_b200.capi import ExprConstants
from ytsaurus_b200.rowset import EValueType as T

COL, CONST, IFNULL, CONCAT, UPPER = capi.EXPR_COLUMN, capi.EXPR_CONSTANT, capi.EXPR_IF_NULL, capi.EXPR_CONCAT, capi.EXPR_UPPER
CMP, AND, IF, IN, LIKE, FARM = capi.EXPR_COMPARE, capi.EXPR_AND, capi.EXPR_IF, capi.EXPR_IN, capi.EXPR_LIKE, capi.EXPR_FARM_HASH
FLOOR, FORMAT = capi.EXPR_TIMESTAMP_FLOOR, capi.EXPR_FORMAT_TIMESTAMP
I64, U64, BOOL, STR = int(T.Int64), int(T.Uint64), int(T.Boolean), int(T.String)
MAX_T = 253402300799
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UNITS = [capi.TIMESTAMP_HOUR, capi.TIMESTAMP_DAY, capi.TIMESTAMP_WEEK, capi.TIMESTAMP_MONTH, capi.TIMESTAMP_YEAR]
SUPPORTED = "aAbBhpCdeHIjmMSuwyYDFRTUWGgVnt%"
WIDTH = dict(a=3, A=9, b=3, B=9, h=3, p=2, C=2, d=2, e=2, H=2, I=2, j=3, m=2, M=2, S=2, u=1, w=1, y=2, Y=4, D=8, F=10, R=5, T=8,
             U=2, W=2, G=4, g=2, V=2, n=1, t=1)
WIDTH["%"] = 1


class Refused(Exception):
    pass


# ------------------------------------------------------------------------------------------------- the model
def floor_model(unit, t):
    if not 0 <= t <= MAX_T:
        raise Refused()
    d = t // 86400
    if unit == capi.TIMESTAMP_HOUR:
        return t - t % 3600
    if unit == capi.TIMESTAMP_DAY:
        return d * 86400
    if unit == capi.TIMESTAMP_WEEK:
        if d < 4:
            raise Refused()
        return (d - (d + 3) % 7) * 86400
    g = time.gmtime(t)
    return calendar.timegm((g.tm_year, g.tm_mon if unit == capi.TIMESTAMP_MONTH else 1, 1, 0, 0, 0))


def floor_numpy(unit, t):
    """floor_model over an array of in-range timestamps (no week before 1970-01-05)."""
    t = np.asarray(t, np.int64)
    if unit == capi.TIMESTAMP_HOUR:
        return t - t % 3600
    d = t // 86400
    if unit == capi.TIMESTAMP_DAY:
        return d * 86400
    if unit == capi.TIMESTAMP_WEEK:  # numpy's weeks start on a Thursday, so integer arithmetic
        return (d - (d + 3) % 7) * 86400
    cast = "datetime64[M]" if unit == capi.TIMESTAMP_MONTH else "datetime64[Y]"
    return t.astype("datetime64[s]").astype(cast).astype("datetime64[s]").astype(np.int64)


def format_model(fmt, t):
    if not 0 <= t <= MAX_T:
        raise Refused()
    return time.strftime(fmt.decode("latin-1"), time.gmtime(t)).encode("latin-1")


def max_output(fmt):
    """The longest output of a supported format, as the library bounds it; None for a refused conversion."""
    n, j = 0, 0
    while j < len(fmt):
        if fmt[j:j + 1] != b"%":
            n, j = n + 1, j + 1
            continue
        c = fmt[j + 1:j + 2].decode("latin-1")
        if not c or c not in WIDTH:
            return None
        n, j = n + WIDTH[c], j + 2
    return n


def c_locale():
    locale.setlocale(locale.LC_TIME, "C")
    assert locale.setlocale(locale.LC_TIME) == "C"


# ------------------------------------------------------------------------------------------------- CPU
def test_model_edges():
    c_locale()
    assert floor_model(capi.TIMESTAMP_HOUR, 3599) == 0 and floor_model(capi.TIMESTAMP_HOUR, 3600) == 3600
    assert floor_model(capi.TIMESTAMP_DAY, 86399) == 0 and floor_model(capi.TIMESTAMP_DAY, 86400) == 86400
    assert floor_model(capi.TIMESTAMP_WEEK, 345600) == 345600  # 1970-01-05, a Monday
    with pytest.raises(Refused):
        floor_model(capi.TIMESTAMP_WEEK, 345599)
    assert time.gmtime(floor_model(capi.TIMESTAMP_WEEK, 1700000000)).tm_wday == 0  # Monday
    feb29 = calendar.timegm((2000, 2, 29, 12, 0, 0))
    assert floor_model(capi.TIMESTAMP_MONTH, feb29) == calendar.timegm((2000, 2, 1, 0, 0, 0))
    assert floor_model(capi.TIMESTAMP_YEAR, MAX_T) == calendar.timegm((9999, 1, 1, 0, 0, 0))
    assert format_model(b"%Y-%m-%dT%H:%M:%S", 0) == b"1970-01-01T00:00:00"
    assert format_model(b"%G-W%V-%u", calendar.timegm((2021, 1, 3, 0, 0, 0))) == b"2020-W53-7"
    rng = np.random.default_rng(1)
    t = rng.integers(345600, MAX_T, 20000, endpoint=True)
    for unit in UNITS:
        assert floor_numpy(unit, t).tolist() == [floor_model(unit, int(x)) for x in t]
    assert max_output(b"%A %B") == 19 and max_output(b"%A %B " + b"x" * 41 + b"%Y") == 65 and max_output(b"%c") is None and max_output(b"%") is None
    assert max(len(format_model(b"%" + c.encode(), int(x))) for c in SUPPORTED for x in t[:500]) <= 10


def test_header_exports_the_ops():
    text = open(os.path.join(ROOT, "include", "ytgpu.h")).read()
    assert "YTGPU_EXPR_TIMESTAMP_FLOOR = 30, YTGPU_EXPR_FORMAT_TIMESTAMP = 31" in text
    assert "#define YTGPU_EXPR_MAX_FORMATTED_BYTES 64" in text
    assert (capi.EXPR_TIMESTAMP_FLOOR, capi.EXPR_FORMAT_TIMESTAMP, capi.EXPR_MAX_FORMATTED_BYTES) == (30, 31, 64)


# ------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def ctx():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from ytsaurus_b200 import GpuContext
    c_locale()
    c = GpuContext(0)
    yield c
    c.close()


def _bm(flags):
    flags = np.asarray(flags, bool)
    out = np.zeros((len(flags) + 63) // 64 * 8, np.uint8)
    packed = np.packbits(flags, bitorder="little")
    out[:len(packed)] = packed
    return out


def column(kind, vtype, t, nulls=None, rng=None):
    """A column of the logical values t (int64) in one encoding: plain, packed (bit-packed above a base), dict or rle."""
    from ytsaurus_b200 import Column
    bits = np.asarray(t, np.int64).view(np.uint64)
    n = len(bits)
    nb = None if nulls is None else _bm(nulls)
    if kind == "plain":
        return Column(vtype, values=bits.copy(), value_count=n, null_bitmap=nb)
    if kind == "packed":
        base = int(bits.min())
        raw = bits - np.uint64(base)
        return Column(vtype, values=oracle.bit_pack(raw, int(raw.max())), bit_width=0, value_count=n, base_value=base)
    if kind == "dict":
        uniq, inv = np.unique(bits, return_inverse=True)
        idx = (inv.reshape(-1) + 1).astype(np.uint32)
        if nulls is not None:
            idx[np.asarray(nulls, bool)] = 0
        return Column(vtype, values=uniq, dictionary_indexes=idx, value_count=n)
    if kind == "rle":
        runs = np.flatnonzero(np.r_[True, bits[1:] != bits[:-1]])
        return Column(vtype, values=bits[runs].copy(), rle_indexes=runs.astype(np.uint64), value_count=n)
    raise ValueError(kind)


def values_of(got, n):
    vals = got["values"].view(np.uint64) if isinstance(got["values"], np.ndarray) else got["values"].cpu().numpy().view(np.uint64)
    nb = np.unpackbits(np.asarray(got["null_bitmap"]), bitorder="little")[:n].astype(bool)
    return vals, nb


def strings_of(got):
    heap, starts = bytes(np.asarray(got["heap"])), np.asarray(got["starts"]).view(np.uint64)
    lengths, nulls = np.asarray(got["lengths"]).view(np.uint32), np.asarray(got["null_bytemap"])
    return [None if nl else heap[int(s):int(s) + int(ln)] for s, ln, nl in zip(starts, lengths, nulls)], (heap, starts, lengths, nulls)


def flat(values):
    lengths = np.array([0 if v is None else len(v) for v in values], np.uint32)
    starts = np.zeros(len(values), np.uint64)
    if len(values):
        starts[1:] = np.cumsum(lengths[:-1], dtype=np.uint64)
    return b"".join(v for v in values if v is not None), starts, lengths, np.array([v is None for v in values], np.uint8)


def evaluate(ctx, cols, prog, consts=b"", selection=None, strings=False):
    sel = None if selection is None else _bm(selection)
    if strings or consts or any(node[0] == FORMAT for node in prog):
        return ctx.evaluate_expression(cols, prog, sel, string_columns=(), string_constants=consts)
    return ctx.evaluate_expression(cols, prog, sel)


def refused(ctx, cols, prog, consts=b"", selection=None, strings=False):
    with pytest.raises(capi.YtGpuError) as e:
        evaluate(ctx, cols, prog, consts, selection, strings)
    return e.value


def check_format(ctx, t, fmt, vtype=I64, nulls=None):
    c = ExprConstants()
    f = c.string(fmt)
    got = evaluate(ctx, [column("plain", vtype, t, nulls)], [(COL, 0), (FORMAT, 0, 0, f)], bytes(c))
    assert got["value_type"] == STR
    want = [None if nulls is not None and nulls[i] else format_model(fmt, int(x)) for i, x in enumerate(t)]
    values, layout = strings_of(got)
    ref = flat(want)
    assert layout[0] == ref[0], fmt
    assert np.array_equal(layout[1], ref[1]) and np.array_equal(layout[2], ref[2]) and np.array_equal(layout[3], ref[3])
    return values


EDGES = [0, 3599, 3600, 86399, 86400, 345599, 345600, calendar.timegm((2000, 2, 29, 0, 0, 0)),
         calendar.timegm((2000, 2, 29, 23, 59, 59)), calendar.timegm((2400, 2, 29, 7, 0, 0)), calendar.timegm((2100, 3, 1, 0, 0, 0)),
         calendar.timegm((2100, 2, 28, 23, 59, 59)), MAX_T, MAX_T - 1]
EDGES += [calendar.timegm((y, 12, 31, 23, 59, 59)) + k for y in range(1970, 2370) for k in (0, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", [I64, U64], ids=["i64", "u64"])
@pytest.mark.parametrize("kind", ["plain", "packed", "dict", "rle"])
def test_gpu_floors_over_encodings_and_edges(ctx, vtype, kind):
    rng = np.random.default_rng(vtype)
    t = np.array(EDGES + list(rng.integers(345600, MAX_T, 3000, endpoint=True)), np.int64)
    if kind == "rle":
        t = np.sort(np.repeat(t, rng.integers(1, 5, len(t))))  # sorted timestamps: the runs users have
    for unit in UNITS:
        ok = t >= (345600 if unit == capi.TIMESTAMP_WEEK else 0)
        tt = t[ok]
        got = evaluate(ctx, [column(kind, vtype, tt)], [(COL, 0), (FLOOR, unit)])
        assert got["value_type"] == vtype
        vals, nb = values_of(got, len(tt))
        assert not nb.any()
        assert vals.view(np.int64).tolist() == [floor_model(unit, int(x)) for x in tt], (kind, unit)
        got_s = evaluate(ctx, [column(kind, vtype, tt)], [(COL, 0), (FLOOR, unit)], strings=True, consts=b"x")
        assert np.array_equal(values_of(got_s, len(tt))[0], vals)


@pytest.mark.gpu
def test_gpu_floors_nulls_selection_and_a_million_rows(ctx):
    rng = np.random.default_rng(7)
    n = 1_000_000
    t = rng.integers(345600, MAX_T, n, endpoint=True)
    nulls = rng.random(n) < 0.1
    sel = rng.random(n) < 0.8
    for unit in UNITS:
        got = evaluate(ctx, [column("plain", I64, t, nulls)], [(COL, 0), (FLOOR, unit)], selection=sel)
        vals, nb = values_of(got, n)
        assert np.array_equal(nb, nulls | ~sel)
        live = ~nb
        assert np.array_equal(vals.view(np.int64)[live], floor_numpy(unit, t[live])), unit
        assert not vals[nb].any()


@pytest.mark.gpu
def test_gpu_refusals_follow_the_data(ctx):
    for vtype, bad in [(I64, -1), (I64, MAX_T + 1), (U64, MAX_T + 1), (I64, -(1 << 63))]:
        t = np.array([400000, bad, 500000], np.int64)
        for unit in UNITS:
            e = refused(ctx, [column("plain", vtype, t)], [(COL, 0), (FLOOR, unit)])
            assert e.code == capi.ERR_UNSUPPORTED, e.message
            # outside the selection: not evaluated
            got = evaluate(ctx, [column("plain", vtype, t)], [(COL, 0), (FLOOR, unit)], selection=[True, False, True])
            assert values_of(got, 3)[1].tolist() == [False, True, False]
    for day in range(4):  # a week floor of 1970-01-01 .. 04 would be negative
        t = np.array([86400 * day + 5, 400000], np.int64)
        assert refused(ctx, [column("plain", I64, t)], [(COL, 0), (FLOOR, capi.TIMESTAMP_WEEK)]).code == capi.ERR_UNSUPPORTED
        got = evaluate(ctx, [column("plain", I64, t)], [(COL, 0), (FLOOR, capi.TIMESTAMP_WEEK)], selection=[False, True])
        assert values_of(got, 2)[0][1] == floor_model(capi.TIMESTAMP_WEEK, 400000)
    # an IF branch not taken and FALSE AND x raise nothing: if(t >= 0, floor(t), 0) and (t >= 0) AND (floor(t) > 0)
    t = np.array([-5, 90000, -1], np.int64)
    cols = [column("plain", I64, t)]
    guard = [(COL, 0), (CONST, 0, I64, 0), (CMP, capi.CMP_GE)]
    prog = guard + [(COL, 0), (FLOOR, capi.TIMESTAMP_DAY), (CONST, 0, I64, 0), (IF,)]
    got = evaluate(ctx, cols, prog)
    assert values_of(got, 3)[0].view(np.int64).tolist() == [0, 86400, 0]
    prog_and = guard + [(COL, 0), (FLOOR, capi.TIMESTAMP_DAY), (CONST, 0, I64, 0), (CMP, capi.CMP_GT), (AND,)]
    assert values_of(evaluate(ctx, cols, prog_and), 3)[0].tolist() == [0, 1, 0]
    assert refused(ctx, cols, [(COL, 0), (FLOOR, capi.TIMESTAMP_DAY), (CONST, 0, I64, 0), (CMP, capi.CMP_GT)]).code == capi.ERR_UNSUPPORTED
    # the same for FORMAT_TIMESTAMP
    c = ExprConstants()
    f = c.string(b"%Y")
    prog = guard + [(COL, 0), (FORMAT, 0, 0, f), (CONST, 0, STR, c.string(b"-")), (IF,)]
    got = evaluate(ctx, cols, prog, bytes(c))
    assert strings_of(got)[0] == [b"-", b"1970", b"-"]
    assert refused(ctx, cols, [(COL, 0), (FORMAT, 0, 0, f)], bytes(c)).code == capi.ERR_UNSUPPORTED
    got = evaluate(ctx, cols, [(COL, 0), (FORMAT, 0, 0, f)], bytes(c), selection=[False, True, False])
    assert strings_of(got)[0] == [None, b"1970", None]


@pytest.mark.gpu
def test_gpu_format_every_conversion(ctx):
    rng = np.random.default_rng(11)
    t = np.r_[np.array(EDGES[:14], np.int64), rng.integers(0, MAX_T, 200_000, endpoint=True)]
    for c in SUPPORTED:
        check_format(ctx, t, b"%" + c.encode())
    nulls = rng.random(len(t)) < 0.1
    check_format(ctx, t, b"[%a %A %b %B %h %p %C %d %e %H %I %j]", U64, nulls)
    check_format(ctx, t, b"%m%M%S%u%w%y%Y|%D|%F|%R|%T")
    check_format(ctx, t, b"%U %W %G %g %V%n%t%%")
    big = rng.integers(0, MAX_T, 1_000_000, endpoint=True)
    check_format(ctx, big, b"%Y-%m-%dT%H:%M:%S")
    check_format(ctx, big, b"%G-W%V-%u %a %j %U %W")


@pytest.mark.gpu
def test_gpu_format_week_edges_of_every_year_type(ctx):
    """Around January 1 of 14 years: each weekday for January 1, leap and common."""
    years, kinds = [], set()
    for y in range(1971, 2100):
        k = (calendar.weekday(y, 1, 1), calendar.isleap(y))
        if k not in kinds:
            kinds.add(k)
            years.append(y)
    assert len(years) == 14
    t = [calendar.timegm((y, m, d, h, 0, 0)) for y in years for (m, d) in [(12, 25), (12, 28), (12, 29), (12, 30), (12, 31)] +
         [(1, dd) for dd in range(1, 12)] for h in (0, 23)]
    t += [calendar.timegm((y - 1, 12, dd, 12, 0, 0)) for y in years for dd in range(25, 32)]
    check_format(ctx, np.array(t, np.int64), b"%G %g %V %U %W %j %u %w %a")


@pytest.mark.gpu
def test_gpu_format_lengths_and_refusals(ctx):
    rng = np.random.default_rng(5)
    t = rng.integers(0, MAX_T, 5000, endpoint=True)
    check_format(ctx, t, b"")
    check_format(ctx, t, b"literal \xff\x01 bytes, 100%% sure")
    for target in (47, 48, 49, 64):  # values on both sides of the 48-byte short / long copy
        fmt = b"%A %B " + b"x" * (target - 24) + b"%Y"
        assert max_output(fmt) == target
        out = check_format(ctx, t, fmt)
        assert max(len(v) for v in out) == target
    c = ExprConstants()
    cols = [column("plain", I64, t[:10])]
    for fmt in [b"%A %B " + b"x" * 41 + b"%Y", b"%c", b"%x", b"%X", b"%r", b"%Z", b"%z", b"%s", b"%k", b"%l", b"%P", b"%+", b"%Ey",
                b"%Od", b"%-d", b"%10Y", b"%_H", b"%0e", b"abc%"]:
        e = refused(ctx, cols, [(COL, 0), (FORMAT, 0, 0, c.string(fmt))], bytes(c) + b"")
        assert e.code == capi.ERR_UNSUPPORTED, (fmt, e.message)
    e = refused(ctx, cols, [(COL, 0), (FORMAT, 0, 0, (1 << 40) | 3)], b"%Y%")
    assert e.code == capi.ERR_INVALID_ARGUMENT
    # the numeric entry point takes no FORMAT_TIMESTAMP; neither op takes a DOUBLE; FARM_HASH refuses a formatted value
    from ytsaurus_b200 import Column
    with pytest.raises(capi.YtGpuError):
        ctx.evaluate_expression([Column(int(T.Double), values=np.zeros(4), value_count=4)], [(COL, 0), (FLOOR, 1)])
    assert refused(ctx, cols, [(COL, 0), (FLOOR, 5)]).code == capi.ERR_INVALID_ARGUMENT
    f = c.string(b"%Y")
    assert refused(ctx, cols, [(COL, 0), (FORMAT, 0, 0, f), (FARM, 1)], bytes(c)).code == capi.ERR_UNSUPPORTED


@pytest.mark.gpu
def test_gpu_formatted_values_under_other_ops(ctx):
    rng = np.random.default_rng(9)
    n = 20000
    t = rng.integers(0, 4102444800, n)  # to 2100
    nulls = rng.random(n) < 0.1
    cols = [column("plain", I64, t, nulls), column("plain", I64, rng.integers(0, MAX_T, n))]
    c = ExprConstants()
    ym, day, long_fmt = c.string(b"%Y-%m"), c.string(b"%d"), c.string(b"%A, %d %B %Y %H:%M:%S (week %V of %G) %%")
    sep, target, none = c.string(b"/"), c.string(b"2024-03"), c.string(b"none")
    pattern = c.string(b"20_4-0%")
    lst = c.in_list([b"2024-03", b"1999-12", b"2050-01"])
    consts = bytes(c)
    fm = lambda fmt, x: None if x is None else format_model(fmt, x)  # noqa: E731
    a = [None if nulls[i] else int(t[i]) for i in range(n)]
    b = [int(x) for x in cols[1].values.view(np.int64)]
    ya, da, la = [fm(b"%Y-%m", x) for x in a], [fm(b"%d", x) for x in b], [fm(b"%A, %d %B %Y %H:%M:%S (week %V of %G) %%", x) for x in a]
    cases = [
        ([(COL, 0), (FORMAT, 0, 0, ym), (CONST, 0, STR, sep), (CONCAT,), (COL, 1), (FORMAT, 0, 0, day), (CONCAT,)],
         [None if x is None else x + b"/" + y for x, y in zip(ya, da)]),                              # two FORMAT nodes
        ([(COL, 0), (FORMAT, 0, 0, long_fmt), (UPPER,)], [None if x is None else x.upper() for x in la]),
        ([(COL, 0), (FORMAT, 0, 0, ym), (CONST, 0, STR, none), (IFNULL, 0, STR)], [x or b"none" for x in ya]),
        ([(COL, 0), (FORMAT, 0, 0, ym), (CONST, 0, STR, target), (CMP, capi.CMP_EQ)], [None if x is None else int(x == b"2024-03") for x in ya]),
        ([(COL, 0), (FORMAT, 0, 0, ym), (IN, 0, 0, lst)], [None if x is None else int(x in (b"2024-03", b"1999-12", b"2050-01")) for x in ya]),
        ([(COL, 0), (FORMAT, 0, 0, ym), (LIKE, -1, 0, pattern)], [None if x is None else int(x[:2] == b"20" and x[3:6] == b"4-0") for x in ya]),
        ([(COL, 1), (CONST, 0, I64, 2000000000), (CMP, capi.CMP_LT), (COL, 0), (FORMAT, 0, 0, long_fmt), (COL, 1), (FORMAT, 0, 0, ym), (IF,)],
         [(la[i] if b[i] < 2000000000 else fm(b"%Y-%m", b[i])) for i in range(n)]),
    ]
    for prog, want in cases:
        got = evaluate(ctx, cols, prog, consts)
        if got["value_type"] == STR:
            vals, layout = strings_of(got)
            ref = flat(want)
            assert layout[0] == ref[0] and all(np.array_equal(x, y) for x, y in zip(layout[1:], ref[1:])), prog
        else:
            v, nb = values_of(got, n)
            assert [None if nb[i] else int(v[i]) for i in range(n)] == want, prog


@pytest.mark.gpu
def test_gpu_host_adapter_timestamps():
    import subprocess
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "timestamp_expression_ut"], stdout=subprocess.DEVNULL)
    r = subprocess.run([os.path.join(ROOT, "host", "timestamp_expression_ut")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "timestamp_expression_ut: 0 failure(s)" in r.stdout
