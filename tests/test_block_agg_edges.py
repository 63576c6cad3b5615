"""YQL block aggregators (ytgpu_block_combine_all) at the edges of the kernel's layout.

The kernel gives each thread 8 consecutive elements (one validity byte pair, one 8-byte filter word), each CTA 2048,
and at most kNumSms * 8 CTAs that stride over longer arrays; a single CTA then combines the per-CTA partials.  These
tests vary what that arithmetic depends on: lengths around 8, 2048 and the grid-stride limit, Arrow offsets that cross
validity bytes, filter and value pointers off their natural alignment, sequences of batches, and the AggLess ties of
double MIN / MAX (both zeros, NaNs with a sign bit or a payload).

The reference is the oracle's sequential AddMany.  The state must match it bit for bit, except the double SUM, whose
order the kernel chooses: it must be within (n - 1) * 2^-53 * sum|x| of the exact sum of the n selected values, and
bitwise the same for two calls and for HOST and DEVICE input of the same length (the header's reproducibility
promise)."""
import math

import numpy as np
import pytest

import oracle
from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import EValueType as T

U = 2.0 ** -53
GRID_STRIDE = 132 * 8 * 2048  # kNumSms * 8 CTAs of 2048 elements: longer arrays make a CTA loop
TYPES = ((T.Int64, np.int64), (T.Uint64, np.uint64), (T.Double, np.float64))
_PZ, _NZ = 0x0000000000000000, 0x8000000000000000
_NANS = (0x7ff8000000000000, 0xfff8000000000000, 0x7ff0000000000123, 0xfff0000000000001)


def _f(*xs):
    """Doubles from Python floats and from bit patterns given as ints."""
    return np.array([np.float64(x).view(np.uint64) if isinstance(x, float) else x for x in xs], dtype=np.uint64).view(np.float64)


def _validity(rng, valid, offset):
    """Arrow validity bitmap of exactly (offset + length + 7) / 8 bytes whose bit (offset + i) is valid[i]; the bits
    before offset and after the last element are random, so reading them shows up."""
    n = len(valid)
    bits = rng.random(offset + n + (-(offset + n)) % 8) < 0.5
    bits[offset:offset + n] = valid
    out = np.packbits(bits, bitorder="little")
    assert out.size == (offset + n + 7) // 8
    return out


def _selected(vals, valid, flt, offset, n):
    x = vals[offset:offset + n]
    sel = np.ones(n, bool)
    if valid is not None:
        sel &= valid
    if flt is not None:
        sel &= flt != 0
    return x[sel]


def _sum_within_bound(got_bits, xs):
    got = float(np.array([got_bits], dtype=np.uint64).view(np.float64)[0])
    err = math.fsum([got] + (-xs).tolist())  # got - sum(xs), exact then rounded once
    return abs(err) <= max(len(xs) - 1, 0) * U * math.fsum(np.abs(xs).tolist())


def _same(got, want, dt, xs=None, info=""):
    """Bit for bit, except a double SUM over finite values, which must be within the summation bound of xs."""
    for f in ("count", "count_all", "sum_valid", "min_valid", "max_valid", "min_value", "max_value"):
        assert getattr(got, f) == getattr(want, f), (info, f, hex(getattr(got, f)), hex(getattr(want, f)))
    if dt is np.float64 and xs is not None:
        assert _sum_within_bound(got.sum, xs), (info, hex(got.sum), hex(want.sum))
    else:
        assert got.sum == want.sum, (info, hex(got.sum), hex(want.sum))


# ---------------------------------------------------------------- the oracle's tie rule (CPU)

def _oracle_min_max(vals_bits, state=None):
    s = state or oracle.block_agg_state(T.Double, nullable=False)
    oracle.block_combine_all(s, _f(*vals_bits), nullable=False)
    return s


def test_oracle_keeps_the_last_equal_value():
    s = _oracle_min_max([_PZ, _NZ])
    assert (s.min_value, s.max_value) == (_NZ, _NZ)
    s = _oracle_min_max([_NZ, _PZ])
    assert (s.min_value, s.max_value) == (_PZ, _PZ)
    # every NaN ties with every other: the last one stays, with its sign and payload; MIN ignores them
    s = _oracle_min_max([0x7ff0000000000123, 0x4000000000000000, 0xfff8000000000000, 0x7ff0000000000001])
    assert (s.min_value, s.max_value) == (0x4000000000000000, 0x7ff0000000000001)
    # a later batch wins a tie with the state
    s = _oracle_min_max([_NZ, 0xfff8000000000000])
    s = _oracle_min_max([_PZ, 0x7ff8000000000abc], s)
    assert (s.min_value, s.max_value) == (_PZ, 0x7ff8000000000abc)


def test_validity_helper_is_exact_and_padding_is_ignored():
    rng = np.random.default_rng(1)
    vals = rng.integers(-100, 100, 80).astype(np.int64)
    valid = rng.random(17) < 0.6
    for offset in (0, 7, 8, 63):
        a = oracle.block_combine_all(oracle.block_agg_state(T.Int64), vals, _validity(rng, valid, offset), offset, 17)
        ones = np.packbits(np.r_[np.ones(offset, bool), valid], bitorder="little")
        b = oracle.block_combine_all(oracle.block_agg_state(T.Int64), vals, ones, offset, 17)
        _same(a, b, np.int64)
        assert a.count == valid.sum() and a.sum == int(vals[offset:offset + 17][valid].sum()) & (2**64 - 1)


def test_sum_bound():
    assert _sum_within_bound(_f(0x3ff0000000000000).view(np.uint64)[0], np.array([1.0, U, U]))  # (1 + u) + u == 1
    assert not _sum_within_bound(np.float64(1.0 + 8 * U).view(np.uint64), np.array([1.0, U, U]))
    assert not _sum_within_bound(np.float64(math.nextafter(0.5, 1)).view(np.uint64), np.array([0.5]))


# ---------------------------------------------------------------- GPU

@pytest.fixture(scope="module")
def ctx():
    from ytsaurus_b200 import GpuContext
    c = GpuContext(0)
    yield c
    c.close()


def _values(rng, dt, size):
    if dt is np.int64:
        return rng.integers(-2**63, 2**63 - 1, size, dtype=np.int64, endpoint=True)
    if dt is np.uint64:
        return rng.integers(0, 2**64 - 1, size, dtype=np.uint64, endpoint=True)
    return rng.standard_normal(size) * 10.0 ** rng.integers(-3, 7, size)


def _device(a):
    import torch
    if a is None:
        return None
    return torch.from_numpy(a.view(np.int64) if a.dtype.itemsize == 8 else a).cuda()


def _both(ctx, vtype, dt, vals, validity, offset, n, flt, nullable=True, info=""):
    """One call with HOST and one with DEVICE input; -> the two states.  Both must match the oracle; a double SUM
    must be the same bits in both."""
    want = oracle.block_combine_all(oracle.block_agg_state(vtype, nullable), vals, validity, offset, n, nullable, flt)
    host = ctx.block_combine_all(ctx.block_agg_state(vtype, nullable), vals.view(np.uint64), validity, offset, n, nullable, flt)
    dev = ctx.block_combine_all(ctx.block_agg_state(vtype, nullable), _device(vals), _device(validity), offset, n, nullable,
                                _device(flt))
    valid = None
    if nullable and validity is not None:
        bits = np.unpackbits(validity, bitorder="little")[offset:offset + n].astype(bool)
        valid = bits
    xs = _selected(vals, valid, flt, offset, n) if dt is np.float64 else None
    for name, got in (("host", host), ("device", dev)):
        _same(got, want, dt, xs, (info, name))
    assert host.sum == dev.sum, (info, hex(host.sum), hex(dev.sum))
    return host, dev


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 7, 8, 9, 15, 2047, 2048, 2049, 256 * 2048 + 8, GRID_STRIDE - 1, GRID_STRIDE,
                               GRID_STRIDE + 1, 3 * GRID_STRIDE + 5])
def test_lengths(ctx, n):
    """Lengths around a thread's 8 elements, a CTA's 2048, 256 CTAs (one partial per combining thread) and the
    grid-stride limit, with and without NULLs and a filter.  Two calls give the same bits."""
    rng = np.random.default_rng(n)
    for vtype, dt in TYPES:
        vals = _values(rng, dt, n)
        for with_nulls, with_filter in ((False, False), (True, True)):
            valid = rng.random(n) < 0.9 if with_nulls else None
            validity = None if valid is None else _validity(rng, valid, 0)
            flt = (rng.random(n) < 0.7).astype(np.uint8) if with_filter else None
            host, dev = _both(ctx, vtype, dt, vals, validity, 0, n, flt, info=(n, vtype, with_nulls))
        again = ctx.block_combine_all(ctx.block_agg_state(vtype), _device(vals), _device(validity), 0, n, True, _device(flt))
        assert (again.sum, again.min_value, again.max_value) == (dev.sum, dev.min_value, dev.max_value), (n, vtype)


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0, 1, 7, 8, 9, 63, 64, 65, 1000])
def test_offsets(ctx, offset):
    """Arrow offsets inside and across validity bytes, for HOST and DEVICE input, with a bitmap of exactly
    (offset + length + 7) / 8 bytes."""
    rng = np.random.default_rng(100 + offset)
    for n in (1, 13, 5000):
        for vtype, dt in TYPES:
            vals = _values(rng, dt, offset + n)
            valid = rng.random(n) < 0.7
            flt = (rng.random(n) < 0.6).astype(np.uint8)
            _both(ctx, vtype, dt, vals, _validity(rng, valid, offset), offset, n, flt, info=(offset, n, vtype))
            _both(ctx, vtype, dt, vals, _validity(rng, valid, offset), offset, n, None, info=(offset, n, vtype, "no filter"))


@pytest.mark.gpu
def test_misaligned_filter_and_values(ctx):
    """A DEVICE filter that starts 1..7 bytes into its buffer (the byte-wise filter path), and a values pointer 8 bytes
    off a 16-byte boundary (the scalar load path)."""
    import torch
    rng = np.random.default_rng(7)
    n = 4099
    for vtype, dt in TYPES:
        vals = _values(rng, dt, n + 2)
        flt = (rng.random(n) < 0.5).astype(np.uint8)
        valid = rng.random(n) < 0.8
        want = oracle.block_combine_all(oracle.block_agg_state(vtype), vals, _validity(rng, valid, 2), 2, n, True, flt)
        xs = _selected(vals, valid, flt, 2, n) if dt is np.float64 else None
        dvals = _device(vals)
        assert dvals.data_ptr() % 16 == 0
        # elements 2.. of the buffer: at offset 2 from the buffer (16-byte aligned) and at offset 1 from element 1
        # (8 bytes off a 16-byte boundary); each with its own validity bitmap
        views = ((dvals, 2, _device(_validity(rng, valid, 2))), (dvals[1:], 1, _device(_validity(rng, valid, 1))))
        sums = set()
        for shift in range(0, 8):
            buf = torch.zeros(n + 8, dtype=torch.uint8, device="cuda")
            buf[shift:shift + n] = torch.from_numpy(flt).cuda()
            f = buf[shift:shift + n]
            for v, offset, validity in views:
                got = ctx.block_combine_all(ctx.block_agg_state(vtype), v, validity, offset, n, True, f)
                _same(got, want, dt, xs, (vtype, shift, offset))
                sums.add(got.sum)
        assert len(sums) == 1, (vtype, [hex(s) for s in sums])


@pytest.mark.gpu
def test_batch_sequences(ctx):
    """Batches folded into one state: all-NULL batches, batches whose filter passes nothing, and equal extremes split
    across batches, where the later batch must win the tie like the reference's row-order loop.  The double SUM of the
    state must stay within the summation bound of every value selected so far, until a NaN makes both sums NaN."""
    rng = np.random.default_rng(8)
    seqs = {
        T.Double: [_f(_NZ, 3.0), _f(_PZ, 5.0), _f(5.0, _NZ), _f(_NANS[1], 1.0), _f(2.0, _NANS[2]), _f(_NANS[0]), _f(_PZ)],
        T.Int64: [np.array([-2**63, 2**63 - 1]), np.array([-2**63, 7]), np.array([2**63 - 1])],
        T.Uint64: [np.array([0, 2**64 - 1], np.uint64), np.array([2**64 - 1, 0], np.uint64)],
    }
    for vtype, dt in TYPES:
        for mem in ("host", "device", "mixed"):
            got, want = ctx.block_agg_state(vtype), oracle.block_agg_state(vtype)
            seen = []  # the values selected so far, over every batch
            batches = [b.astype(dt) for b in seqs[vtype]]
            # random long batches around them: some all NULL, some whose filter passes nothing
            mixed = []
            for b in batches:
                mixed.append((b, None, None))
                m = int(rng.integers(1, 3000))
                filler = _values(rng, dt, m)
                kind = rng.integers(0, 3)
                if kind == 0:
                    mixed.append((filler, np.zeros(m, bool), None))
                elif kind == 1:
                    mixed.append((filler, rng.random(m) < 0.5, np.zeros(m, np.uint8)))
                else:
                    mixed.append((b.copy(), np.ones(len(b), bool), np.ones(len(b), np.uint8)))
            for i, (vals, valid, flt) in enumerate(mixed):
                validity = None if valid is None else _validity(rng, valid, 0)
                oracle.block_combine_all(want, vals, validity, 0, len(vals), True, flt)
                on_device = mem == "device" or (mem == "mixed" and i % 2)
                if on_device:
                    ctx.block_combine_all(got, _device(vals), _device(validity), 0, len(vals), True, _device(flt))
                else:
                    ctx.block_combine_all(got, vals.view(np.uint64), validity, 0, len(vals), True, flt)
                for f in ("count", "count_all", "sum_valid", "min_valid", "max_valid", "min_value", "max_value"):
                    assert getattr(got, f) == getattr(want, f), (vtype, mem, i, f, hex(getattr(got, f)), hex(getattr(want, f)))
                if dt is np.float64:
                    seen.append(_selected(vals, valid, flt, 0, len(vals)))
                    xs = np.concatenate(seen)
                    if np.isnan(xs).any():
                        assert np.isnan(_f(got.sum)[0]) and np.isnan(_f(want.sum)[0]), (mem, i)
                    else:
                        assert _sum_within_bound(want.sum, xs), (mem, i, hex(want.sum))  # pins the model
                        assert _sum_within_bound(got.sum, xs), (mem, i, hex(got.sum), hex(want.sum))
                else:
                    assert got.sum == want.sum, (vtype, mem, i)


@pytest.mark.gpu
def test_non_nullable_column_ignores_validity(ctx):
    """A non-optional column given a validity pointer: the bitmap is not read, NULL bits and all."""
    rng = np.random.default_rng(9)
    n = 10_007
    for vtype, dt in TYPES:
        vals = _values(rng, dt, n + 9)
        validity = _validity(rng, rng.random(n) < 0.3, 9)
        flt = (rng.random(n) < 0.5).astype(np.uint8)
        host, dev = _both(ctx, vtype, dt, vals, validity, 9, n, flt, nullable=False, info=vtype)
        plain = ctx.block_combine_all(ctx.block_agg_state(vtype, False), _device(vals), None, 9, n, False, _device(flt))
        for f in ("sum", "count", "count_all", "min_value", "max_value", "sum_valid", "min_valid", "max_valid"):
            assert getattr(dev, f) == getattr(plain, f), (vtype, f)


@pytest.mark.gpu
def test_misaligned_device_values_are_refused(ctx):
    """DEVICE values that are not 8-byte aligned (a uint8 slice at byte 3) are INVALID_ARGUMENT, refused before any
    launch; the context stays usable."""
    import torch
    n = 100
    vals = np.arange(n, dtype=np.int64)
    buf = torch.zeros(8 * n + 8, dtype=torch.uint8, device="cuda")
    for shift in (1, 3, 4, 7):
        bad = buf[shift:shift + 8 * n]
        with pytest.raises(capi.YtGpuError) as e:
            ctx.block_combine_all(ctx.block_agg_state(T.Int64), bad, None, 0, n)
        assert e.value.code == capi.ERR_INVALID_ARGUMENT, shift
    got = ctx.block_combine_all(ctx.block_agg_state(T.Int64), _device(vals), None, 0, n)
    want = oracle.block_combine_all(oracle.block_agg_state(T.Int64), vals)
    _same(got, want, np.int64)
