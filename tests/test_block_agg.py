"""YQL block aggregators, combine-all form (SURVEY.md §8 a18 / (f) rank 4).

CPU: the oracle restates one AddMany of the reference's sum/avg/min/max/count/count_all aggregators and is pinned by the
reference's own unit tests (yql/essentials/minikql/comp_nodes/ut/mkql_block_agg_ut.cpp:232-265; its ui32 vectors run
here through the 64-bit instantiations of the same templates).
GPU: ytgpu_block_combine_all must leave the SAME state: integers bit for bit, double sums to 1e-12 relative (the
reference's running sum is order dependent), min/max bit for bit: under AggLess (NaN is the biggest value, all NaNs
and both zeros are equal) the last equal value in row order stays, with its sign and NaN payload."""
import numpy as np
import pytest

import oracle
from ytsaurus_b200.rowset import EValueType as T


def _bits(x, dtype):
    return int(np.array([x], dtype=dtype).view(np.uint64)[0])


def _as(state_value, dtype):
    return np.array([state_value], dtype=np.uint64).view(dtype)[0]


def _validity(valid_bool, offset):
    """Arrow validity bitmap whose bit (offset + i) describes element i."""
    bits = np.concatenate([np.ones(offset, dtype=bool), np.asarray(valid_bool, dtype=bool)])
    return np.packbits(bits, bitorder="little")


def test_oracle_reference_unit_test_vectors():
    # CombineAllMultipleAggsMixedTypes (:242-249): min 2, max 9 over {5, 2, 9, 2}
    s = oracle.block_combine_all(oracle.block_agg_state(T.Uint64, nullable=False), np.array([5, 2, 9, 2], dtype=np.uint64), nullable=False)
    assert (s.min_value, s.max_value, s.count, s.count_all) == (2, 9, 4, 4)
    # CombineAllWithFilterColumn (:251-259): count_all 3, min 1
    s = oracle.block_combine_all(oracle.block_agg_state(T.Uint64, nullable=False), np.arange(1, 6, dtype=np.uint64), nullable=False,
                                 filter=np.array([1, 0, 1, 0, 1], dtype=np.uint8))
    assert (s.count_all, s.min_value, s.sum, s.max_value) == (3, 1, 9, 5)
    # CombineAllCountOverNullableArray (:232-236): count skips nulls
    s = oracle.block_combine_all(oracle.block_agg_state(T.Int64), np.array([10, 0, 30], dtype=np.int64),
                                 validity=_validity([1, 0, 1], 0))
    assert (s.count, s.count_all, s.sum, s.sum_valid) == (2, 3, 40, 1)
    # CombineAllEmptyInput (:261-265): nothing is produced, the state stays initial
    s = oracle.block_combine_all(oracle.block_agg_state(T.Int64), np.zeros(0, dtype=np.int64))
    assert (s.count_all, s.sum_valid, s.min_valid) == (0, 0, 0)


def test_oracle_isvalid_rules_and_float_order():
    vals = np.array([3.5, np.nan, -1.0, 7.25], dtype=np.float64)
    # no nulls, filter passes nothing: sum's IsValid is still raised (mkql_block_agg_sum.cpp:221-228), min/max's is not
    s = oracle.block_combine_all(oracle.block_agg_state(T.Double), vals, filter=np.zeros(4, np.uint8))
    assert (s.sum_valid, s.min_valid, s.max_valid, s.count, s.count_all) == (1, 0, 0, 0, 0)
    # with nulls in the batch the filtered sum only becomes valid when something was added (:208-220)
    s = oracle.block_combine_all(oracle.block_agg_state(T.Double), vals, validity=_validity([1, 1, 0, 1], 0), filter=np.zeros(4, np.uint8))
    assert s.sum_valid == 0
    # an all-null batch changes nothing but count_all
    s = oracle.block_combine_all(oracle.block_agg_state(T.Double), vals, validity=_validity([0, 0, 0, 0], 0))
    assert (s.sum_valid, s.count, s.count_all) == (0, 0, 4)
    # NaN is the biggest value: max is NaN, min ignores it
    s = oracle.block_combine_all(oracle.block_agg_state(T.Double), vals)
    assert np.isnan(_as(s.max_value, np.float64)) and _as(s.min_value, np.float64) == -1.0
    # integers wrap
    s = oracle.block_combine_all(oracle.block_agg_state(T.Uint64), np.array([2**64 - 1, 5], dtype=np.uint64))
    assert s.sum == 4


# Doubles that AggLess ranks equal but whose bits differ: both zeros, and NaNs with a sign bit or a payload.
_TIES = np.array([0x0000000000000000, 0x8000000000000000, 0x7ff8000000000000, 0xfff8000000000000,
                  0x7ff0000000000123, 0xfff0000000000001, 0x3ff0000000000000], dtype=np.uint64).view(np.float64)


def _cases(rng):
    out = []
    for n in (1, 2, 7, 8, 9, 1000, 100_003):
        for vtype, dt in ((T.Int64, np.int64), (T.Uint64, np.uint64), (T.Double, np.float64)):
            if dt is np.float64:
                vals = rng.normal(0, 1e6, n + 5)
                if n > 8:
                    vals[rng.integers(0, n, 3)] = [np.nan, np.inf, -np.inf]
                # MIN is mostly a zero and MAX a NaN; at n = 2 offsets 0 and 3 see [+0.0, -0.0] and [-0.0, +0.0]
                ties = np.resize(_TIES[:2], n + 5) if n == 2 else rng.choice(_TIES, n + 5)
                domains = (vals, ties)
            elif dt is np.int64:
                domains = (rng.integers(-2**62, 2**62, n + 5, dtype=np.int64),)
            else:
                domains = (rng.integers(0, 2**64 - 1, n + 5, dtype=np.uint64),)
            for vals in domains:
                for offset in (0, 3):
                    for with_nulls in (False, True):
                        for with_filter in (False, True):
                            valid = rng.random(n) < 0.8 if with_nulls else None
                            flt = (rng.random(n) < 0.5).astype(np.uint8) if with_filter else None
                            out.append((vtype, dt, vals.astype(dt), offset, n, valid, flt))
    return out


def _same_state(got, want, dt, ctxinfo):
    assert (got.count, got.count_all) == (want.count, want.count_all), ctxinfo
    assert (got.sum_valid, got.min_valid, got.max_valid) == (want.sum_valid, want.min_valid, want.max_valid), ctxinfo
    if dt is np.float64:
        a, b = _as(got.sum, dt), _as(want.sum, dt)
        assert (np.isnan(a) and np.isnan(b)) or a == b or abs(a - b) <= 1e-12 * max(abs(a), abs(b), 1e6), (ctxinfo, a, b)
    else:
        assert got.sum == want.sum, ctxinfo
    assert (hex(got.min_value), hex(got.max_value)) == (hex(want.min_value), hex(want.max_value)), ctxinfo


@pytest.fixture(scope="module")
def ctx():
    from ytsaurus_b200 import GpuContext
    return GpuContext(0)


@pytest.mark.gpu
@pytest.mark.parametrize("device_memory", [False, True])
def test_gpu_combine_all_matches_oracle(ctx, device_memory):
    import torch
    rng = np.random.default_rng(31)
    for vtype, dt, vals, offset, n, valid, flt in _cases(rng):
        validity = None if valid is None else _validity(valid, offset)
        want = oracle.block_combine_all(oracle.block_agg_state(vtype), vals, validity, offset, n, True, flt)
        v, vb, f = vals.view(np.uint64), validity, flt
        if device_memory:
            v = torch.from_numpy(vals.view(np.int64)).cuda()
            vb = None if validity is None else torch.from_numpy(validity).cuda()
            f = None if flt is None else torch.from_numpy(flt).cuda()
        got = ctx.block_combine_all(ctx.block_agg_state(vtype), v, vb, offset, n, True, f)
        _same_state(got, want, dt, (vtype, offset, n, valid is not None, flt is not None))


@pytest.mark.gpu
def test_gpu_combine_all_accumulates_batches_and_non_optional(ctx):
    rng = np.random.default_rng(32)
    for nullable in (True, False):
        got, want = ctx.block_agg_state(T.Int64, nullable), oracle.block_agg_state(T.Int64, nullable)
        for _ in range(6):
            n = int(rng.integers(0, 5000))
            vals = rng.integers(-10**9, 10**9, n, dtype=np.int64)
            valid = rng.random(n) < rng.choice([0.0, 0.5, 1.0])
            flt = (rng.random(n) < rng.choice([0.0, 0.7])).astype(np.uint8) if rng.random() < 0.6 else None
            validity = _validity(valid, 0) if nullable else None
            oracle.block_combine_all(want, vals, validity, 0, n, nullable, flt)
            ctx.block_combine_all(got, vals.view(np.uint64), validity, 0, n, nullable, flt)
            _same_state(got, want, np.int64, (nullable, n))


@pytest.mark.gpu
def test_gpu_combine_all_reference_vectors_and_errors(ctx):
    from ytsaurus_b200.capi import YtGpuError
    s = ctx.block_combine_all(ctx.block_agg_state(T.Uint64, nullable=False), np.arange(1, 6, dtype=np.uint64), nullable=False,
                              filter=np.array([1, 0, 1, 0, 1], dtype=np.uint8))
    assert (s.count_all, s.min_value, s.sum, s.max_value) == (3, 1, 9, 5)
    s = ctx.block_combine_all(ctx.block_agg_state(T.Double), np.array([3.5, np.nan, -1.0, 7.25]).view(np.uint64))
    assert np.isnan(_as(s.max_value, np.float64)) and _as(s.min_value, np.float64) == -1.0
    with pytest.raises(YtGpuError):
        ctx.block_combine_all(ctx.block_agg_state(T.Boolean), np.zeros(4, np.uint64))
    empty = ctx.block_combine_all(ctx.block_agg_state(T.Int64), np.zeros(0, np.uint64))  # CombineAllEmptyInput
    assert (empty.count_all, empty.sum_valid, empty.min_valid) == (0, 0, 0)


@pytest.mark.gpu
def test_gpu_combine_hashed_over_arrow_blocks(ctx):
    """BlockCombineHashed with sum/count over one 64-bit key == ytgpu_scan_filter_groupby on columns whose bitmaps are
    Arrow validity bitmaps (YTGPU_COLUMN_ARROW_VALIDITY): same groups as the oracle's hash aggregation, and identical to
    the result obtained from the inverted (YT-style null) bitmaps."""
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(33)
    n = 200_000
    keys = rng.integers(0, 3000, n, dtype=np.uint64)
    vals = rng.integers(-10**12, 10**12, n, dtype=np.int64)
    key_valid, val_valid = rng.random(n) < 0.97, rng.random(n) < 0.9
    arrow = ctx.scan_filter_groupby(
        Column(T.Uint64, values=keys, null_bitmap=np.packbits(key_valid, bitorder="little"), arrow_validity=True),
        Column(T.Int64, values=vals.view(np.uint64), null_bitmap=np.packbits(val_valid, bitorder="little"), arrow_validity=True),
        None, group_count_hint=3002)
    yt = ctx.scan_filter_groupby(
        Column(T.Uint64, values=keys, null_bitmap=np.packbits(~key_valid, bitorder="little")),
        Column(T.Int64, values=vals.view(np.uint64), null_bitmap=np.packbits(~val_valid, bitorder="little")),
        None, group_count_hint=3002)
    for field in ("keys", "key_null", "sum", "sum_null", "count"):
        assert (np.asarray(arrow[field]) == np.asarray(yt[field])).all(), field
    want = oracle.groupby_sum_count(keys, vals, oracle.VAL_INT64, (~key_valid).astype(np.uint8), (~val_valid).astype(np.uint8),
                                    style=oracle.STYLE_CH)
    order = np.lexsort((want["keys"], want["key_null"]))
    for field in ("keys", "key_null", "sum", "sum_null", "count"):
        got = np.asarray(arrow[field])
        if field == "sum":  # the sum of a group without any non-null value is NULL; its payload is unspecified
            live = np.asarray(arrow["sum_null"]) == 0
            assert (got[live] == want[field][order][live]).all(), field
        else:
            assert (got == want[field][order]).all(), field


@pytest.mark.gpu
def test_gpu_combine_all_large_block(ctx):
    import torch
    n = 20_000_000
    g = torch.Generator(device="cuda").manual_seed(3)
    vals = torch.randint(-2**40, 2**40, (n,), device="cuda", generator=g, dtype=torch.int64)
    flt = (torch.rand(n, device="cuda", generator=g) < 0.5).to(torch.uint8)
    s = ctx.block_combine_all(ctx.block_agg_state(T.Int64, nullable=False), vals, nullable=False, filter=flt)
    sel = flt.bool()
    assert s.count_all == int(sel.sum()) and s.count == s.count_all
    assert _as(s.sum, np.int64) == int(vals[sel].sum()) and _as(s.min_value, np.int64) == int(vals[sel].min())
    assert _as(s.max_value, np.int64) == int(vals[sel].max())
