"""GROUP BY tables with string-valued aggregates (ytgpu_groupby_table_*_strings): MIN, MAX, FIRST, COUNT, ARGMIN and ARGMAX
over strings, folded block by block, must give exactly what the one-shot ytgpu_scan_filter_groupby_multi_strings gives over
the concatenated blocks, and carry the selected strings' bytes, which the table owns."""
import ctypes as C
import importlib.util
import os
import re
import subprocess
import zlib

import numpy as np
import pytest

from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import EValueType as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name):
    spec = importlib.util.spec_from_file_location("_groupby_table_strings_" + name[:-3], os.path.join(os.path.dirname(os.path.abspath(__file__)), name))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


GT = _load("test_groupby_table.py")  # values(), column(), string_block(), keys_for(), host()
M = GT.M
host = GT.host
S, MN, MX, CNT, AVG, AMIN, AMAX, FIRST = GT.S, GT.MN, GT.MX, GT.CNT, GT.AVG, GT.AMIN, GT.AMAX, GT.FIRST
VALUE_TYPES = GT.VALUE_TYPES  # 0 int64, 1 uint64, 2 double, 3 boolean; string values are columns 4 and 5
V = len(VALUE_TYPES)
S0, S1 = V, V + 1
STRING_OPS = [(MN, S0), (MX, S0), (FIRST, S0), (CNT, S0), (MN, S1), (MX, S1),
              (AMIN, S0, 0), (AMAX, S0, 1),   # the string as the value
              (AMIN, 1, S1), (AMAX, 0, S0),   # the string as the bound
              (AMIN, S0, S1), (AMAX, S1, S0)]  # both
AGGREGATES = STRING_OPS + [(S, 0), (MN, 2), (AMIN, 1, 0), (FIRST, 3), (CNT, 1)]


def string_valued(agg):
    return agg[1] >= V and agg[0] != CNT


@pytest.fixture(scope="module")
def ctx():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from ytsaurus_b200 import GpuContext
    c = GpuContext(0)
    yield c
    c.close()


# ------------------------------------------------------------------------------------------------- inputs
EDGES = [b"", b"a", b"ab", b"a\x00", b"\x00", b"\x00\x00", b"a\x00b", bytes([0x80]), bytes([0xff, 0x00]), bytes([0x7f]), b"b", b"ba"]


def string_values(rng, n, distinct, long_values=()):
    pool = [bytes(rng.integers(0, 256, rng.integers(0, 301), dtype=np.uint8)) for _ in range(distinct)]
    pool += [bytes(rng.integers(0, 4, L, dtype=np.uint8)) for L in range(0, 301, 7)] + EDGES  # lengths 0..300, shared prefixes
    vals = [pool[i] for i in rng.integers(0, len(pool), n)]
    for i, v in long_values:
        vals[i] = v
    return vals, rng.random(n) < 0.1


def string_keys(rng, n, distinct):
    pool = [bytes(rng.integers(0, 256, rng.integers(0, 20), dtype=np.uint8)) for _ in range(distinct)] + [b""]
    return [pool[i] for i in rng.integers(0, len(pool), n)], rng.random(n) < 0.05


def ids_of(vals, nulls):
    """String keys as dense int64 ids (NULL stays NULL): the one-shot call groups them exactly as the table groups strings."""
    seen = {}
    ids = np.asarray([seen.setdefault(v, len(seen)) for v in vals], np.uint64)
    return np.where(nulls, 0, ids).astype(np.uint64), nulls.copy()


def pass_mask(vals, pred, a, b):
    if pred is None:
        return np.ones(b - a, bool)
    op, c = pred
    x, nl = vals[0][0][a:b].view(np.int64), vals[0][1][a:b]
    return {capi.CMP_GT: x > c, capi.CMP_LT: x < c}[op] & ~nl


class Case:
    """One table's inputs: numeric keys, string keys, numeric values and string values over n rows."""

    def __init__(self, rng, n, shape, groups=300, long_values=()):
        numeric, nstr = {"numeric": ([T.Int64, T.Boolean], 0), "string": ([], 1), "mixed": ([T.Int64], 1)}[shape]
        self.numeric = numeric
        self.nkeys = GT.keys_for(rng, numeric, n, groups)
        self.skeys = [string_keys(rng, n, groups) for _ in range(nstr)]
        self.vals = GT.values(rng, n)
        self.svals = [string_values(rng, n, 200, long_values), string_values(rng, n, 50)]
        self.n = n


def feed(t, case, bounds, preds, rng, device=False):
    passes = []
    for i in range(len(bounds) - 1):
        a, b = bounds[i], bounds[i + 1]
        kc = [GT.column(tp, v[a:b], nl[a:b]) for tp, (v, nl) in zip(case.numeric, case.nkeys)]
        vc = [GT.column(tp, v[a:b], nl[a:b]) for tp, (v, nl) in zip(VALUE_TYPES, case.vals)]
        if device:
            for c in kc + vc:
                M.to_device(c)
        sk = [GT.string_block(sv[a:b], sn[a:b], rng, device) for sv, sn in case.skeys]
        sv = [GT.string_block(sv[a:b], sn[a:b], rng, device) for sv, sn in case.svals]
        pred = preds[i]
        t.update(kc, vc, string_keys=sk, predicate=pred, predicate_column=0 if pred else -1, string_values=sv)
        passes.append(pass_mask(case.vals, pred, a, b))
    return np.concatenate(passes)


def one_shot(ctx, case, aggs, passes):
    """The one-shot call over the concatenated rows: string keys as ids, the pass flags as an extra value column."""
    rng = np.random.default_rng(0)
    kc = [GT.column(tp, v, nl) for tp, (v, nl) in zip(case.numeric, case.nkeys)]
    kc += [GT.column(T.Int64, *ids_of(sv, sn)) for sv, sn in case.skeys]
    vc = [GT.column(tp, v, nl) for tp, (v, nl) in zip(VALUE_TYPES, case.vals)]
    vc.append(GT.column(T.Uint64, passes.astype(np.uint64), np.zeros(case.n, bool), "plain"))
    shift = [(a[0],) + tuple(c + 1 if c >= V else c for c in a[1:]) for a in aggs]  # string columns move past the flags
    sc = [GT.string_block(sv, sn, rng) for sv, sn in case.svals]
    return ctx.scan_filter_groupby_multi(kc, vc, shift, predicate=(capi.CMP_EQ, 1), predicate_column=len(vc) - 1, string_columns=sc)


def string_at(res, j, o):
    heap, starts, lengths, nulls = (host(x) for x in res["string_values"][j])
    if nulls[o]:
        return None
    return bytes(heap[int(starts[o]):int(starts[o]) + int(lengths[o])])


def assert_matches_one_shot(got, ref, case, aggs):
    g = len(host(ref["count"]))
    assert len(host(got["count"])) == g
    for k in ("count", "first_row"):
        assert (host(got[k]).view(np.uint64) == host(ref[k]).view(np.uint64)).all(), k
    for k in range(len(case.numeric)):
        kn = host(ref["key_null"][k]).astype(bool)
        assert (host(got["key_null"][k]).astype(bool) == kn).all()
        assert (host(got["keys"][k]).view(np.uint64)[~kn] == host(ref["keys"][k]).view(np.uint64)[~kn]).all()
    # string keys: the bytes of the id the one-shot grouped by
    for s, (sv, sn) in enumerate(case.skeys):
        kn = host(ref["key_null"][len(case.numeric) + s]).astype(bool)
        first = host(ref["first_row"])
        heap, starts, lengths, nulls = (host(x) for x in got["string_keys"][s])
        assert (nulls.astype(bool) == kn).all()
        for o in np.flatnonzero(~kn):
            assert bytes(heap[int(starts[o]):int(starts[o]) + int(lengths[o])]) == sv[int(first[o])]
    j = 0
    for a, agg in enumerate(aggs):
        vn = host(ref["value_null"][a]).astype(bool)
        assert (host(got["value_null"][a]).astype(bool) == vn).all(), agg
        gv, rv = host(got["values"][a]).view(np.uint64), host(ref["values"][a]).view(np.uint64)
        assert (gv[~vn] == rv[~vn]).all(), agg
        if string_valued(agg):
            col = case.svals[agg[1] - V][0]
            heap, starts, lengths, nulls = (host(x) for x in got["string_values"][j])
            assert (nulls.astype(bool) == vn).all(), agg
            assert (lengths[vn] == 0).all()
            for o in np.flatnonzero(~vn):
                assert bytes(heap[int(starts[o]):int(starts[o]) + int(lengths[o])]) == col[int(gv[o])], (agg, o)
            j += 1
    assert j == len(got["string_values"])


def dict_group_by(case, passes, aggs):
    """A plain GROUP BY over the string ops (MIN / MAX / FIRST / COUNT; ARGMIN / ARGMAX by int64 column 0 or a string):
    group key -> list of (row or count) per aggregate, None for NULL."""
    def key(i):
        return (tuple(None if nl[i] else int(v[i]) for v, nl in case.nkeys) + tuple(None if sn[i] else sv[i] for sv, sn in case.skeys))

    def arg(c, i):
        if c >= V:
            sv, sn = case.svals[c - V]
            return None if sn[i] else sv[i]
        v, nl = case.vals[c]
        return None if nl[i] else int(v[i].view(np.int64)) if c == 0 else int(v[i])

    groups = {}
    for i in np.flatnonzero(passes):
        g = groups.setdefault(key(i), [None] * len(aggs))
        for a, agg in enumerate(aggs):
            op, c = agg[0], agg[1]
            if not any(x >= V for x in agg[1:]):
                continue
            x = arg(c, i)
            if op == CNT:
                g[a] = (g[a] or 0) + (x is not None)
                continue
            if x is None:
                continue
            if op == FIRST:
                g[a] = g[a] if g[a] is not None else (i, None)
                continue
            by = x if op in (MN, MX) else arg(agg[2], i)
            if by is None:
                continue
            larger = op in (MX, AMAX)
            if g[a] is None or (by > g[a][1] if larger else by < g[a][1]):
                g[a] = (i, by)
    return {k: [x if isinstance(x, int) or x is None else x[0] for x in v] for k, v in groups.items()}


def assert_matches_dict(got, case, passes, aggs):
    ref = dict_group_by(case, passes, aggs)
    first = host(got["first_row"])
    assert len(first) == len(ref)
    for o in range(len(first)):
        i = int(first[o])
        k = (tuple(None if nl[i] else int(v[i]) for v, nl in case.nkeys) + tuple(None if sn[i] else sv[i] for sv, sn in case.skeys))
        for a, agg in enumerate(aggs):
            if not any(x >= V for x in agg[1:]):
                continue
            want = ref[k][a]
            if host(got["value_null"][a])[o]:
                assert want is None or (agg[0] == CNT and want == 0), (agg, o)
            elif agg[0] == CNT:
                assert int(host(got["values"][a])[o]) == want, agg
            elif string_valued(agg):
                assert int(host(got["values"][a])[o]) == want, (agg, o)


CUTS = [1, 31, 2049, 65537]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["numeric", "string", "mixed"])
@pytest.mark.parametrize("device", [False, True])
def test_blocks_match_one_shot_and_a_dict_group_by(ctx, shape, device):
    rng = np.random.default_rng(zlib.crc32(f"{shape}{device}".encode()))
    bounds = list(np.cumsum([0] + CUTS)) + [sum(CUTS) + 3001]
    n = bounds[-1]
    case = Case(rng, n, shape)
    preds = [None, (capi.CMP_GT, -10), None, (capi.CMP_LT, 30), (capi.CMP_GT, -45)]
    with ctx.groupby_table(case.numeric, len(case.skeys), VALUE_TYPES, AGGREGATES, string_value_count=2) as t:
        passes = feed(t, case, bounds, preds, rng, device)
        got = t.result(out_mem=capi.MEM_DEVICE if device else capi.MEM_HOST)
    assert_matches_one_shot(got, one_shot(ctx, case, AGGREGATES, passes), case, AGGREGATES)
    assert_matches_dict(got, case, passes, AGGREGATES)


@pytest.mark.gpu
def test_string_edges(ctx):
    """"" against NULL, prefixes, embedded zeros, bytes >= 0x80, lengths 0..300, two 64 KiB values, a tie across blocks
    and a group whose only non-NULL value arrives in the last block."""
    rng = np.random.default_rng(11)
    n = 6000
    big = [(100, bytes([0x41]) * 65536), (4500, bytes([0x41]) * 65535 + b"\x00")]
    case = Case(rng, n, "numeric", groups=40, long_values=big)
    key, knull = case.nkeys[0]
    key[:], knull[:] = rng.integers(0, 40, n), False
    case.nkeys[1] = (np.zeros(n, np.uint64), np.zeros(n, bool))
    # group 1000: "" at rows 10 and 3010 (a tie across blocks), NULL elsewhere; group 1001: NULL until the last block;
    # group 1002: equal string bounds in two blocks; group 1003: the two 64 KiB values, equal but for the last byte
    s0, s0n = case.svals[0]
    s1, s1n = case.svals[1]
    for r in range(20, 5900, 97):
        key[r], s0n[r] = 1000, True
    for r in range(30, 6000, 89):
        key[r], s0n[r] = 1001, r < 5000
    for r in (10, 3010):
        key[r], s0[r], s0n[r] = 1000, b"", False
    for r in (40, 3040):
        key[r], s1[r], s1n[r], s0n[r] = 1002, b"tie", False, False
    for r, _ in big:
        key[r], s0n[r] = 1003, False
    bounds = [0, 3000, 5000, n]
    with ctx.groupby_table(case.numeric, 0, VALUE_TYPES, AGGREGATES, string_value_count=2) as t:
        passes = feed(t, case, bounds, [None] * 3, rng)
        got = t.result()
    assert_matches_one_shot(got, one_shot(ctx, case, AGGREGATES, passes), case, AGGREGATES)
    assert_matches_dict(got, case, passes, AGGREGATES)
    keys = list(host(got["keys"][0]))
    j = {agg: sum(string_valued(x) for x in AGGREGATES[:a]) for a, agg in enumerate(AGGREGATES)}  # string output index

    def result(agg, group):
        o = keys.index(group)
        a = AGGREGATES.index(agg)
        return int(host(got["values"][a])[o]), string_at(got, j[agg], o)

    assert result((MN, S0), 1000) == (10, b"")  # "" is a value, NULL is not; the earlier block keeps the tie
    assert result((MX, S0), 1000) == (10, b"")
    first_late = min(r for r in range(30, 6000, 89) if r >= 5000)
    assert result((FIRST, S0), 1001) == (first_late, s0[first_late])
    assert result((AMIN, S0, S1), 1002) == (40, s0[40])
    assert result((MN, S0), 1003) == (4500, big[1][1]) and result((MX, S0), 1003) == (100, big[0][1])


@pytest.mark.gpu
def test_reclaiming_under_strictly_improving_minimums(ctx):
    """Every update improves every group's MIN, so the MIN heap fills with replaced values and is compacted again and
    again; MAX and FIRST keep their first values."""
    groups, updates, width = 10**4, 300, 100
    rng = np.random.default_rng(12)
    tail = rng.integers(0, 256, (groups, width - 1), dtype=np.uint8)
    gkeys = rng.permutation(groups).astype(np.uint64)
    vals = [(np.zeros(groups, np.uint64), np.zeros(groups, bool)) for _ in VALUE_TYPES]
    vc = [GT.column(tp, v, nl) for tp, (v, nl) in zip(VALUE_TYPES, vals)]
    kc = [GT.column(T.Int64, gkeys, np.zeros(groups, bool))]
    aggs = [(MN, S0), (MX, S0), (FIRST, S0), (AMIN, 0, S0)]
    starts = np.arange(groups, dtype=np.uint64) * width
    lengths = np.full(groups, width, np.uint32)

    def block(u):
        rows = np.concatenate([np.full((groups, 1), 255 - u // 2, np.uint8), tail], axis=1)
        rows[:, 1] = (rows[:, 1] & 0x7f) | (0x80 if u % 2 == 0 else 0)  # two steps per leading byte: still descending
        return rows

    with ctx.groupby_table([T.Int64], 0, VALUE_TYPES, aggs, string_value_count=1) as t:
        for u in range(updates):
            rows = block(u)
            t.update(kc, vc, string_values=[(rows.reshape(-1).copy(), starts, lengths, None)])
            if u % 25 == 24 or u == updates - 1:
                got = t.result()
                order = host(got["keys"][0]).astype(np.int64)
                assert (order == gkeys.astype(np.int64)).all()
                last, firsts = rows, block(0)
                for j, (want_rows, want_block) in enumerate([(u, last), (0, firsts), (0, firsts)]):
                    assert (host(got["values"][j]) == np.arange(groups, dtype=np.uint64) + want_rows * groups).all()
                    heap, st, ln, nl = (host(x) for x in got["string_values"][j])
                    assert not nl.any() and (ln == width).all()
                    assert (heap.reshape(groups, width) == want_block).all()
                assert (host(got["values"][3]) == 0).all()  # ARGMIN's value: column 0, all zero


# ------------------------------------------------------------------------------------------------- refusals
def _code(fn):
    with pytest.raises(capi.YtGpuError) as e:
        fn()
    return e.value.code


@pytest.mark.gpu
def test_refusals(ctx):
    rng = np.random.default_rng(13)
    n = 800
    case = Case(rng, n, "mixed", groups=30)
    aggs = [(MN, S0), (AMAX, 0, S1), (CNT, S1), (S, 0)]
    kc = [GT.column(T.Int64, *case.nkeys[0])]
    vc = [GT.column(tp, v, nl) for tp, (v, nl) in zip(VALUE_TYPES, case.vals)]
    sk = [GT.string_block(*case.skeys[0], rng)]
    t = ctx.groupby_table([T.Int64], 1, VALUE_TYPES, aggs, string_value_count=2)
    sv = [GT.string_block(*c, rng) for c in case.svals]
    t.update(kc, vc, string_keys=sk, string_values=sv)
    before = t.result()

    def same_as_before():
        after = t.result()
        for k in ("count", "first_row"):
            assert (host(after[k]) == host(before[k])).all()
        assert all((host(a) == host(b)).all() for a, b in zip(after["values"], before["values"]))
        for a, b in zip(after["string_values"] + after["string_keys"], before["string_values"] + before["string_keys"]):
            assert all((host(x) == host(y)).all() for x, y in zip(a, b))

    # a value outside its heap, in a row the predicate drops, with a new string key that must not reach the dictionary
    x = case.vals[0][0].view(np.int64)
    dropped = int(np.flatnonzero((x <= 0) & ~case.vals[0][1])[0])
    for c in (0, 1):
        bad = list(GT.string_block(*case.svals[c], rng))
        bad[1], bad[2], bad[3] = bad[1].copy(), bad[2].copy(), np.zeros(n, np.uint8)
        bad[1][dropped], bad[2][dropped] = len(bad[0]) - 2, 3
        new_keys = ([b"never seen" if i == 0 else v for i, v in enumerate(case.skeys[0][0])], case.skeys[0][1])
        block = [sv[0], tuple(bad)] if c else [tuple(bad), sv[1]]
        assert _code(lambda: t.update(kc, vc, string_keys=[GT.string_block(*new_keys, rng)], predicate=(capi.CMP_GT, 0), predicate_column=0,
                                      string_values=block)) == capi.ERR_INVALID_ARGUMENT
        same_as_before()
    # mismatched counts
    assert _code(lambda: t.update(kc, vc, string_keys=sk, string_values=sv[:1])) == capi.ERR_INVALID_ARGUMENT
    assert _code(lambda: t.update(kc, vc, string_keys=sk)) == capi.ERR_INVALID_ARGUMENT
    short = GT.string_block(case.svals[1][0][:-1], case.svals[1][1][:-1], rng)
    assert _code(lambda: t.update(kc, vc, string_keys=sk, string_values=[sv[0], short])) == capi.ERR_INVALID_ARGUMENT
    same_as_before()
    # the result with the wrong number of value outputs
    err = capi.Error()
    empty = (C.c_void_p * 1)()
    res = capi.GroupByMultiResult(0, 0, empty, empty, empty, empty, None, None)
    skeys = (capi.GroupByStringKeys * 1)()
    assert ctx.lib.ytgpu_groupby_table_result(ctx.handle, t.handle, C.byref(res), C.cast(skeys, C.c_void_p), 1, capi.MEM_HOST,
                                              C.byref(err)) == capi.ERR_INVALID_ARGUMENT
    # updates continue and give the full answer
    t.update(kc, vc, string_keys=sk, string_values=sv)
    assert (host(t.result()["count"]) == 2 * host(before["count"])).all()
    t.close()
    # create
    assert _code(lambda: ctx.groupby_table([T.Int64], 0, VALUE_TYPES, [(S, S0)], string_value_count=1)) == capi.ERR_UNSUPPORTED
    assert _code(lambda: ctx.groupby_table([T.Int64], 0, VALUE_TYPES, [(AVG, S0)], string_value_count=1)) == capi.ERR_UNSUPPORTED
    assert _code(lambda: ctx.groupby_table([T.Int64], 0, VALUE_TYPES, [(MN, S1)], string_value_count=1)) == capi.ERR_INVALID_ARGUMENT
    assert _code(lambda: ctx.groupby_table([T.Int64], 0, VALUE_TYPES, [(AMIN, 0, S1)], string_value_count=1)) == capi.ERR_INVALID_ARGUMENT
    assert _code(lambda: ctx.groupby_table([T.Int64], 0, VALUE_TYPES, [(MN, S0)])) == capi.ERR_UNSUPPORTED


@pytest.mark.gpu
@pytest.mark.parametrize("out_mem", [capi.MEM_HOST, capi.MEM_DEVICE])
def test_value_heap_capacity_protocol(ctx, out_mem):
    import torch
    rng = np.random.default_rng(14)
    n = 1000
    case = Case(rng, n, "numeric", groups=50)
    aggs = [(MX, S0), (CNT, S0), (FIRST, S1)]
    kc = [GT.column(tp, v, nl) for tp, (v, nl) in zip(case.numeric, case.nkeys)]
    vc = [GT.column(tp, v, nl) for tp, (v, nl) in zip(VALUE_TYPES, case.vals)]
    with ctx.groupby_table(case.numeric, 0, VALUE_TYPES, aggs, string_value_count=2) as t:
        t.update(kc, vc, string_values=[GT.string_block(*c, rng) for c in case.svals])
        full = t.result(out_mem=out_mem)
        g = len(host(full["count"]))
        hb = [len(host(h)) for h, _, _, _ in full["string_values"]]
        assert hb[0] > 0 and hb[1] > 0
        with pytest.raises(capi.YtGpuError) as e:  # the count query's answer, through a refused call
            t.result(capacity=g, heap_capacity=[hb[0] - 1, hb[1]], out_mem=out_mem)
        assert e.value.code == capi.ERR_INVALID_ARGUMENT and e.value.heap_bytes == hb and e.value.group_count == g
        # nothing written on a short value heap: the outputs keep their guard bytes
        guard = 0xA5

        def buf(nbytes):
            x = np.full(nbytes, guard, np.uint8)
            return torch.from_numpy(x).cuda() if out_mem == capi.MEM_DEVICE else x

        def ptr(x):
            return x.data_ptr() if torch.is_tensor(x) else x.ctypes.data

        nk, na = len(case.numeric), len(aggs)
        outs = [buf(g * 8) for _ in range(2 * nk + 2 * na + 2)]
        sv = [(buf(h + 8), buf(g * 8), buf(g * 4), buf(g)) for h in hb]
        arr = lambda xs: (C.c_void_p * len(xs))(*[ptr(x) for x in xs])  # noqa: E731
        res = capi.GroupByMultiResult(0, g, arr(outs[:nk]), arr(outs[nk:2 * nk]), arr(outs[2 * nk:2 * nk + na]),
                                      arr(outs[2 * nk + na:2 * nk + 2 * na]), ptr(outs[-2]), ptr(outs[-1]))
        for short in (0, 1):
            vs = (capi.GroupByStringKeys * 2)(*[capi.GroupByStringKeys(ptr(h), hb[j] - (j == short), 0, ptr(s), ptr(ln), ptr(nl))
                                                for j, (h, s, ln, nl) in enumerate(sv)])
            err = capi.Error()
            assert ctx.lib.ytgpu_groupby_table_result_strings(ctx.handle, t.handle, C.byref(res), None, 0, C.cast(vs, C.c_void_p), 2, out_mem,
                                                              C.byref(err)) == capi.ERR_INVALID_ARGUMENT
            assert [vs[j].heap_bytes for j in range(2)] == hb and res.group_count == g
            torch.cuda.synchronize()
            for x in outs + [y for s in sv for y in s]:
                assert (host(x).view(np.uint8) == guard).all()
        again = t.result(out_mem=out_mem)
        assert all((host(a) == host(b)).all() for a, b in zip(again["string_values"][0], full["string_values"][0]))


# ------------------------------------------------------------------------------------------------- no GPU
CTYPES = {"uint32_t": C.c_uint32, "uint64_t": C.c_uint64, "int": C.c_int, "int32_t": C.c_int32}


def _header_params(name):
    text = open(os.path.join(ROOT, "include", "ytgpu.h")).read()
    m = re.search(r"\bint\s+" + name + r"\(([^)]*)\);", text)
    assert m, name
    return [" ".join(p.split()) for p in m.group(1).split(",")]


@pytest.mark.parametrize("name", ["ytgpu_groupby_table_create_strings", "ytgpu_groupby_table_update_strings",
                                  "ytgpu_groupby_table_result_strings"])
def test_bindings_match_the_header(name):
    params = _header_params(name)
    lib = capi.load()
    assert name in capi.EXPORTED_SYMBOLS
    argtypes = getattr(lib, name).argtypes
    assert len(argtypes) == len(params), name
    for p, a in zip(params, argtypes):
        if "*" in p:
            assert a is C.c_void_p or issubclass(a, C._Pointer), (name, p, a)
        else:
            ctype = p.replace("const ", "").split()[0]
            assert a is CTYPES[ctype], (name, p, a)


@pytest.mark.gpu
def test_yql_block_combine_keys_string_values():
    """STRING values in the YQL adapter (host/gpu_block_combine_keys.cpp) against its std::map reference
    (host/tests/block_combine_keys_strings_ut.cpp)."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "block_combine_keys_strings_ut"], stdout=subprocess.DEVNULL)
    r = subprocess.run([os.path.join(ROOT, "host", "block_combine_keys_strings_ut")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
