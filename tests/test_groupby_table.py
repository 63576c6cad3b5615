"""GROUP BY tables (ytgpu_groupby_table_*): blocks folded one by one must give exactly what the one-shot GROUP BY gives over
the concatenated blocks, with each block's predicate on its own rows.  The reference is the one-shot call for numeric
keys and a plain dict GROUP BY for string keys."""
import ctypes as C
import importlib.util
import os
import subprocess
import tempfile
import zlib

import numpy as np
import pytest

from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import EValueType as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name):
    spec = importlib.util.spec_from_file_location("_groupby_table_" + name[:-3], os.path.join(os.path.dirname(os.path.abspath(__file__)), name))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


J = _load("test_join_table.py")  # make_column(), ENCODINGS, DOMAINS, _dbits
M = J.M

S, MN, MX, CNT, AVG, AMIN, AMAX, FIRST = (capi.AGG_SUM, capi.AGG_MIN, capi.AGG_MAX, capi.AGG_COUNT, capi.AGG_AVG, capi.AGG_ARGMIN,
                                          capi.AGG_ARGMAX, capi.AGG_FIRST)
# value columns: 0 int64, 1 uint64, 2 double, 3 boolean; the predicate reads column 0
VALUE_TYPES = [T.Int64, T.Uint64, T.Double, T.Boolean]
AGGREGATES = ([(op, c) for op in (S, AVG) for c in (0, 1, 2)] + [(op, c) for op in (MN, MX, CNT, FIRST) for c in (0, 1, 2, 3)]
              + [(op, c, b) for op in (AMIN, AMAX) for c, b in ((1, 0), (0, 2), (2, 3))])


def test_string_keys_struct_matches_the_header():
    prog = '#include <stdio.h>\n#include "include/ytgpu.h"\nint main(void) { printf("%zu\\n", sizeof(ytgpu_groupby_string_keys)); return 0; }\n'
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "abi.c"), os.path.join(d, "abi")
        open(src, "w").write(prog)
        subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", ROOT, src, "-o", exe])
        assert int(subprocess.check_output([exe], text=True)) == C.sizeof(capi.GroupByStringKeys) == 48


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
def values(rng, n, null_rate=0.1):
    """The four value columns' (values, nulls)."""
    specials = np.asarray([J._dbits(x) for x in (0.0, -0.0, 1.5, -2.5, float("inf"), float("-inf"))] + [0x7FF8000000000000], np.uint64)
    dbl = rng.normal(0, 100, n).view(np.uint64).copy()
    pick = rng.random(n) < 0.2
    dbl[pick] = specials[rng.integers(0, len(specials), int(pick.sum()))]
    cols = [rng.integers(-50, 50, n).astype(np.int64).view(np.uint64), rng.integers(0, 2**64 - 1, n, dtype=np.uint64, endpoint=True), dbl,
            rng.integers(0, 2, n).astype(np.uint64)]
    return [(v, rng.random(n) < null_rate) for v in cols]


def column(vtype, vals, nulls, kind="bitmap", rng=None):
    col, real = J.make_column(kind, vtype, vals, nulls, rng or np.random.default_rng(0))
    return col


def pass_mask(block_vals, pred):
    if pred is None:
        return np.ones(len(block_vals[0][0]), bool)
    op, c = pred
    v, nl = block_vals[0]
    x = v.view(np.int64)
    m = {capi.CMP_GT: x > c, capi.CMP_LT: x < c, capi.CMP_GE: x >= c}[op]
    return m & ~nl


def one_shot(ctx, key_types, keys, vals, aggregates, passes):
    """The one-shot call over whole columns, with the per-row pass flags as a fifth value column and its predicate."""
    kc = [column(t, v, nl) for t, (v, nl) in zip(key_types, keys)]
    vc = [column(t, v, nl) for t, (v, nl) in zip(VALUE_TYPES, vals)]
    vc.append(column(T.Uint64, passes.astype(np.uint64), np.zeros(len(passes), bool), "plain"))
    return ctx.scan_filter_groupby_multi(kc, vc, aggregates, predicate=(capi.CMP_EQ, 1), predicate_column=len(vc) - 1)


def feed(table, key_types, keys, vals, bounds, preds, kinds=("bitmap",), rng=None, device=False):
    """Updates over the rows [bounds[i], bounds[i + 1]) with preds[i] -> the pass flags of every row."""
    rng = rng or np.random.default_rng(1)
    passes = []
    for i in range(len(bounds) - 1):
        a, b = bounds[i], bounds[i + 1]
        bk = [(v[a:b], nl[a:b]) for v, nl in keys]
        bv = [(v[a:b], nl[a:b]) for v, nl in vals]
        kc = [column(t, v, nl, kinds[(k + i) % len(kinds)], rng) for k, (t, (v, nl)) in enumerate(zip(key_types, bk))]
        vc = [column(t, v, nl, "bitmap", rng) for t, (v, nl) in zip(VALUE_TYPES, bv)]
        if device:
            for c in kc + vc:
                M.to_device(c)
        pred = preds[i]
        table.update(kc, vc, predicate=pred, predicate_column=0 if pred else -1)
        passes.append(pass_mask(bv, pred))
    return np.concatenate(passes) if passes else np.zeros(0, bool)


def host(x):
    import torch
    return x.cpu().numpy() if torch.is_tensor(x) else np.asarray(x)


def assert_same(got, ref, aggregates):
    g = len(host(ref["count"]))
    assert len(host(got["count"])) == g
    for k in range(len(ref["keys"])):
        kn = host(ref["key_null"][k]).astype(bool)
        assert (host(got["key_null"][k]).astype(bool) == kn).all()
        assert (host(got["keys"][k]).view(np.uint64)[~kn] == host(ref["keys"][k]).view(np.uint64)[~kn]).all()
    assert (host(got["count"]).view(np.uint64) == host(ref["count"]).view(np.uint64)).all()
    assert (host(got["first_row"]).view(np.uint64) == host(ref["first_row"]).view(np.uint64)).all()
    for a, agg in enumerate(aggregates):
        vn = host(ref["value_null"][a]).astype(bool)
        assert (host(got["value_null"][a]).astype(bool) == vn).all(), agg
        gv, rv = host(got["values"][a]).view(np.uint64)[~vn], host(ref["values"][a]).view(np.uint64)[~vn]
        if agg[0] in (S, AVG) and VALUE_TYPES[agg[1]] == T.Double:
            x, y = gv.view(np.float64), rv.view(np.float64)
            assert np.allclose(x, y, rtol=1e-9, atol=1e-6, equal_nan=True), agg
        else:
            assert (gv == rv).all(), agg


def splits(n, how, rng):
    if how == "one":
        return [0, n]
    if how == "equal":
        return list(range(0, n, n // 4)) + [n] if n % 4 else list(range(0, n + 1, n // 4))
    cuts = sorted(set([0, n] + rng.integers(0, n, 6).tolist()))
    out = [0]
    for c in cuts[1:]:  # blocks of 0 and 1 rows too
        out += [out[-1], out[-1] + 1, c] if c > out[-1] + 1 else [c]
    return out


def keys_for(rng, key_types, n, groups, kinds=("plain",)):
    dom = {t: np.asarray(J.DOMAINS[t], np.uint64) for t in J.DOMAINS}
    out = []
    for k, t in enumerate(key_types):
        if t == T.Int64 and k == 0:
            v = rng.integers(0, groups, n).astype(np.uint64)
        else:
            v = dom[t][rng.integers(0, len(dom[t]), n)]
        out.append((v, rng.random(n) < 0.05))
    return out


# ------------------------------------------------------------------------------------------------- numeric keys
SHAPES = {"int64": [T.Int64], "two": [T.Int64, T.Double], "eight": [T.Int64, T.Uint64, T.Double, T.Boolean] * 2}


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["int64", "two"])
@pytest.mark.parametrize("how", ["one", "equal", "random"])
@pytest.mark.parametrize("pred", [None, (capi.CMP_GT, -10)])
def test_numeric_blocks_match_one_shot(ctx, shape, how, pred):
    rng = np.random.default_rng(zlib.crc32(f"{shape}{how}{pred}".encode()))
    key_types = SHAPES[shape]
    n = 4000
    keys = keys_for(rng, key_types, n, 300)
    vals = values(rng, n)
    bounds = splits(n, how, rng)
    with ctx.groupby_table(key_types, 0, VALUE_TYPES, AGGREGATES) as t:
        passes = feed(t, key_types, keys, vals, bounds, [pred] * (len(bounds) - 1), ("bitmap", "dict"), rng)
        got = t.result()
    assert_same(got, one_shot(ctx, key_types, keys, vals, AGGREGATES, passes), AGGREGATES)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
def test_eight_keys_every_encoding(ctx, device):
    rng = np.random.default_rng(8)
    key_types = SHAPES["eight"]
    n, per = 3000, 500
    keys = keys_for(rng, key_types, n, 40)
    vals = values(rng, n)
    real = [(v.copy(), nl.copy()) for v, nl in keys]
    aggs = [(S, 0), (FIRST, 2), (AMIN, 1, 2)]
    with ctx.groupby_table(key_types, 0, VALUE_TYPES, aggs) as t:
        for i, a in enumerate(range(0, n, per)):
            kc = []
            for k, tp in enumerate(key_types):
                kind = J.ENCODINGS[(k + i) % len(J.ENCODINGS)]
                col, nulls = J.make_column(kind, tp, keys[k][0][a:a + per], keys[k][1][a:a + per], rng)
                real[k][1][a:a + per] = nulls
                kc.append(col)
            vc = [column(tp, v[a:a + per], nl[a:a + per]) for tp, (v, nl) in zip(VALUE_TYPES, vals)]
            if device:
                for c in kc + vc:
                    M.to_device(c)
            t.update(kc, vc)
        got = t.result(out_mem=capi.MEM_DEVICE if device else capi.MEM_HOST)
    real = [(np.where(nl, 0, v).astype(np.uint64), nl) for v, nl in real]
    assert_same(got, one_shot(ctx, key_types, real, vals, aggs, np.ones(n, bool)), aggs)


@pytest.mark.gpu
def test_per_block_predicates_and_a_block_with_no_passing_row(ctx):
    rng = np.random.default_rng(3)
    n = 6000
    keys = keys_for(rng, [T.Int64], n, 500)
    vals = values(rng, n)
    bounds = [0, 1000, 2000, 3000, 6000]
    preds = [(capi.CMP_GT, 0), (capi.CMP_GT, 1000), None, (capi.CMP_LT, 10)]  # block 2: no row passes
    with ctx.groupby_table([T.Int64], 0, VALUE_TYPES, AGGREGATES) as t:
        passes = feed(t, [T.Int64], keys, vals, bounds, preds)
        assert not passes[1000:2000].any()
        assert_same(t.result(), one_shot(ctx, [T.Int64], keys, vals, AGGREGATES, passes), AGGREGATES)


@pytest.mark.gpu
def test_growth_past_shared_memory_and_capacity_mid_stream(ctx):
    rng = np.random.default_rng(4)
    small, big = 20000, 60000
    k1 = rng.integers(0, 1000, small)
    k2 = rng.integers(0, 30000, big)  # pushes past 4096 groups and past the initial capacity
    keys = [(np.concatenate([k1, k2]).astype(np.uint64), np.zeros(small + big, bool))]
    vals = values(rng, small + big)
    bounds = [0, 5000, 10000, 20000, 30000, 50000, 80000]
    with ctx.groupby_table([T.Int64], 0, VALUE_TYPES, AGGREGATES, hint=100) as t:
        passes = feed(t, [T.Int64], keys, vals, bounds, [None] * 6)
        assert_same(t.result(), one_shot(ctx, [T.Int64], keys, vals, AGGREGATES, passes), AGGREGATES)


@pytest.mark.gpu
def test_result_midway_then_more_updates(ctx):
    rng = np.random.default_rng(5)
    n = 8000
    keys = keys_for(rng, [T.Int64, T.Double], n, 700)
    vals = values(rng, n)
    with ctx.groupby_table([T.Int64, T.Double], 0, VALUE_TYPES, AGGREGATES) as t:
        p1 = feed(t, [T.Int64, T.Double], keys, vals, [0, 2000, 3000], [None, None])
        cut = [(v[:3000], nl[:3000]) for v, nl in keys], [(v[:3000], nl[:3000]) for v, nl in vals]
        assert_same(t.result(), one_shot(ctx, [T.Int64, T.Double], cut[0], cut[1], AGGREGATES, p1), AGGREGATES)
        tail_keys = [(v[3000:], nl[3000:]) for v, nl in keys]
        tail_vals = [(v[3000:], nl[3000:]) for v, nl in vals]
        p2 = feed(t, [T.Int64, T.Double], tail_keys, tail_vals, [0, 5000], [None])
        assert_same(t.result(), one_shot(ctx, [T.Int64, T.Double], keys, vals, AGGREGATES, np.concatenate([p1, p2])), AGGREGATES)


@pytest.mark.gpu
def test_cross_block_selection(ctx):
    """FIRST NULL in early blocks; ARGMIN reached in block 1, tied in block 2 (block 1 wins), strictly improved in block 3
    (block 3's first attaining row wins); a key seen only as NULL until a late block; MIN / MAX with NaN and +-0."""
    d = J._dbits
    key = np.asarray([7, 7, 8, 7, 7, 8, 7, 7, 7, 0], np.uint64)
    knull = np.asarray([0, 0, 1, 0, 0, 1, 0, 0, 0, 0], bool)
    by = np.asarray([5, 3, 1, 9, 3, 1, 2, 4, 2, 0], np.uint64).view(np.int64).astype(np.uint64)
    ret = np.arange(10, dtype=np.uint64) + 100
    first_nulls = np.asarray([1, 1, 1, 1, 0, 1, 0, 0, 0, 0], bool)
    dbl = np.asarray([d(0.0), d(-0.0), d(1.0), d(float("nan")), d(-0.0), d(2.0), d(0.0), d(-1.0), d(float("nan")), d(3.0)], np.uint64)
    vals = [(by, np.zeros(10, bool)), (ret, np.zeros(10, bool)), (dbl, first_nulls), (np.ones(10, np.uint64), np.zeros(10, bool))]
    keys = [(key, knull)]
    aggs = [(AMIN, 1, 0), (AMAX, 1, 0), (FIRST, 2), (MN, 2), (MX, 2)]
    with ctx.groupby_table([T.Int64], 0, VALUE_TYPES, aggs) as t:
        passes = feed(t, [T.Int64], keys, vals, [0, 3, 6, 10], [None] * 3)
        got = t.result()
    ref = one_shot(ctx, [T.Int64], keys, vals, aggs, passes)
    assert_same(got, ref, aggs)
    # group 7: ARGMIN by 3 at row 1 (tied at row 4), then 2 at row 6 -> 106; FIRST: the first non-NULL double, row 4's -0.0
    g7 = list(host(got["keys"][0])).index(7)
    assert host(got["values"][0])[g7] == 106 and host(got["values"][2])[g7] == d(-0.0)


# ------------------------------------------------------------------------------------------------- string keys
def strings_for(rng, n, distinct, extra=()):
    pool = [bytes(rng.integers(0, 256, rng.integers(0, 301), dtype=np.uint8)) for _ in range(distinct)]
    pool += [b"", b"\x00", b"a\x00b", bytes([0x80, 0xff]), *extra]
    idx = rng.integers(0, len(pool), n)
    vals = [pool[i] for i in idx]
    nulls = rng.random(n) < 0.05
    return vals, nulls


def string_block(vals, nulls, rng, device=False):
    """(heap, starts, lengths, nulls) with the values in shuffled heap order."""
    order = rng.permutation(len(vals))
    heap = bytearray(b"\xee" * 3)
    starts = np.zeros(len(vals), np.uint64)
    for i in order:
        starts[i] = len(heap)
        heap += vals[i]
    cols = (np.frombuffer(bytes(heap), np.uint8).copy(), starts, np.asarray([len(v) for v in vals], np.uint32),
            nulls.astype(np.uint8))
    if device:
        import torch
        cols = tuple(torch.from_numpy(c.view({1: np.uint8, 4: np.int32, 8: np.int64}[c.dtype.itemsize])).cuda() for c in cols)
    return cols


def dict_groupby(key_rows, vals, passes, aggs):
    groups = {}
    for i, k in enumerate(key_rows):
        if not passes[i]:
            continue
        g = groups.setdefault(k, dict(first=i, count=0, sum=0, nn=0, min=None))
        g["count"] += 1
        v, nl = vals[0][0][i], vals[0][1][i]
        if not nl:
            g["sum"] = (g["sum"] + int(v)) % 2**64
            g["nn"] += 1
            x = int(np.uint64(v).view(np.int64))
            g["min"] = x if g["min"] is None else min(g["min"], x)
    return sorted(groups.items(), key=lambda kv: kv[1]["first"])


def got_string(res, s, o):
    heap, starts, lengths, nulls = (host(x) for x in res["string_keys"][s])
    if nulls[o]:
        return None
    return bytes(heap[int(starts[o]):int(starts[o]) + int(lengths[o])])


STRING_SHAPES = {"one": ([], 1), "int64_string": ([T.Int64], 1), "double_bool_two": ([T.Double, T.Boolean], 2)}


@pytest.mark.gpu
@pytest.mark.parametrize("shape", list(STRING_SHAPES))
@pytest.mark.parametrize("device", [False, True])
def test_string_keys_match_a_dict_group_by(ctx, shape, device):
    rng = np.random.default_rng(len(shape) + 10 * device)
    numeric, nstr = STRING_SHAPES[shape]
    n = 5000
    nkeys = keys_for(rng, numeric, n, 50) if numeric else []
    if numeric and numeric[0] == T.Int64:
        nkeys[0] = (nkeys[0][0] % 20, nkeys[0][1])
    skeys = [strings_for(rng, n, 40 + 200 * s, extra=(bytes(65536),) if s == 0 else ()) for s in range(nstr)]
    late = skeys[0][0][7]  # a key seen only as NULL until the last block
    skeys[0][1][:2500] |= np.asarray([v == late for v in skeys[0][0][:2500]])
    vals = values(rng, n)
    aggs = [(S, 0), (CNT, 0), (MN, 0)]
    bounds = [0, 1, 1, 700, 2500, 5000]  # the dictionary grows across blocks
    pred = (capi.CMP_GT, -40)
    with ctx.groupby_table(numeric, nstr, VALUE_TYPES, aggs) as t:
        passes = []
        for i in range(len(bounds) - 1):
            a, b = bounds[i], bounds[i + 1]
            kc = [column(tp, v[a:b], nl[a:b]) for tp, (v, nl) in zip(numeric, nkeys)]
            vc = [column(tp, v[a:b], nl[a:b]) for tp, (v, nl) in zip(VALUE_TYPES, vals)]
            if device:
                for c in kc + vc:
                    M.to_device(c)
            sk = [string_block(sv[a:b], sn[a:b], rng, device) for sv, sn in skeys]
            t.update(kc, vc, string_keys=sk, predicate=pred, predicate_column=0)
            passes.append(pass_mask([(v[a:b], nl[a:b]) for v, nl in vals], pred))
        got = t.result(out_mem=capi.MEM_DEVICE if device else capi.MEM_HOST)
    passes = np.concatenate(passes)
    rows = []
    for i in range(n):
        k = tuple(None if nl[i] else int(v[i]) for v, nl in nkeys) + tuple(None if sn[i] else sv[i] for sv, sn in skeys)
        rows.append(k)
    ref = dict_groupby(rows, vals, passes, aggs)
    assert len(host(got["count"])) == len(ref)
    for o, (k, g) in enumerate(ref):
        numk = tuple(None if host(got["key_null"][c])[o] else int(host(got["keys"][c]).view(np.uint64)[o]) for c in range(len(numeric)))
        assert numk + tuple(got_string(got, s, o) for s in range(nstr)) == k
        assert int(host(got["first_row"])[o]) == g["first"] and int(host(got["count"])[o]) == g["count"]
        assert int(host(got["values"][1])[o]) == g["nn"]
        if g["nn"]:
            assert int(host(got["values"][0]).view(np.uint64)[o]) == g["sum"]
            assert int(host(got["values"][2]).view(np.int64)[o]) == g["min"]
        else:
            assert host(got["value_null"][0])[o] and host(got["value_null"][2])[o]


@pytest.mark.gpu
def test_capacity_protocol(ctx):
    rng = np.random.default_rng(6)
    n = 1000
    sv, sn = strings_for(rng, n, 30)
    vals = values(rng, n)
    with ctx.groupby_table([], 1, VALUE_TYPES, [(S, 0)]) as t:
        assert t.result(count_only=True) == 0
        t.update([], [column(tp, v, nl) for tp, (v, nl) in zip(VALUE_TYPES, vals)], string_keys=[string_block(sv, sn, rng)])
        g = t.result(count_only=True)
        full = t.result()
        hb = len(full["string_keys"][0][0])
        with pytest.raises(capi.YtGpuError) as e:
            t.result(capacity=g - 1, heap_capacity=[hb])
        assert e.value.code == capi.ERR_INVALID_ARGUMENT and e.value.group_count == g and e.value.heap_bytes == [hb]
        if hb:
            with pytest.raises(capi.YtGpuError) as e:
                t.result(capacity=g, heap_capacity=[hb - 1])
            assert e.value.code == capi.ERR_INVALID_ARGUMENT and e.value.heap_bytes == [hb]
        again = t.result()
        assert (host(again["count"]) == host(full["count"])).all()


# ------------------------------------------------------------------------------------------------- refusals
def _code(fn):
    with pytest.raises(capi.YtGpuError) as e:
        fn()
    return e.value.code


@pytest.mark.gpu
def test_refusals_leave_the_table_as_it_was(ctx):
    from ytsaurus_b200 import Column, GpuContext
    rng = np.random.default_rng(7)
    n = 500
    keys = keys_for(rng, [T.Int64], n, 40)
    vals = values(rng, n)
    sv, sn = strings_for(rng, n, 20)
    vc = [column(tp, v, nl) for tp, (v, nl) in zip(VALUE_TYPES, vals)]
    kc = [column(T.Int64, *keys[0])]
    t = ctx.groupby_table([T.Int64], 1, VALUE_TYPES, [(S, 0), (AMIN, 1, 2)])
    t.update(kc, vc, string_keys=[string_block(sv, sn, rng)])
    before = t.result()
    bad_heap = list(string_block(sv, sn, rng))
    bad_heap[1] = bad_heap[1].copy()
    bad_heap[1][n // 2] = len(bad_heap[0]) - 1
    bad_heap[2] = bad_heap[2].copy()
    bad_heap[2][n // 2] = 5
    bad_heap[3] = np.zeros(n, np.uint8)
    huge = Column(T.Int64, values=np.zeros(4, np.uint64), value_count=(1 << 30) + 1)
    other = GpuContext(0)
    refusals = [
        (capi.ERR_INVALID_ARGUMENT, lambda: t.update([], vc, string_keys=[string_block(sv, sn, rng)])),
        (capi.ERR_INVALID_ARGUMENT, lambda: t.update(kc, vc[:3], string_keys=[string_block(sv, sn, rng)])),
        (capi.ERR_INVALID_ARGUMENT, lambda: t.update([column(T.Uint64, *keys[0])], vc, string_keys=[string_block(sv, sn, rng)])),
        (capi.ERR_INVALID_ARGUMENT, lambda: t.update(kc, vc[:1] + [column(T.Int64, *vals[1])] + vc[2:], string_keys=[string_block(sv, sn, rng)])),
        (capi.ERR_INVALID_ARGUMENT, lambda: t.update(kc, vc)),
        (capi.ERR_INVALID_ARGUMENT, lambda: t.update(kc, vc, string_keys=[tuple(bad_heap)])),
    ]
    for want, fn in refusals:
        assert _code(fn) == want
        after = t.result()
        for k in ("count", "first_row"):
            assert (host(after[k]) == host(before[k])).all()
        assert all((host(a) == host(b)).all() for a, b in zip(after["values"], before["values"]))
    # a table of another context
    lib, err = ctx.lib, capi.Error()
    karr = (capi.ColumnView * 1)(kc[0].view())
    assert lib.ytgpu_groupby_table_update(other.handle, t.handle, C.cast(karr, C.c_void_p), 1, None, 0, None, 0, None, -1,
                                          C.byref(err)) == capi.ERR_INVALID_ARGUMENT
    assert lib.ytgpu_groupby_table_destroy(None, C.byref(err)) == capi.OK
    other.close()
    # updates still work and give the full answer
    t.update(kc, vc, string_keys=[string_block(sv, sn, rng)])
    assert (host(t.result()["count"]) == 2 * host(before["count"])).all()
    assert _code(lambda: ctx.groupby_table([T.Int64], 0, VALUE_TYPES, [(MN, 4)])) == capi.ERR_UNSUPPORTED
    t.close()
    with ctx.groupby_table([T.Int64], 0, VALUE_TYPES, [(S, 0)]) as t2:  # a view over 2^30 rows, refused from the view alone
        t2.update(kc, vc)
        assert _code(lambda: t2.update([huge], [Column(tp, values=np.zeros(4, np.uint64), value_count=(1 << 30) + 1)
                                                for tp in VALUE_TYPES])) == capi.ERR_UNSUPPORTED
        t2.update(kc, vc)
        assert host(t2.result()["count"]).sum() == 2 * n


@pytest.mark.gpu
def test_large_blocks_against_one_shot(ctx):
    import torch
    n, block = 10**7, 1 << 20
    g = torch.Generator(device="cuda").manual_seed(9)
    key = torch.randint(0, 10**6, (n,), device="cuda", generator=g, dtype=torch.int64)
    v = torch.randint(-1000, 1000, (n,), device="cuda", generator=g, dtype=torch.int64)
    dv = torch.randn(n, device="cuda", generator=g, dtype=torch.float64).view(torch.int64)
    from ytsaurus_b200 import Column
    aggs = [(S, 0), (CNT, 0), (MN, 0), (AVG, 1), (AMAX, 0, 1), (FIRST, 1)]
    with ctx.groupby_table([T.Int64], 0, [T.Int64, T.Double], aggs) as t:
        for a in range(0, n, block):
            b = min(n, a + block)
            t.update([Column(T.Int64, values=key[a:b].contiguous())],
                     [Column(T.Int64, values=v[a:b].contiguous()), Column(T.Double, values=dv[a:b].contiguous())])
        got = t.result()
    ref = ctx.scan_filter_groupby_multi([Column(T.Int64, values=key)], [Column(T.Int64, values=v), Column(T.Double, values=dv)], aggs)
    assert len(got["count"]) == len(host(ref["count"])) > 900000
    for k in ("count", "first_row"):
        assert (host(got[k]).view(np.uint64) == host(ref[k]).view(np.uint64)).all()
    assert (host(got["keys"][0]).view(np.uint64) == host(ref["keys"][0]).view(np.uint64)).all()
    for a, agg in enumerate(aggs):
        x, y = host(got["values"][a]).view(np.uint64), host(ref["values"][a]).view(np.uint64)
        if agg[0] == AVG:
            assert np.allclose(x.view(np.float64), y.view(np.float64), rtol=1e-9)
        else:
            assert (x == y).all(), agg


@pytest.mark.gpu
def test_yql_block_combine_keys_adapter():
    """The YQL adapter (host/gpu_block_combine_keys.cpp) against its std::map reference (host/tests/block_combine_keys_ut.cpp)."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "block_combine_keys_ut"], stdout=subprocess.DEVNULL)
    r = subprocess.run([os.path.join(ROOT, "host", "block_combine_keys_ut")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
