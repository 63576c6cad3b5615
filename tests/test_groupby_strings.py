"""String-valued aggregates of the general GROUP BY (ytgpu_scan_filter_groupby_multi_strings).

YT QL defines min, max, first, argmin and argmax on strings (builtin_function_types.cpp:201-254; the string branches of
engine/udf/min.c and max.c: memcmp over the common length, then the shorter value first — Python's bytes order; argmin /
argmax in builtin_function_profiler.cpp:1442-1482 replace their state only on a strict comparison, so the first row that
attains the bound wins).  A string-valued result is the index of the row that holds it, and for MIN / MAX the smallest
such row.  `oracle_strings` runs the oracle's QL GROUP BY over the strings' ranks; `reference` restates the semantics row
at a time in Python, and the two must agree.  The GPU must agree with the oracle exactly: keys, counts, first rows, rows,
nulls."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import oracle
from oracle import AGG_ARGMAX, AGG_ARGMIN, AGG_AVG, AGG_COUNT, AGG_FIRST, AGG_MAX, AGG_MIN, AGG_SUM
from ytsaurus_b200.rowset import EValueType as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def reference(keys, key_nulls, columns, aggregates, filt=None):
    """QL GROUP BY, row at a time, first-seen order.  keys: lists of ints; key_nulls: lists of 0/1 or None;
    columns: lists of bytes / int / None (a string or an int64 column); aggregates: [(op, column[, by_column])].
    -> dict(keys, key_null, count, first_row, values, value_null); a string-valued result is a row index."""
    n = len(keys[0])
    key_nulls = [kn if kn is not None else [0] * n for kn in key_nulls]
    groups, order = {}, []
    for i in range(n):
        if filt is not None and not filt[i]:
            continue
        k = tuple(None if kn[i] else int(k[i]) for k, kn in zip(keys, key_nulls))
        st = groups.get(k)
        if st is None:
            st = groups[k] = dict(first=i, count=0, agg=[dict(row=None, best=None, n=0) for _ in aggregates])
            order.append(k)
        st["count"] += 1
        for a, s in zip(aggregates, st["agg"]):
            op, v = a[0], columns[a[1]][i]
            if v is None:
                continue
            if op in (AGG_SUM, AGG_AVG):  # scalar only: left to the oracle
                continue
            if op == AGG_COUNT:
                s["n"] += 1
            elif op == AGG_FIRST:
                if s["row"] is None:
                    s["row"] = i
            else:
                b = v if op in (AGG_MIN, AGG_MAX) else columns[a[2]][i]
                if b is None:
                    continue
                smaller = op in (AGG_MIN, AGG_ARGMIN)
                if s["row"] is None or (b < s["best"] if smaller else b > s["best"]):  # strict: the first row keeps a tie
                    s["row"], s["best"] = i, b
    out = dict(keys=[[0 if k[j] is None else k[j] for k in order] for j in range(len(keys))],
               key_null=[[int(k[j] is None) for k in order] for j in range(len(keys))],
               count=[groups[k]["count"] for k in order], first_row=[groups[k]["first"] for k in order], values=[], value_null=[])
    for ai, a in enumerate(aggregates):
        vals, nulls = [], []
        for k in order:
            s = groups[k]["agg"][ai]
            if a[0] == AGG_COUNT:
                vals.append(s["n"])
                nulls.append(0)
            elif s["row"] is None:
                vals.append(0)
                nulls.append(1)
            else:
                v = columns[a[1]][s["row"]]
                vals.append(s["row"] if isinstance(v, bytes) else v & 0xFFFFFFFFFFFFFFFF)
                nulls.append(0)
        out["values"].append(vals)
        out["value_null"].append(nulls)
    return out


MASK = 0xFFFFFFFFFFFFFFFF


def _is_string_column(column):
    return any(isinstance(x, bytes) for x in column)


def oracle_strings(keys, key_nulls, columns, aggregates, filt=None):
    """The oracle's QL GROUP BY (oracle.groupby_multi) over string columns, same arguments and result as `reference`.
    Every string column is replaced by the rank of its value among the column's distinct values in bytes order — memcmp
    over the common length, then the shorter first, the order of udf/min.c / max.c — so the oracle's own int64 MIN / MAX /
    ARGMIN / ARGMAX rules decide.  A string-valued result is selected as the row index (a column of row numbers with the
    string's NULLs): MIN / MAX of a string is ARGMIN / ARGMAX(row, rank), whose strict comparison keeps the smallest row
    that holds the bound; FIRST is FIRST(row); COUNT counts the ranks."""
    n = len(keys[0])
    vals, nulls, cache = [], [], {}

    def add(name, c, bits, nul):
        if (name, c) not in cache:
            vals.append(np.ascontiguousarray(bits, dtype=np.uint64))
            nulls.append(np.asarray(nul, dtype=np.uint8))
            cache[(name, c)] = len(vals) - 1
        return cache[(name, c)]

    def null_of(c):
        return [x is None for x in columns[c]]

    def plain(c):
        return add("plain", c, [0 if x is None else x & MASK for x in columns[c]], null_of(c))

    def rank(c):
        order = {v: r for r, v in enumerate(sorted({x for x in columns[c] if x is not None}))}
        return add("rank", c, [0 if x is None else order[x] for x in columns[c]], null_of(c))

    def row(c):
        return add("row", c, np.arange(n, dtype=np.uint64), null_of(c))

    def value(c):  # the returned argument: a string as its row, a scalar as itself
        return row(c) if _is_string_column(columns[c]) else plain(c)

    def bound(c):  # the compared argument
        return rank(c) if _is_string_column(columns[c]) else plain(c)
    aggs = []
    for op, c, *by in aggregates:
        if op in (AGG_MIN, AGG_MAX) and _is_string_column(columns[c]):
            aggs.append((AGG_ARGMIN if op == AGG_MIN else AGG_ARGMAX, row(c), rank(c)))
        elif op in (AGG_ARGMIN, AGG_ARGMAX):
            aggs.append((op, value(c), bound(by[0])))
        elif op == AGG_FIRST:
            aggs.append((op, value(c)))
        elif op == AGG_COUNT:
            aggs.append((op, bound(c)))
        else:
            aggs.append((op, plain(c)))
    kbits = [np.asarray([x & MASK for x in k], dtype=np.uint64) for k in keys]
    knull = [None if kn is None else np.asarray(kn, dtype=np.uint8) for kn in key_nulls]
    w = oracle.groupby_multi(kbits, knull, vals, nulls, [T.Int64] * len(vals), aggs,
                             filt=None if filt is None else np.asarray(filt, dtype=np.uint8))
    return dict(keys=[k.tolist() for k in w["keys"]], key_null=[k.tolist() for k in w["key_null"]], count=w["count"].tolist(),
                first_row=w["first_row"].tolist(), values=[v.tolist() for v in w["values"]],
                value_null=[v.tolist() for v in w["value_null"]])


def _plain_model(group_of_row, column, by, op):
    """Per group from whole lists, with Python's min / max: the smallest (value, row) pair (MAX: largest value, then smallest
    row)."""
    rows = {}
    for i, g in enumerate(group_of_row):
        rows.setdefault(g, []).append(i)
    res = {}
    for g, rs in rows.items():
        cand = [i for i in rs if column[i] is not None and (by is None or by[i] is not None)]
        key = (lambda i: column[i]) if by is None else (lambda i: by[i])
        if not cand:
            res[g] = None
        elif op in (AGG_MIN, AGG_ARGMIN):
            res[g] = min(cand, key=lambda i: (key(i), i))
        else:
            best = max(key(i) for i in cand)
            res[g] = min(i for i in cand if key(i) == best)
    return res


EDGE_WORDS = [b"", b"a", b"a\0", b"ab", b"\0", b"\0\0", b"\xff", b"abcdefg", b"abcdefgh", b"abcdefg\0", b"x" * 257 + b"a",
              b"x" * 257, b"x" * 300]


def _words(rng, count, max_len=40, prefix=b""):
    return [prefix + bytes(rng.integers(0, 256, int(rng.integers(0, max_len)), dtype=np.uint8)) for _ in range(count)]


def _random_strings(rng, n, words, null_p):
    return [None if rng.random() < null_p else words[int(rng.integers(0, len(words)))] for _ in range(n)]


def test_reference_edge_order_and_ties():
    col = [b"ab", b"a\0", b"a", None, b"", b"a", b"\xff", b"a\0"]
    ts = [1, 5, 5, 9, None, 1, 5, 0]
    r = reference([[0] * 8], [None], [col, ts], [(AGG_MIN, 0), (AGG_MAX, 0), (AGG_FIRST, 0), (AGG_COUNT, 0),
                                                 (AGG_ARGMAX, 0, 1), (AGG_ARGMIN, 1, 0), (AGG_ARGMIN, 0, 0)])
    assert r["values"] == [[4], [6], [0], [7], [1], [5], [4]]
    # "" is the smallest; "\xff" the largest (unsigned bytes); argmax(col, ts): rows 1, 2, 6 tie on 5 -> row 1;
    # argmin(ts, col): the min string "" has a NULL ts, so the next smallest with both arguments is "a" at row 2 -> ts 5
    # a group without values is NULL; COUNT is 0
    r = reference([[0, 1]], [None], [[b"a", None]], [(AGG_MAX, 0), (AGG_COUNT, 0), (AGG_FIRST, 0)])
    assert r["value_null"] == [[0, 1], [0, 0], [0, 1]] and r["values"][1] == [1, 0]


@pytest.mark.parametrize("seed", [1, 2])
def test_oracle_string_aggregates_agree_with_the_python_model(seed):
    """The oracle (through ranks) and the row-at-a-time model agree: two keys with NULLs, a filter, all six ops over two
    string columns and an int64 column, edge strings, 1000-byte shared prefixes, ties and groups without values."""
    rng = np.random.default_rng(seed)
    n = 30000
    words = EDGE_WORDS + _words(rng, 300) + _words(rng, 50, prefix=b"p" * 1000)
    s1 = _random_strings(rng, n, words, 0.1)
    s2 = _random_strings(rng, n, words[:25], 0.1)
    ts = [None if rng.random() < 0.1 else int(x) for x in rng.integers(-5, 5, n)]
    k0 = rng.integers(0, 150, n).tolist()
    k0n = (rng.random(n) < 0.02).astype(np.uint8).tolist()
    k1 = rng.integers(-2, 2, n).tolist()
    for i in range(40):  # groups without string values
        k0[i], k1[i], s1[i], s2[i] = 10**6 + i, 0, None, None
    filt = (rng.random(n) < 0.9).astype(np.uint8).tolist()
    aggs = ALL_OPS + [(AGG_FIRST, 2), (AGG_COUNT, 2), (AGG_ARGMIN, 1, 1), (AGG_SUM, 0), (AGG_MIN, 0)]
    cols = [ts, s1, s2]
    want = oracle_strings([k0, k1], [k0n, None], cols, aggs, filt=filt)
    got = reference([k0, k1], [k0n, None], cols, aggs, filt=filt)
    assert [[x & MASK for x in k] for k in got["keys"]] == want["keys"]
    for field in ("key_null", "count", "first_row"):
        assert got[field] == want[field], field
    for a in range(len(aggs)):
        if aggs[a][0] == AGG_SUM:
            continue
        assert got["value_null"][a] == want["value_null"][a], a
        assert got["values"][a] == want["values"][a], a


def test_reference_agrees_with_plain_model_and_oracle_grouping():
    rng = np.random.default_rng(5)
    n = 20000
    words = EDGE_WORDS + _words(rng, 300) + _words(rng, 50, prefix=b"p" * 1000)
    s = _random_strings(rng, n, words, 0.1)
    by = _random_strings(rng, n, words[:20], 0.1)  # many ties
    ts = [None if rng.random() < 0.1 else int(x) for x in rng.integers(-5, 5, n)]
    k = rng.integers(0, 200, n, dtype=np.uint64)
    k[:50] = 10**6 + np.arange(50)  # groups of one row
    s[:50] = [None] * 50  # ... without values
    aggs = [(AGG_MIN, 0), (AGG_MAX, 0), (AGG_ARGMIN, 0, 1), (AGG_ARGMAX, 0, 1), (AGG_ARGMAX, 0, 2), (AGG_ARGMIN, 2, 1)]
    r = reference([k.tolist()], [None], [s, by, ts], aggs)
    w = oracle.groupby_multi([k], None, [k], None, [T.Uint64], [(AGG_COUNT, 0)])
    assert r["keys"][0] == w["keys"][0].tolist() and r["count"] == w["count"].tolist() and r["first_row"] == w["first_row"].tolist()
    cols = [s, by, ts]
    for a, (op, c, *b) in enumerate(aggs):
        model = _plain_model(k.tolist(), cols[c], cols[b[0]] if b else None, op)
        for g, key in enumerate(r["keys"][0]):
            row = model[key]
            assert r["value_null"][a][g] == (row is None), (a, g)
            if row is not None:
                want = row if isinstance(cols[c][row], bytes) else cols[c][row] & 0xFFFFFFFFFFFFFFFF
                assert r["values"][a][g] == want, (a, g)


def test_new_symbol_is_declared_and_exported():
    from ytsaurus_b200 import capi
    assert "ytgpu_scan_filter_groupby_multi_strings" in capi.EXPORTED_SYMBOLS
    assert "ytgpu_scan_filter_groupby_multi_strings(" in open(os.path.join(ROOT, "include", "ytgpu.h")).read()
    assert capi.StringColumn.row_count.offset == 40 and ctypes.sizeof(capi.StringColumn) == 56  # the C struct's layout


def test_string_column_arguments_are_checked():
    from ytsaurus_b200.runtime import _string_column
    heap, starts, lengths, nulls = oracle.flatten_strings([b"a", None, b"bc"])
    c = _string_column(heap, starts, lengths, nulls)
    assert c.heap_bytes == heap.size and c.row_count == 3 and c.null_bytemap
    assert not _string_column(np.zeros(0, np.uint8), starts, lengths).null_bytemap
    for bad in ((heap.astype(np.uint16), starts, lengths, nulls), (heap, starts.astype(np.int32), lengths, nulls),
                (heap, starts, lengths.astype(np.uint64), nulls), (heap, starts.astype(np.float64), lengths, nulls),
                (heap, starts, lengths, nulls.astype(np.uint32)), (heap, starts[:2], lengths, nulls),
                (heap, starts.reshape(3, 1), lengths, nulls)):
        with pytest.raises(ValueError):
            _string_column(*bad)


def test_host_adapter_builds_and_refuses_cpu():
    import torch
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "aggregate_strings_ut"], stdout=subprocess.DEVNULL)
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([os.path.join(ROOT, "host", "aggregate_strings_ut")], capture_output=True, text=True, timeout=120)
    assert r.returncode == 100 and "no CPU fallback" in r.stderr


# ---------------------------------------------------------------------------------------------------------------- GPU
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
    a = np.ascontiguousarray(a)
    view = {np.dtype(np.uint64): np.int64, np.dtype(np.uint32): np.int32}.get(a.dtype)
    return torch.from_numpy(a.view(view) if view else a).cuda()


def _np(x, dtype):
    return np.asarray(x.cpu().numpy() if hasattr(x, "cpu") else x).view(dtype)


def _strings(values, device=False, pad=0):
    heap, starts, lengths, nulls = oracle.flatten_strings(values)
    if pad:  # every value at an odd offset
        heap = np.concatenate([np.zeros(pad, np.uint8), heap])
        starts = starts + pad
    arrs = (heap, starts, lengths, nulls)
    return tuple(_dev(a) for a in arrs) if device else arrs


def _col(vtype, bits, nulls=None, device=False):
    from ytsaurus_b200 import Column
    bits = np.ascontiguousarray(bits, dtype=np.uint64)
    bitmap = None if nulls is None else np.packbits(np.asarray(nulls, dtype=np.uint8), bitorder="little")
    if device:
        return Column(vtype, values=_dev(bits), null_bitmap=None if bitmap is None else _dev(bitmap))
    return Column(vtype, values=bits, null_bitmap=bitmap)


def _int_column(values):
    bits = np.asarray([0 if v is None else v for v in values], dtype=np.int64).view(np.uint64)
    return bits, np.asarray([v is None for v in values], dtype=np.uint8)


def _check(got, want):
    g = len(want["count"])
    assert len(got["count"]) == g
    for a, b in zip(got["keys"], want["keys"]):
        assert _np(a, np.uint64).tolist() == [x & 0xFFFFFFFFFFFFFFFF for x in b]
    for a, b in zip(got["key_null"], want["key_null"]):
        assert _np(a, np.uint8).tolist() == b
    assert _np(got["count"], np.uint64).tolist() == want["count"]
    assert _np(got["first_row"], np.uint64).tolist() == want["first_row"]
    for a in range(len(want["values"])):
        assert _np(got["value_null"][a], np.uint8).tolist() == want["value_null"][a], f"aggregate {a} nulls"
        assert _np(got["values"][a], np.uint64).tolist() == want["values"][a], f"aggregate {a}"


ALL_OPS = [(AGG_MIN, 1), (AGG_MAX, 1), (AGG_FIRST, 1), (AGG_COUNT, 1), (AGG_ARGMIN, 1, 0), (AGG_ARGMAX, 0, 2), (AGG_ARGMAX, 1, 2),
           (AGG_ARGMIN, 2, 1), (AGG_MAX, 2), (AGG_MIN, 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("nkeys", [1, 2, 3])
def test_gpu_all_ops_with_a_string_key(ctx, device, nkeys):
    rng = np.random.default_rng(nkeys * 10 + device)
    n = 40000
    words = EDGE_WORDS + _words(rng, 400) + _words(rng, 40, max_len=8)
    gkey = _random_strings(rng, n, _words(rng, 60, max_len=6) + [b"", b"a", b"a\0"], 0.02)
    s1 = _random_strings(rng, n, words, 0.15)
    s2 = _random_strings(rng, n, words[:30], 0.1)  # ties
    ts = [None if rng.random() < 0.1 else int(x) for x in rng.integers(-20, 20, n)]
    gh = _strings(gkey)
    ids, id_null = ctx.string_value_ids(*gh)
    keys, knulls = [ids.tolist()], [id_null.tolist()]
    kcols = [_col(T.Uint64, ids, id_null, device)]
    for extra in range(nkeys - 1):
        k = rng.integers(0, 3 + extra, n, dtype=np.int64)
        keys.append(k.tolist())
        knulls.append(None)
        kcols.append(_col(T.Int64, k.view(np.uint64), device=device))
    tsb, tsn = _int_column(ts)
    got = ctx.scan_filter_groupby_multi(kcols, [_col(T.Int64, tsb, tsn, device)], ALL_OPS,
                                        string_columns=[_strings(s1, device), _strings(s2, device)])
    want = oracle_strings(keys, knulls, [ts, s1, s2], ALL_OPS)
    _check(got, want)
    # the group key is the string at its id row
    for k, kn, f in zip(_np(got["keys"][0], np.uint64).tolist(), _np(got["key_null"][0], np.uint8).tolist(),
                        _np(got["first_row"], np.uint64).tolist()):
        assert kn == (gkey[f] is None) and (kn or gkey[k] == gkey[f])


@pytest.mark.gpu
def test_gpu_mixed_scalar_and_string_with_predicate(ctx):
    from ytsaurus_b200 import capi
    rng = np.random.default_rng(77)
    n = 60000
    k = rng.integers(0, 500, n, dtype=np.uint64)
    v = rng.integers(-1000, 1000, n, dtype=np.int64)
    vn = (rng.random(n) < 0.1).astype(np.uint8)
    s = _random_strings(rng, n, EDGE_WORDS + _words(rng, 500), 0.1)
    aggs = [(AGG_SUM, 0), (AGG_MAX, 1), (AGG_MIN, 0), (AGG_ARGMIN, 1, 0), (AGG_COUNT, 1), (AGG_AVG, 0), (AGG_FIRST, 1), (AGG_ARGMAX, 0, 1)]
    filt = ((v > -300) & (vn == 0)).astype(np.uint8)  # a NULL never passes the predicate
    got = ctx.scan_filter_groupby_multi([_col(T.Uint64, k)], [_col(T.Int64, v.view(np.uint64), vn)], aggs,
                                        predicate=(capi.CMP_GT, -300), predicate_column=0, string_columns=[_strings(s)])
    vals = [None if vn[i] else int(v[i]) for i in range(n)]
    _check(got, oracle_strings([k.tolist()], [None], [vals, s], aggs, filt=filt.tolist()))  # integer sums and averages are exact


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
def test_gpu_unaligned_heap_and_long_shared_prefixes(ctx, device):
    rng = np.random.default_rng(3)
    n = 20000
    prefix = bytes(rng.integers(0, 256, 1000, dtype=np.uint8))
    words = [prefix + w for w in _words(rng, 300, max_len=20)] + [prefix, prefix[:999], prefix + b"\0"]
    s = _random_strings(rng, n, words, 0.05)
    k = rng.integers(0, 50, n, dtype=np.uint64)
    ts = [int(x) for x in rng.integers(0, 3, n)]
    aggs = [(AGG_MIN, 1), (AGG_MAX, 1), (AGG_ARGMAX, 1, 0), (AGG_ARGMIN, 0, 1)]
    got = ctx.scan_filter_groupby_multi([_col(T.Uint64, k, device=device)], [_col(T.Int64, _int_column(ts)[0], device=device)], aggs,
                                        string_columns=[_strings(s, device, pad=3)])
    _check(got, oracle_strings([k.tolist()], [None], [ts, s], aggs))


def _decimal_strings(values, width):
    """Fixed-width zero-padded decimals as one heap: row order == numeric order."""
    digits = np.zeros((len(values), width), np.uint8)
    x = np.asarray(values, dtype=np.int64)
    for j in range(width - 1, -1, -1):
        digits[:, j] = 48 + x % 10
        x = x // 10
    return digits.reshape(-1), np.arange(len(values), dtype=np.uint64) * width, np.full(len(values), width, np.uint32), None


@pytest.mark.gpu
def test_gpu_one_group_heavy_contention(ctx):
    n = 10**7
    key = _col(T.Uint64, np.zeros(n, np.uint64), device=True)
    desc = tuple(_dev(a) if a is not None else None for a in _decimal_strings(np.arange(n - 1, -1, -1), 8))
    asc = tuple(_dev(a) if a is not None else None for a in _decimal_strings(np.arange(n), 8))
    got = ctx.scan_filter_groupby_multi([key], [], [(AGG_MIN, 0), (AGG_MAX, 1), (AGG_MAX, 0), (AGG_MIN, 1)],
                                        string_columns=[desc, asc], capacity=1)
    assert [int(_np(v, np.uint64)[0]) for v in got["values"]] == [n - 1, n - 1, 0, 0]
    assert all(int(_np(v, np.uint8)[0]) == 0 for v in got["value_null"])


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["sorted", "clustered", "million_groups"])
def test_gpu_key_shapes(ctx, shape):
    rng = np.random.default_rng(11)
    if shape == "million_groups":  # more groups than the shared-memory table
        n = 1_500_000
        k = rng.integers(0, 10**6, n, dtype=np.uint64)
    else:
        n = 1_000_000
        k = np.repeat(np.arange(n // 1000, dtype=np.uint64), 1000)  # runs of 1000 rows: whole warps in one group
        if shape == "clustered":
            k = k[np.argsort(rng.integers(0, 3, n) + np.arange(n) // 5000 * 8, kind="stable")]
    words = _words(rng, 3000, max_len=24, prefix=b"https://")
    s = _random_strings(rng, n, words, 0.05)
    ts = [int(x) for x in rng.integers(0, 100, n)]
    aggs = [(AGG_MIN, 1), (AGG_MAX, 1), (AGG_ARGMAX, 1, 0)]
    got = ctx.scan_filter_groupby_multi([_col(T.Uint64, k, device=True)], [_col(T.Int64, _int_column(ts)[0], device=True)], aggs,
                                        string_columns=[_strings(s, device=True)])
    _check(got, oracle_strings([k.tolist()], [None], [ts, s], aggs))


@pytest.mark.gpu
def test_gpu_capacity_protocol(ctx):
    from ytsaurus_b200 import capi
    s = [b"b", b"a", b"c", None]
    k = np.asarray([0, 1, 0, 2], np.uint64)
    with pytest.raises(capi.YtGpuError) as e:
        ctx.scan_filter_groupby_multi([_col(T.Uint64, k)], [], [(AGG_MIN, 0)], capacity=2, string_columns=[_strings(s)])
    assert e.value.code == capi.ERR_INVALID_ARGUMENT and "3 groups" in e.value.message
    got = ctx.scan_filter_groupby_multi([_col(T.Uint64, k)], [], [(AGG_MIN, 0), (AGG_MAX, 0)], capacity=3, string_columns=[_strings(s)])
    assert got["values"][0].tolist() == [0, 1, 0] and got["values"][1].tolist() == [2, 1, 0]
    assert got["value_null"][0].tolist() == [0, 0, 1]


@pytest.mark.gpu
def test_gpu_errors(ctx):
    from ytsaurus_b200 import capi
    k = _col(T.Uint64, np.asarray([0, 1, 0], np.uint64))
    v = _col(T.Int64, np.asarray([1, 2, 3], np.uint64))
    s = _strings([b"a", b"bb", None])

    def code(aggs, strings=(s,), **kw):
        with pytest.raises(capi.YtGpuError) as e:
            ctx.scan_filter_groupby_multi([k], [v], aggs, string_columns=list(strings), **kw)
        return e.value.code
    assert code([(AGG_SUM, 1)]) == capi.ERR_UNSUPPORTED
    assert code([(AGG_AVG, 1)]) == capi.ERR_UNSUPPORTED
    assert code([(AGG_MIN, 2)]) == capi.ERR_INVALID_ARGUMENT  # column out of range
    assert code([(AGG_ARGMIN, 1, 2)]) == capi.ERR_INVALID_ARGUMENT
    assert code([(AGG_MIN, 1)], predicate=(capi.CMP_GT, 0), predicate_column=1) == capi.ERR_INVALID_ARGUMENT  # a string predicate column
    assert code([(AGG_MIN, 1)], strings=[_strings([b"a", b"b"])]) == capi.ERR_INVALID_ARGUMENT  # row-count mismatch
    heap, starts, lengths, nulls = s
    bad = starts.copy()
    bad[1] = heap.size - 1  # "bb" runs one byte past the heap
    assert code([(AGG_COUNT, 1)], strings=[(heap, bad, lengths, nulls)]) == capi.ERR_INVALID_ARGUMENT
    assert code([(AGG_MAX, 1)], strings=[(heap, np.asarray([0, 2**63, 0], np.uint64), lengths, nulls)]) == capi.ERR_INVALID_ARGUMENT
    # the context stays usable, and a NULL row's start / length are ignored
    got = ctx.scan_filter_groupby_multi([k], [v], [(AGG_MAX, 1)], string_columns=[(heap, starts, lengths, np.asarray([0, 1, 0], np.uint8))])
    assert got["values"][0].tolist() == [0, 0] and got["value_null"][0].tolist() == [0, 1]


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
def test_gpu_empty_heap_and_flavour_checks(ctx, device, monkeypatch):
    """All values "" or NULL: the heap may be empty (a null pointer with heap_bytes = 0); it is never read."""
    import torch
    from ytsaurus_b200 import capi, runtime
    n = 1000
    k = np.arange(n, dtype=np.uint64) % 3
    nulls = (np.arange(n) % 5 == 0).astype(np.uint8)
    starts, lengths = np.zeros(n, np.uint64), np.zeros(n, np.uint32)
    heap = torch.empty(0, dtype=torch.uint8, device="cuda") if device else np.zeros(0, np.uint8)
    col = (heap, _dev(starts), _dev(lengths), _dev(nulls)) if device else (heap, starts, lengths, nulls)
    aggs = [(AGG_MIN, 0), (AGG_MAX, 0), (AGG_COUNT, 0), (AGG_FIRST, 0)]
    got = ctx.scan_filter_groupby_multi([_col(T.Uint64, k, device=device)], [], aggs, string_columns=[col])
    values = [None if z else b"" for z in nulls.tolist()]
    _check(got, oracle_strings([k.tolist()], [None], [values], aggs))
    if device:
        with pytest.raises(ValueError):  # one flavour per string column
            ctx.scan_filter_groupby_multi([_col(T.Uint64, k, device=True)], [], aggs, string_columns=[(heap, starts, _dev(lengths), None)])
    make = runtime._string_column

    def bad_mem(*a):
        c = make(*a)
        c.mem = 7
        return c
    monkeypatch.setattr(runtime, "_string_column", bad_mem)
    with pytest.raises(capi.YtGpuError) as e:
        ctx.scan_filter_groupby_multi([_col(T.Uint64, k, device=device)], [], aggs, string_columns=[col])
    assert e.value.code == capi.ERR_INVALID_ARGUMENT


class _ViaStrings:
    """The library with ytgpu_scan_filter_groupby_multi routed to the new entry point with string_count = 0."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def ytgpu_scan_filter_groupby_multi(self, *args):
        *head, err = args
        return self._lib.ytgpu_scan_filter_groupby_multi_strings(*head, None, 0, err)


@pytest.mark.gpu
def test_gpu_new_entry_point_without_strings_matches_the_old_one(ctx):
    from ytsaurus_b200 import capi
    rng = np.random.default_rng(1000 + 7)
    n = 100003
    k0 = rng.integers(0, 333, n, dtype=np.uint64)
    k1 = rng.integers(0, 3, n, dtype=np.int64)
    v_i = rng.integers(-2**62, 2**62, n, dtype=np.int64)
    v_d = rng.standard_normal(n) * 1e3
    small = rng.integers(0, 50, n, dtype=np.int64)
    aggs = [(AGG_SUM, 0), (AGG_SUM, 1), (AGG_MIN, 0), (AGG_MAX, 1), (AGG_COUNT, 0), (AGG_AVG, 0), (AGG_ARGMIN, 1, 2),
            (AGG_ARGMAX, 0, 2), (AGG_FIRST, 1)]
    cols = ([_col(T.Uint64, k0), _col(T.Int64, k1.view(np.uint64))],
            [_col(T.Int64, v_i.view(np.uint64)), _col(T.Double, v_d.view(np.uint64)), _col(T.Int64, small.view(np.uint64))])
    old = ctx.scan_filter_groupby_multi(*cols, aggs, group_count_hint=1000)
    lib = ctx.lib
    ctx.lib = _ViaStrings(lib)
    try:
        new = ctx.scan_filter_groupby_multi(*cols, aggs, group_count_hint=1000)
        with pytest.raises(capi.YtGpuError) as e:
            ctx.scan_filter_groupby_multi(*cols, [(AGG_SUM, 3)])
        assert e.value.code == capi.ERR_INVALID_ARGUMENT
    finally:
        ctx.lib = lib
    for key in ("count", "first_row"):
        assert new[key].tolist() == old[key].tolist()
    for key in ("keys", "key_null", "value_null"):
        assert [x.tolist() for x in new[key]] == [x.tolist() for x in old[key]]
    for a in range(len(aggs)):
        if a == 1:  # a double sum: atomics add in arbitrary order
            assert np.allclose(new["values"][a].view(np.float64), old["values"][a].view(np.float64), rtol=1e-12, atol=0)
        else:
            assert new["values"][a].tolist() == old["values"][a].tolist()


@pytest.mark.gpu
def test_gpu_host_adapter_over_strings():
    exe = os.path.join(ROOT, "host", "aggregate_strings_ut")
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "aggregate_strings_ut"], stdout=subprocess.DEVNULL)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
