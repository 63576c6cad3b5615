"""ORDER BY ... OFFSET ... LIMIT on the GPU (ytgpu_order_rows in csrc/capi_sort.cu) against a Python model of the order, and
the QL evaluator's ORDER BY / LIMIT / OFFSET clauses and queries without GROUP BY (host/tests/order_ut.cpp).

The model restates the header's rules: items compared in turn; NULL below every value; false below true; a NaN above +inf
and all NaNs equal; -0.0 equal to +0.0; strings as unsigned bytes, a prefix first; `descending` reverses one item, NULLs
included; ties keep their order in `rows`.  compare_model() is that rule written out value by value; order_model() is the
same order through stable numpy lexsort keys, fast enough for 10^7 rows.  The CPU tests pin compare_model() with
hand-written cases, check that both models agree with each other and with the oracle's stable sort_rows, and every GPU
result is compared with order_model() for exact equality."""
import copy
import functools
import importlib.util
import os
import struct
import subprocess
import tempfile

import numpy as np
import pytest

from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import VALUE_DTYPE
from ytsaurus_b200.rowset import EValueType as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name):
    """A sibling test module's helpers, loaded by path so no import mode matters."""
    spec = importlib.util.spec_from_file_location("_order_" + name[:-3], os.path.join(os.path.dirname(os.path.abspath(__file__)), name))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


M = _load("test_groupby_kernel_matrix.py")  # encode(), to_device(), _bm()

TYPES = [T.Int64, T.Uint64, T.Double, T.Boolean]
# every encoding encode() builds, a 32-bit plain vector, a boolean bitmap, an Arrow validity bitmap and has_values = 0
ENCODINGS = ["plain", "base", "bitmap", "dict", "rle", "packed", "width32", "boolbits", "arrow", "novalues"]
NULLABLE = ("bitmap", "dict", "rle", "arrow")


def _dbits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


NAN_A, NAN_B, NAN_NEG = 0x7FF8000000000000, 0x7FF0000000000123, 0xFFF8000000000001
DOMAINS = {
    T.Int64: [2**63, 2**64 - 1, 0, 1, 7, 2**63 - 1, 12345, 2**62 + 5],  # INT64_MIN, -1, 0, ..., INT64_MAX
    T.Uint64: [0, 1, 5, 2**63, 2**64 - 1, 99, 2**40],
    T.Double: [_dbits(0.0), _dbits(-0.0), _dbits(1.5), _dbits(-2.25), NAN_A, NAN_B, NAN_NEG, _dbits(float("inf")),
               _dbits(float("-inf")), 1, 0x8000000000000001],  # the last two: subnormals
    T.Boolean: [0, 1],
}


# ------------------------------------------------------------------------------------------------- models
def _is_nan(bits):
    return (bits & 0x7FF0000000000000) == 0x7FF0000000000000 and (bits & 0x000FFFFFFFFFFFFF) != 0


def order_key(vtype, bits):
    """A non-NULL value -> an unsigned integer whose order is the value order (strings: the bytes themselves)."""
    if vtype == "string":
        return bits
    bits = int(bits)
    if vtype == T.Int64:
        return bits ^ (1 << 63)
    if vtype == T.Boolean:
        return int(bits != 0)
    if vtype == T.Double:
        if _is_nan(bits):
            return 1 << 64  # above every double, all NaNs equal
        if bits & ((1 << 63) - 1) == 0:
            bits = 0  # -0.0 == +0.0
        return (~bits) & ((1 << 64) - 1) if bits >> 63 else bits | (1 << 63)
    return bits


def compare_model(items, a, b):
    """items: [(vtype or "string", values, nulls, descending)]; a, b row indexes -> -1 / 0 / 1."""
    for vtype, values, nulls, desc in items:
        na, nb = bool(nulls[a]), bool(nulls[b])
        if na or nb:
            c = (not na) - (not nb)
        else:
            x, y = order_key(vtype, values[a]), order_key(vtype, values[b])
            c = (x > y) - (x < y)
        if desc:
            c = -c
        if c:
            return c
    return 0


def order_slow(items, rows, offset=0, limit=None):
    """The stable order by compare_model of `rows` -> the window's row indexes."""
    s = sorted(rows, key=functools.cmp_to_key(lambda a, b: compare_model(items, a, b)))
    limit = len(s) if limit is None else limit
    return np.asarray(s[offset:offset + limit], np.uint32)


def _rank_strings(values, nulls):
    present = sorted({v for v, nl in zip(values, nulls) if not nl})
    rank = {v: i for i, v in enumerate(present)}
    return np.asarray([0 if nl else rank[v] for v, nl in zip(values, nulls)], np.uint64)


def _sortable(vtype, values, nulls):
    """Item values -> uint64 words in the value order (NULLs handled by the caller)."""
    if vtype == "string":
        return _rank_strings(values, nulls)
    v = np.asarray(values, np.uint64)
    if vtype == T.Int64:
        return v ^ np.uint64(1 << 63)
    if vtype == T.Boolean:
        return (v != 0).astype(np.uint64)
    if vtype == T.Double:
        nan = ((v & np.uint64(0x7FF0000000000000)) == np.uint64(0x7FF0000000000000)) & ((v & np.uint64(0x000FFFFFFFFFFFFF)) != 0)
        v = np.where((v & np.uint64((1 << 63) - 1)) == 0, np.uint64(0), v)
        neg = (v >> np.uint64(63)) != 0
        k = np.where(neg, ~v, v | np.uint64(1 << 63))
        return np.where(nan, np.uint64(2**64 - 1), k)  # +inf maps below 2^64 - 1
    return v


def order_model(items, rows=None, offset=0, limit=None):
    """order_slow through numpy: one stable lexsort of `rows` (None: every row) -> the window's row indexes."""
    n = len(items[0][2])
    rows = np.arange(n, dtype=np.uint32) if rows is None else np.asarray(rows, np.uint32)
    keys = []
    for vtype, values, nulls, desc in items:
        nl = np.asarray(nulls, bool)
        k = _sortable(vtype, values, nl)
        present = (~nl).astype(np.uint8)
        if desc:
            k, present = ~k, (1 - present).astype(np.uint8)
        keys += [present[rows], np.where(nl, np.uint64(0), k)[rows]]
    order = np.lexsort(keys[::-1]) if keys else np.arange(len(rows))
    limit = len(rows) if limit is None else limit
    return rows[order][offset:offset + limit]


# ------------------------------------------------------------------------------------------------- CPU tests
def test_model_pins_hand_written_cases():
    def order(vtype, vals, desc=False):
        nulls = [v is None for v in vals]
        values = [0 if v is None else v for v in vals] if vtype != "string" else [b"" if v is None else v for v in vals]
        items = [(vtype, values, nulls, desc)]
        slow = order_slow(items, list(range(len(vals)))).tolist()
        assert order_model(items).tolist() == slow
        return slow
    # INT64_MIN, -1, 0, INT64_MAX, NULL
    assert order(T.Int64, [2**63 - 1, 2**64 - 1, 0, None, 2**63]) == [3, 4, 1, 2, 0]
    assert order(T.Int64, [2**63 - 1, 2**64 - 1, 0, None, 2**63], desc=True) == [0, 2, 1, 4, 3]
    # UINT64_MAX and 2^63 are the largest unsigned values
    assert order(T.Uint64, [2**64 - 1, 2**63, 0, 1, None]) == [4, 2, 3, 1, 0]
    # -inf < -2.25 < -subnormal < -0.0 == +0.0 < subnormal < +inf < NaNs (all equal, any payload or sign)
    d = [NAN_B, _dbits(float("inf")), _dbits(-0.0), _dbits(0.0), 0x8000000000000001, 1, NAN_NEG, _dbits(float("-inf")),
         _dbits(-2.25), NAN_A, None]
    assert order(T.Double, d) == [10, 7, 8, 4, 2, 3, 5, 1, 0, 6, 9]
    assert order(T.Double, d, desc=True) == [0, 6, 9, 1, 5, 2, 3, 4, 8, 7, 10]
    assert order(T.Boolean, [1, 0, None, 1, 0]) == [2, 1, 4, 0, 3]
    # "" < "\0" < "a" < "ab" < "ab\0" < "b" < "\x80" < "\xff"; NULL first, last when descending
    s = [b"\xff", b"ab\x00", b"", None, b"a", b"\x00", b"ab", b"\x80", b"b"]
    assert order("string", s) == [3, 2, 5, 4, 6, 1, 8, 7, 0]
    assert order("string", s, desc=True) == [0, 7, 8, 1, 6, 4, 5, 2, 3]
    # two items: the second breaks ties of the first; equal rows keep their order
    items = [(T.Int64, [1, 1, 0, 1], [False, False, False, True], False), ("string", [b"b", b"a", b"z", b"a"], [False] * 4, True)]
    assert order_slow(items, [0, 1, 2, 3]).tolist() == [3, 2, 0, 1]
    assert order_model(items, [1, 0, 3, 2], offset=1, limit=2).tolist() == [2, 0]


def _random_items(rng, n, specs):
    items = []
    for vtype, desc in specs:
        nulls = rng.random(n) < 0.15
        if vtype == "string":
            pool = [b"", b"\x00", b"a", b"ab", b"abc", b"ab\x00", b"\xff", b"\x80z", b"zz"]
            values = [pool[i] for i in rng.integers(0, len(pool), n)]
        else:
            dom = np.asarray(DOMAINS[vtype], np.uint64)
            values = dom[rng.integers(0, len(dom), n)]
        items.append((vtype, values, nulls, desc))
    return items


def _oracle_rowset(items):
    """The items as an unversioned rowset for the oracle: one value per item, strings in one heap."""
    n = len(items[0][2])
    rows = np.zeros((n, len(items)), VALUE_DTYPE)
    heap = bytearray()
    for k, (vtype, values, nulls, _) in enumerate(items):
        for i in range(n):
            v = rows[i, k]
            v["id"] = k
            if nulls[i]:
                v["type"] = T.Null
            elif vtype == "string":
                v["type"], v["length"], v["data"] = T.String, len(values[i]), len(heap)
                heap += values[i]
            else:
                v["type"], v["data"] = vtype, (int(values[i]) != 0) if vtype == T.Boolean else int(values[i])
    return rows, np.frombuffer(bytes(heap) or b"\x00", np.uint8).copy()


@pytest.mark.parametrize("seed", range(6))
def test_models_agree_with_each_other_and_the_oracle(seed):
    import oracle
    rng = np.random.default_rng(seed)
    n = 400
    specs = [(TYPES[(seed + k) % 4] if k % 3 else "string", bool((seed >> k) & 1)) for k in range(1 + seed % 4)]
    items = _random_items(rng, n, specs)
    rows = rng.permutation(n)[: n - 37].astype(np.uint32)
    fast = order_model(items, rows, 5, 300)
    assert fast.tolist() == order_slow(items, rows.tolist(), 5, 300).tolist()
    values, heap = _oracle_rowset(items)
    perm, _ = oracle.sort_rows(values, heap, len(items), [d for _, d in specs], oracle.SORT_STABLE)
    assert order_model(items).tolist() == perm.tolist()


HEADER_PROGRAM = r"""
#include <stdio.h>
#include "include/ytgpu.h"
int main(void) {
    ytgpu_order_item item = {3, 1, 1, 0};
    printf("%u %u %u %u %u\n", (unsigned)sizeof(ytgpu_order_item), item.column, item.is_string, item.descending, item.reserved);
    return 0;
}
"""


def test_header_compiles_as_c99_with_the_order_call():
    import ctypes
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "o.c"), os.path.join(d, "o")
        open(src, "w").write(HEADER_PROGRAM)
        subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", ROOT, src, "-o", exe])
        out = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    assert out == [ctypes.sizeof(capi.OrderItem), 3, 1, 1, 0] and out[0] == 8
    assert "ytgpu_order_rows" in capi.EXPORTED_SYMBOLS


def test_host_adapter_builds_and_refuses_cpu():
    import torch
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "order_ut"], stdout=subprocess.DEVNULL)
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([os.path.join(ROOT, "host", "order_ut")], capture_output=True, text=True, timeout=120)
    assert r.returncode == 100 and "no CPU fallback" in r.stderr


# ------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def ctx():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from ytsaurus_b200 import GpuContext
    c = GpuContext(0)
    yield c
    c.close()


def make_column(kind, vtype, values, nulls, rng, start):
    """A Column of `kind` whose rows [start, start + n) decode to `values` (NULL where nulls) -> (Column, its real nulls)."""
    from ytsaurus_b200 import Column
    n = len(values)
    values = np.asarray(values, np.uint64)
    if kind == "novalues":
        return Column(vtype, values=None, value_count=n, null_bitmap=M._bm(np.zeros(n, bool))), np.ones(n, bool)
    if kind == "arrow":
        pad = np.zeros(start, bool)
        return Column(vtype, values=np.r_[np.zeros(start, np.uint64), values], null_bitmap=M._bm(np.r_[pad, ~nulls]), arrow_validity=True,
                      start_index=start, value_count=n), nulls
    if kind == "width32":
        return Column(vtype, values=np.r_[np.full(start, 7, np.uint32), values.astype(np.uint32)], bit_width=32, start_index=start,
                      value_count=n), np.zeros(n, bool)
    if kind == "boolbits":
        bits = np.r_[np.ones(start, bool), values != 0]
        return Column(vtype, values=M._bm(bits), bit_width=1, start_index=start, value_count=n), np.zeros(n, bool)
    if kind not in NULLABLE:
        nulls = np.zeros(n, bool)
    return M.encode(kind, vtype, values, nulls if kind in NULLABLE else None, start, rng), nulls


def _values_for(kind, vtype, rng, n):
    if kind == "width32":
        return rng.integers(0, 2**32, n, dtype=np.uint64) % np.uint64(1000)
    if kind == "boolbits":
        return rng.integers(0, 2, n).astype(np.uint64)
    dom = np.asarray(DOMAINS[vtype], np.uint64)
    return dom[rng.integers(0, len(dom), n)]


def on_host(x):
    import torch
    if torch.is_tensor(x):
        x = x.cpu().numpy()
    return np.asarray(x).view(np.uint32)


def to_dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view({1: np.uint8, 4: np.int32, 8: np.int64}[a.dtype.itemsize])).cuda()


def string_column(values, nulls, device=False, pad=b""):
    """Flat string column arrays (heap, starts, lengths, nulls) of `values`, the heap starting with `pad`."""
    heap = bytearray(pad)
    starts, lengths = [], []
    for v, nl in zip(values, nulls):
        starts.append(len(heap))
        lengths.append(0 if nl else len(v))
        if not nl:
            heap += v
    arrays = (np.frombuffer(bytes(heap) or b"\x00", np.uint8).copy(), np.asarray(starts, np.uint64), np.asarray(lengths, np.uint32),
              np.asarray(nulls, np.uint8))
    return tuple(to_dev(a) for a in arrays) if device else arrays


@pytest.mark.gpu
@pytest.mark.parametrize("desc", [False, True], ids=["asc", "desc"])
@pytest.mark.parametrize("start", [0, 1, 3])
@pytest.mark.parametrize("kind", ENCODINGS)
def test_gpu_item_types_and_encodings(ctx, kind, start, desc):
    rng = np.random.default_rng(ENCODINGS.index(kind) * 10 + start)
    n = 3000
    for vtype in TYPES:
        if kind == "boolbits" and vtype != T.Boolean:
            continue
        values = _values_for(kind, vtype, rng, n)
        col, nulls = make_column(kind, vtype, values, rng.random(n) < 0.2, rng, start)
        items = [(vtype, values, nulls, desc)]
        for device in (False, True):
            c = M.to_device(copy.copy(col)) if device else col
            got = ctx.order_rows([c], items=[(0, False, desc)])
            np.testing.assert_array_equal(on_host(got), order_model(items))


@pytest.mark.gpu
@pytest.mark.parametrize("count", [1, 2, 3, 5, 8, 32])
def test_gpu_mixed_items(ctx, count):
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(100 + count)
    n = 5000
    cols, scols, items, model = [], [], [], []
    for k in range(count):
        desc = bool(rng.integers(0, 2))
        if k % 4 == 3:
            vals = [[b"", b"a", b"ab", b"b\x00", b"\xfe"][i] for i in rng.integers(0, 5, n)]
            nulls = rng.random(n) < 0.1
            scols.append(string_column(vals, nulls, pad=bytes([k]) * k))
            items.append((len(scols) - 1, True, desc))
            model.append(("string", vals, nulls, desc))
        else:
            vtype = TYPES[k % 4]
            dom = np.asarray(DOMAINS[vtype], np.uint64)
            vals = dom[rng.integers(0, min(3, len(dom)), n)]  # few values: long tie runs
            nulls = rng.random(n) < 0.1
            cols.append(Column(vtype, values=vals, null_bitmap=M._bm(nulls)))
            items.append((len(cols) - 1, False, desc))
            model.append((vtype, vals, nulls, desc))
    rows = rng.permutation(n)[:4000].astype(np.uint32)
    got = ctx.order_rows(cols, scols, items, rows=rows, offset=17, limit=3000)
    np.testing.assert_array_equal(on_host(got), order_model(model, rows, 17, 3000))


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_string_columns_with_separate_heaps(ctx, device):
    rng = np.random.default_rng(7)
    n = 20000
    pools = [[b"http://a.com/" + bytes([65 + i]) * (i % 7) for i in range(20)], [b"", b"\x00", b"x", b"xy", b"\xff\xff"],
             [bytes([i]) for i in range(256)]]
    scols, model = [], []
    for k, pool in enumerate(pools):
        vals = [pool[i] for i in rng.integers(0, len(pool), n)]
        nulls = rng.random(n) < 0.05
        scols.append(string_column(vals, nulls, device, pad=b"#" * (k * 5 + 1)))
        model.append(("string", vals, nulls, k == 1))
    got = ctx.order_rows([], scols, [(0, True, False), (1, True, True), (2, True, False)])
    np.testing.assert_array_equal(on_host(got), order_model(model))


@pytest.mark.gpu
def test_gpu_long_string_keys_take_the_refinement_rounds(ctx):
    rng = np.random.default_rng(9)
    n = 6000
    stems = [b"q" * 300, b"q" * 299 + b"r", b"q" * 400, b"p" * 310]
    vals = [stems[i] + bytes([j % 3]) for i, j in zip(rng.integers(0, 4, n), rng.integers(0, 3, n))]
    nulls = rng.random(n) < 0.05
    model = [("string", vals, nulls, False), (T.Int64, rng.integers(0, 3, n).astype(np.uint64), np.zeros(n, bool), True)]
    from ytsaurus_b200 import Column
    got = ctx.order_rows([Column(T.Int64, values=model[1][1])], [string_column(vals, nulls)], [(0, True, False), (0, False, True)])
    np.testing.assert_array_equal(on_host(got), order_model(model))
    assert ctx.get_option("last_sort_refine_rounds") > 0


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_stability_and_row_lists(ctx, device):
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(11)
    n = 5000
    equal = Column(T.Double, values=np.full(n, _dbits(-0.0), np.uint64))
    vals = np.where(rng.random(n) < 0.5, np.uint64(_dbits(0.0)), np.uint64(_dbits(-0.0)))
    zeros = Column(T.Double, values=vals)
    subset = rng.permutation(n)[:1234].astype(np.uint32)
    descending = np.sort(subset)[::-1].copy()
    r = (lambda a: to_dev(a)) if device else (lambda a: a)
    c1, c2 = (M.to_device(copy.copy(c)) for c in (equal, zeros)) if device else (equal, zeros)
    # all keys equal (-0.0 == +0.0): the order of `rows`, whatever it is
    np.testing.assert_array_equal(on_host(ctx.order_rows([c1], items=[(0, False, True)])), np.arange(n))
    np.testing.assert_array_equal(on_host(ctx.order_rows([c2], items=[(0, False, False)], rows=r(subset))), subset)
    np.testing.assert_array_equal(on_host(ctx.order_rows([c2], items=[(0, False, True)], rows=r(descending))), descending)
    keys = Column(T.Int64, values=rng.integers(0, 4, n).astype(np.uint64))
    model = [(T.Int64, keys.values, np.zeros(n, bool), True)]
    kc = M.to_device(copy.copy(keys)) if device else keys
    np.testing.assert_array_equal(on_host(ctx.order_rows([kc], items=[(0, False, True)], rows=r(descending), offset=3, limit=900)),
                                  order_model(model, descending, 3, 900))


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_offset_and_limit_edges(ctx, device):
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(13)
    n = 777
    vals = rng.integers(0, 50, n).astype(np.uint64)
    col = Column(T.Uint64, values=vals)
    if device:
        col = M.to_device(col)
    model = [(T.Uint64, vals, np.zeros(n, bool), False)]
    for offset in (0, 1, n - 1, n, n + 5):
        for limit in (0, 1, n - 1, n, n + 5):
            got = ctx.order_rows([col], items=[(0, False, False)], offset=offset, limit=limit)
            want = order_model(model, None, offset, limit)
            np.testing.assert_array_equal(on_host(got), want)
            assert ctx.order_rows([col], items=[(0, False, False)], offset=offset, limit=limit, count_only=True) == len(want)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 4097, 1 << 18, (1 << 18) + 12345, 10**7])
def test_gpu_sizes(ctx, n):
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(n % 1000)
    a = rng.integers(0, 2**64 - 1, n, dtype=np.uint64, endpoint=True)
    anull = rng.random(n) < 0.01
    model = [(T.Int64, a, anull, True)]
    cols = [Column(T.Int64, values=a, null_bitmap=M._bm(anull))]
    items = [(0, False, True)]
    if n <= 1 << 19:  # a second item with long ties where the sizes allow the model's time
        b = rng.integers(0, 3, n).astype(np.uint64)
        a2 = (a % np.uint64(5)).astype(np.uint64)
        model = [(T.Uint64, a2, np.zeros(n, bool), False), (T.Double, b, np.zeros(n, bool), True)]
        cols = [Column(T.Uint64, values=a2), Column(T.Double, values=b)]
        items = [(0, False, False), (1, False, True)]
    dcols = [M.to_device(copy.copy(c)) for c in cols]
    limit = min(n, 100000)
    got = ctx.order_rows(dcols, items=items, offset=n // 3, limit=limit, out_mem=capi.MEM_DEVICE)
    np.testing.assert_array_equal(on_host(got), order_model(model, None, n // 3, limit))


def _code(fn):
    with pytest.raises(capi.YtGpuError) as e:
        fn()
    return e.value.code


@pytest.mark.gpu
def test_gpu_refusals(ctx):
    from ytsaurus_b200 import Column
    n = 100
    col = Column(T.Int64, values=np.arange(n, dtype=np.uint64))
    short = Column(T.Int64, values=np.arange(n - 1, dtype=np.uint64))
    heap, starts, lengths, nulls = string_column([b"ab"] * n, np.zeros(n, bool))
    inv, uns = capi.ERR_INVALID_ARGUMENT, capi.ERR_UNSUPPORTED
    one = [(0, False, False)]
    assert _code(lambda: ctx.order_rows([col], items=[])) == inv
    assert _code(lambda: ctx.order_rows([col] * 33, items=[(i, False, False) for i in range(33)])) == inv
    assert _code(lambda: ctx.order_rows([col], items=[(1, False, False)])) == inv                     # a missing column
    assert _code(lambda: ctx.order_rows([col], [(heap, starts, lengths, nulls)], items=[(1, True, False)])) == inv
    assert _code(lambda: ctx.order_rows([col, short], items=[(0, False, False), (1, False, False)])) == inv  # lengths differ
    assert _code(lambda: ctx.order_rows([col], [(heap, starts[:50], lengths[:50], nulls[:50])], items=[(0, False, False), (0, True, False)])) == inv
    assert _code(lambda: ctx.order_rows([Column(T.String, values=np.zeros(n, np.uint64))], items=one)) == uns
    assert _code(lambda: ctx.order_rows([Column(0x11, values=np.zeros(n, np.uint64))], items=one)) == uns
    bad_rows = np.arange(10, dtype=np.uint32)
    bad_rows[4] = n  # a row index past the columns: checked on the device
    assert _code(lambda: ctx.order_rows([col], items=one, rows=bad_rows)) == inv
    assert _code(lambda: ctx.order_rows([M.to_device(copy.copy(col))], items=one, rows=to_dev(bad_rows))) == inv
    assert _code(lambda: ctx.order_rows([col], items=one, row_count=n + 1)) == inv                 # no rows: past the columns
    bad_start = starts.copy()
    bad_start[7] = len(heap)  # "ab" past the end of its heap
    assert _code(lambda: ctx.order_rows([], [(heap, bad_start, lengths, nulls)], items=[(0, True, False)])) == inv
    # the radix sort's 2^30 bound, refused before any access: the row list pointer is never read
    # (called directly: the wrapper would size an output of 2^30 entries)
    import ctypes as C
    iarr = (capi.OrderItem * 1)(capi.OrderItem(0, 0, 0, 0))
    view = (capi.ColumnView * 1)(col.view())
    cnt, err = C.c_uint64(0), capi.Error()
    one_row = np.zeros(1, np.uint32)
    out = np.zeros(1, np.uint32)
    assert ctx.lib.ytgpu_order_rows(ctx.handle, C.cast(view, C.c_void_p), 1, None, 0, iarr, 1, one_row.ctypes.data, capi.ORDER_MAX_ROWS, 0, 1,
                                    out.ctypes.data, C.byref(cnt), capi.MEM_HOST, C.byref(err)) == uns
    # a non-zero reserved field
    iarr[0].reserved = 1
    assert ctx.lib.ytgpu_order_rows(ctx.handle, C.cast(view, C.c_void_p), 1, None, 0, iarr, 1, None, n, 0, n, None, C.byref(cnt), capi.MEM_HOST,
                                    C.byref(err)) == inv
    # a null out_count
    iarr[0].reserved = 0
    assert ctx.lib.ytgpu_order_rows(ctx.handle, C.cast(view, C.c_void_p), 1, None, 0, iarr, 1, None, n, 0, n, None, None, capi.MEM_HOST,
                                    C.byref(err)) == inv


@pytest.mark.gpu
def test_gpu_materialisation_is_timed_as_key_extraction(ctx):
    """The sort's key normalisation is timed as key extraction too: the call records exactly one launch of that class more
    than ytgpu_sort_rowset over the rowset it materialises, with the same key spec."""
    from ytsaurus_b200 import Column
    n = 100000
    vals = np.arange(n, dtype=np.uint64)[::-1].copy()
    rowset = np.zeros((n, 1), VALUE_DTYPE)
    rowset["type"], rowset["data"] = T.Int64, vals[:, None]
    ctx.enable_timers(True)
    ctx.reset_timers()
    ctx.sort_rowset(rowset, np.zeros(1, np.uint8), [(0, 0, T.Int64, 0, 0)])
    _, sort_launches = ctx.kernel_ms(capi.KC_EXTRACT)
    ctx.reset_timers()
    got = ctx.order_rows([Column(T.Int64, values=vals)], items=[(0, False, False)], limit=10)
    ms, launches = ctx.kernel_ms(capi.KC_EXTRACT)
    ctx.enable_timers(False)
    np.testing.assert_array_equal(on_host(got), np.arange(n - 1, n - 11, -1))
    assert sort_launches > 0 and launches == sort_launches + 1 and ms > 0


@pytest.mark.gpu
def test_gpu_host_adapter_order_clauses(ctx):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "order_ut"], stdout=subprocess.DEVNULL)
    r = subprocess.run([os.path.join(ROOT, "host", "order_ut")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    assert "order_ut: 0 failure(s)" in r.stdout
