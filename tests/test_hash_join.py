"""Hash JOIN on the GPU (csrc/join.cu): ytgpu_hash_join, ytgpu_gather_column and ytgpu_gather_string_column against a plain
Python dict join, and the QL evaluator's JOIN clause (host/tests/join_ut.cpp).

The reference builds a dict from each foreign key tuple to its foreign rows in ascending order, then walks the primary rows
in order: one pair per foreign row of the row's tuple, or (row, JOIN_NO_ROW) for a LEFT join's unmatched row.  A tuple is
(None or the 64-bit payload) per column, so NULL equals NULL and doubles compare by bit pattern, as the header states.
Both index arrays are compared for exact equality.

hj_probe_kernel<DIRECT, NK> compiles six ways: DIRECT when every key column of both sides is a plain 64-bit vector without
base / zig-zag, NK = 1, 2, else 0 (3..8 key columns).  PROBE_CASES names the input that reaches each, as ASSIGN_CASES of
test_groupby_kernel_matrix.py does for the build step."""
import copy
import importlib.util
import os
import struct
import subprocess
import tempfile

import numpy as np
import pytest

from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import EValueType as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_ROW = capi.JOIN_NO_ROW


def _load(name):
    """A sibling test module's helpers, loaded by path so no import mode matters."""
    spec = importlib.util.spec_from_file_location("_join_" + name[:-3], os.path.join(os.path.dirname(os.path.abspath(__file__)), name))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


M = _load("test_groupby_kernel_matrix.py")  # encode(), to_device(), _bm()

TYPES = [T.Int64, T.Uint64, T.Double, T.Boolean]
# (DIRECT, key column count)
PROBE_CASES = [(True, 1), (True, 2), (True, 3), (True, 8), (False, 1), (False, 2), (False, 3), (False, 8)]
# every encoding encode() builds, plus an Arrow validity bitmap and has_values = 0 (every row NULL)
ENCODINGS = ["plain", "base", "bitmap", "dict", "rle", "packed", "arrow", "novalues"]
NULLABLE = ("bitmap", "dict", "rle", "arrow")


def _dbits(x):
    return struct.unpack("<Q", struct.pack("<d", x))[0]


# key domains: each holds 0 and, where the type has it, the all-ones pattern (the table's empty-slot marker)
DOMAINS = {
    T.Int64: [0, 1, 2, 3, 7, 2**63, 2**64 - 1, 12345, 2**62 + 5],
    T.Uint64: [0, 1, 5, 9, 2**63, 2**64 - 1, 99, 2**40],
    T.Double: [_dbits(0.0), _dbits(-0.0), _dbits(1.5), _dbits(-2.25), 0x7FF8000000000000, 0x7FF8000000000001, 0xFFF8000000000000,
               _dbits(float("inf"))],
    T.Boolean: [0, 1],
}


# ------------------------------------------------------------------------------------------------- reference
def tuples(cols):
    """[(values, nulls)] per column -> one key tuple per row: None for NULL, else the payload."""
    per = [[None if nl else v for v, nl in zip(np.asarray(vals, np.uint64).tolist(), np.asarray(nulls, bool).tolist())]
           for vals, nulls in cols]
    return list(zip(*per)) if per else []


def ref_join(primary, foreign, left):
    """The plain dict join: primary / foreign are lists of key tuples -> (primary rows, foreign rows) as uint32 arrays."""
    table = {}
    for f, t in enumerate(foreign):
        table.setdefault(t, []).append(f)
    table = {t: np.asarray(rows, np.uint32) for t, rows in table.items()}
    counts, fs = [], []
    no_row = np.asarray([NO_ROW], np.uint32)
    for t in primary:
        m = table.get(t)
        if m is not None:
            counts.append(len(m))
            fs.append(m)
        elif left:
            counts.append(1)
            fs.append(no_row)
        else:
            counts.append(0)
    ps = np.repeat(np.arange(len(primary), dtype=np.uint32), counts)
    return ps, (np.concatenate(fs) if fs else np.zeros(0, np.uint32))


# ------------------------------------------------------------------------------------------------- inputs
def make_column(kind, vtype, values, nulls, rng, start=3):
    """A Column of `kind` decoding to `values` (NULL where nulls) -> (Column, the nulls it really has)."""
    from ytsaurus_b200 import Column
    n = len(values)
    if kind == "novalues":
        return Column(vtype, values=None, value_count=n, null_bitmap=M._bm(np.zeros(n, bool))), np.ones(n, bool)
    if kind == "arrow":
        return Column(vtype, values=np.asarray(values, np.uint64), null_bitmap=M._bm(~nulls), arrow_validity=True), nulls
    if kind not in NULLABLE:
        nulls = np.zeros(n, bool)
    return M.encode(kind, vtype, np.asarray(values, np.uint64), nulls if kind in NULLABLE else None, start, rng), nulls


def side(rng, n, key_types, kinds, domains=None, null_rate=0.1):
    """One side's key columns -> (Columns, [(values, nulls)] for the reference)."""
    cols, ref = [], []
    for k, vtype in enumerate(key_types):
        dom = np.asarray((domains or DOMAINS)[vtype], np.uint64)
        values = dom[rng.integers(0, len(dom), n)] if n else np.zeros(0, np.uint64)
        kind = kinds[k % len(kinds)]
        nulls = rng.random(n) < null_rate if kind in NULLABLE else np.zeros(n, bool)
        col, real = make_column(kind, vtype, values, nulls, rng)
        cols.append(col)
        ref.append((values, real))
    return cols, ref


def on_host(x):
    """A result array as an unsigned numpy array of its element size."""
    import torch
    if torch.is_tensor(x):
        x = x.cpu().numpy()
    x = np.asarray(x)
    return x.view({1: np.uint8, 4: np.uint32, 8: np.uint64}[x.dtype.itemsize])


def u32(x):
    return on_host(x).view(np.uint32)


def check_join(ctx, pcols, pref, fcols, fref, kind, device=False):
    if device:
        pcols = [M.to_device(copy.copy(c)) for c in pcols]
        fcols = [M.to_device(copy.copy(c)) for c in fcols]
    want_p, want_f = ref_join(tuples(pref), tuples(fref), kind == capi.JOIN_LEFT)
    got_p, got_f = ctx.hash_join(pcols, fcols, kind)
    np.testing.assert_array_equal(u32(got_p), want_p)
    np.testing.assert_array_equal(u32(got_f), want_f)
    assert ctx.hash_join(pcols, fcols, kind, count_only=True) == len(want_p)
    return len(want_p)


# ------------------------------------------------------------------------------------------------- header (no GPU)
HEADER_PROGRAM = r"""
#include <stdio.h>
#include "include/ytgpu.h"
int main(void) {
    ytgpu_join_kind inner = YTGPU_JOIN_INNER, left = YTGPU_JOIN_LEFT;
    printf("%d %d %u %d\n", (int)inner, (int)left, (unsigned)YTGPU_JOIN_NO_ROW, YTGPU_JOIN_MAX_KEYS);
    return 0;
}
"""


def test_header_compiles_as_c99_with_the_join_calls():
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "j.c"), os.path.join(d, "j")
        open(src, "w").write(HEADER_PROGRAM)
        subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", ROOT, src, "-o", exe])
        out = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    assert out == [capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_NO_ROW, capi.JOIN_MAX_KEYS] == [0, 1, 0xFFFFFFFF, 8]
    for name in ("ytgpu_hash_join", "ytgpu_gather_column", "ytgpu_gather_string_column"):
        assert name in capi.EXPORTED_SYMBOLS
    assert capi.KC_JOIN == 11


def test_reference_join_order_and_null_rule():
    p = [(1,), (None,), (2,), (3,)]
    f = [(2,), (1,), (None,), (2,)]
    ps, fs = ref_join(p, f, left=True)
    assert ps.tolist() == [0, 1, 2, 2, 3] and fs.tolist() == [1, 2, 0, 3, NO_ROW]
    ps, fs = ref_join(p, f, left=False)
    assert ps.tolist() == [0, 1, 2, 2] and fs.tolist() == [1, 2, 0, 3]


def test_host_adapter_builds_and_refuses_cpu():
    import torch
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "join_ut"], stdout=subprocess.DEVNULL)
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([os.path.join(ROOT, "host", "join_ut")], capture_output=True, text=True, timeout=120)
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


@pytest.mark.gpu
@pytest.mark.parametrize("vtype", TYPES, ids=["i64", "u64", "dbl", "bool"])
@pytest.mark.parametrize("case", PROBE_CASES, ids=lambda c: ("D" if c[0] else "g") + str(c[1]))
def test_gpu_probe_specialisations(ctx, case, vtype):
    direct, nk = case
    rng = np.random.default_rng(hash((direct, nk, int(vtype))) & 0xFFFF)
    key_types = [vtype] if nk <= 2 else [TYPES[(TYPES.index(vtype) + k) % 4] for k in range(nk)]
    key_types = key_types * nk if nk <= 2 else key_types
    for trial, kind in enumerate((capi.JOIN_INNER, capi.JOIN_LEFT)):
        if direct:
            pk = fk = ["plain"]
        else:  # every encoding on each side, independently, shifted so that the two sides differ
            pk = ENCODINGS[trial:] + ENCODINGS[:trial]
            fk = ENCODINGS[3 + trial:] + ENCODINGS[:3 + trial]
        pcols, pref = side(rng, 3001, key_types, pk)
        fcols, fref = side(rng, 1999, key_types, fk)
        check_join(ctx, pcols, pref, fcols, fref, kind, device=trial == 1)
        if not direct:  # each encoding on key 0 of either side
            for e in ENCODINGS:
                pcols, pref = side(rng, 700, key_types, [e] + pk[1:])
                fcols, fref = side(rng, 500, key_types, fk)
                check_join(ctx, pcols, pref, fcols, fref, kind)
                pcols, pref = side(rng, 700, key_types, pk)
                fcols, fref = side(rng, 500, key_types, [e] + fk[1:])
                check_join(ctx, pcols, pref, fcols, fref, kind)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_edges(ctx, device):
    rng = np.random.default_rng(5)
    t = [T.Int64]
    empty_p, empty_pref = side(rng, 0, t, ["plain"])
    empty_f, empty_fref = side(rng, 0, t, ["plain"])
    pcols, pref = side(rng, 1000, t, ["bitmap"])
    fcols, fref = side(rng, 600, t, ["dict"])
    for kind in (capi.JOIN_INNER, capi.JOIN_LEFT):
        assert check_join(ctx, empty_p, empty_pref, fcols, fref, kind, device) == 0
        n = check_join(ctx, pcols, pref, empty_f, empty_fref, kind, device)
        assert n == (1000 if kind == capi.JOIN_LEFT else 0)
        # no match at all: disjoint domains, no NULLs
        a, aref = side(rng, 900, t, ["plain"], {T.Int64: [1, 2, 3]})
        b, bref = side(rng, 400, t, ["rle"], {T.Int64: [4, 5]}, null_rate=0)
        assert check_join(ctx, a, aref, b, bref, kind, device) == (900 if kind == capi.JOIN_LEFT else 0)
        # every primary row matching exactly once: unique foreign keys
        keys = np.arange(1000, dtype=np.uint64) * 3
        f, _ = make_column("plain", T.Int64, keys, np.zeros(1000, bool), rng)
        pv = keys[rng.integers(0, 1000, 5000)]
        p, _ = make_column("packed", T.Int64, pv, np.zeros(5000, bool), rng)
        assert check_join(ctx, [p], [(pv, np.zeros(5000, bool))], [f], [(keys, np.zeros(1000, bool))], kind, device) == 5000


@pytest.mark.gpu
def test_gpu_null_and_float_rules(ctx):
    rng = np.random.default_rng(9)
    nan_a, nan_b = 0x7FF8000000000000, 0x7FF8000000000001
    pv = np.asarray([_dbits(0.0), _dbits(-0.0), nan_a, nan_b, 0, _dbits(1.0)], np.uint64)
    pn = np.asarray([0, 0, 0, 0, 1, 0], bool)
    fv = np.asarray([_dbits(-0.0), nan_a, 0, _dbits(0.0), _dbits(2.0)], np.uint64)
    fn = np.asarray([0, 0, 1, 0, 0], bool)
    p, _ = make_column("bitmap", T.Double, pv, pn, rng)
    f, _ = make_column("bitmap", T.Double, fv, fn, rng)
    got_p, got_f = ctx.hash_join([p], [f], capi.JOIN_LEFT)
    # +0.0 matches +0.0 only, -0.0 -0.0 only, the same NaN bits only, NULL the NULL
    assert u32(got_p).tolist() == [0, 1, 2, 3, 4, 5]
    assert u32(got_f).tolist() == [3, 0, 1, NO_ROW, 2, NO_ROW]
    check_join(ctx, [p], [(pv, pn)], [f], [(fv, fn)], capi.JOIN_INNER)


@pytest.mark.gpu
def test_gpu_fanout_and_skew(ctx):
    import torch
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(13)
    # one key with 10^5 foreign rows among 10^4 unique ones; 10^6 primary rows, three of them on the hot key
    fv = np.concatenate([np.full(100_000, 7, np.uint64), np.arange(10_000, dtype=np.uint64) + 100])
    fv = fv[rng.permutation(len(fv))]
    pv = (rng.integers(0, 10_000, 1_000_000) + 100).astype(np.uint64)
    pv[[5, 500_000, 999_999]] = 7
    pv[rng.integers(0, 1_000_000, 1000)] = 3  # misses
    dev = lambda a: torch.from_numpy(a.view(np.int64)).cuda()
    p, f = Column(T.Int64, values=dev(pv)), Column(T.Int64, values=dev(fv))
    z = lambda a: np.zeros(len(a), bool)
    for kind in (capi.JOIN_INNER, capi.JOIN_LEFT):
        n = check_join(ctx, [p], [(pv, z(pv))], [f], [(fv, z(fv))], kind)
        assert n > 300_000
    # every key equal: P x F pairs, each primary row's list crossing write tiles
    pv, fv = np.full(3000, 42, np.uint64), np.full(2500, 42, np.uint64)
    p, f = Column(T.Int64, values=dev(pv)), Column(T.Int64, values=dev(fv))
    assert check_join(ctx, [p], [(pv, z(pv))], [f], [(fv, z(fv))], capi.JOIN_INNER) == 3000 * 2500


@pytest.mark.gpu
@pytest.mark.parametrize("covered", [((0, 1), (99, 100)), ((99, 100),), ((0, 1),), ((45, 55),)],
                         ids=["ends", "last", "first", "middle"])
def test_gpu_long_runs_of_inner_misses(ctx, covered):
    """A primary table sorted by key against a dimension that covers only parts of the key range: the pair write crosses
    runs of up to ~10^6 rows without pairs (INNER) between consecutive output positions."""
    import torch
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(41)
    D = 1_000_000
    pv = np.sort(rng.integers(0, D, 1_000_000)).astype(np.uint64)
    fv = np.concatenate([np.arange(lo * D // 100, hi * D // 100, dtype=np.uint64) for lo, hi in covered])
    fv = np.concatenate([fv, fv[rng.integers(0, len(fv), len(fv) // 3)]])  # some keys with two or three foreign rows
    fv = fv[rng.permutation(len(fv))]
    dev = lambda a: torch.from_numpy(a.view(np.int64)).cuda()
    z = lambda a: np.zeros(len(a), bool)
    p, f = Column(T.Int64, values=dev(pv)), Column(T.Int64, values=dev(fv))
    for kind in (capi.JOIN_INNER, capi.JOIN_LEFT):
        n = check_join(ctx, [p], [(pv, z(pv))], [f], [(fv, z(fv))], kind)
        assert n > 0


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_foreign_lists_on_the_large_sort_path(ctx, device):
    """At least 2^18 shuffled foreign rows with duplicated keys: the per-key lists come from the radix sort's packed and
    hybrid schedules, and must still hold each key's foreign rows in ascending order."""
    rng = np.random.default_rng(43)
    dom = {T.Int64: list(range(5000))}
    pcols, pref = side(rng, 20_000, [T.Int64], ["plain"], {T.Int64: list(range(6000))})
    fcols, fref = side(rng, 300_000, [T.Int64], ["dict"], dom, null_rate=0.001)
    assert len(fref[0][0]) >= 2**18
    for kind in (capi.JOIN_INNER, capi.JOIN_LEFT):
        assert check_join(ctx, pcols, pref, fcols, fref, kind, device) > 500_000


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_count_query_and_capacity(ctx, device):
    import ctypes as C
    rng = np.random.default_rng(17)
    pcols, pref = side(rng, 2000, [T.Uint64], ["dict"])
    fcols, fref = side(rng, 1500, [T.Uint64], ["bitmap"])
    if device:
        pcols, fcols = [M.to_device(c) for c in pcols], [M.to_device(c) for c in fcols]
    want_p, _ = ref_join(tuples(pref), tuples(fref), False)
    count = ctx.hash_join(pcols, fcols, capi.JOIN_INNER, count_only=True)
    assert count == len(want_p) > 0
    with pytest.raises(capi.YtGpuError) as e:
        ctx.hash_join(pcols, fcols, capi.JOIN_INNER, capacity=count - 1)
    assert e.value.code == capi.ERR_INVALID_ARGUMENT and e.value.pair_count == count
    # exactly one output NULL
    pv, fv = (capi.ColumnView * 1)(pcols[0].view()), (capi.ColumnView * 1)(fcols[0].view())
    out = np.zeros(count, np.uint32)
    n, err = C.c_uint64(0), capi.Error()
    code = ctx.lib.ytgpu_hash_join(ctx.handle, C.cast(pv, C.c_void_p), C.cast(fv, C.c_void_p), 1, capi.JOIN_INNER, out.ctypes.data, None,
                                   count, C.byref(n), capi.MEM_HOST, C.byref(err))
    assert code == capi.ERR_INVALID_ARGUMENT


def _code(fn):
    try:
        fn()
    except capi.YtGpuError as e:
        return e.code
    return capi.OK


@pytest.mark.gpu
def test_gpu_refusals(ctx):
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(19)
    p, _ = side(rng, 100, [T.Int64], ["plain"])
    f, _ = side(rng, 100, [T.Int64], ["plain"])
    fu, _ = side(rng, 100, [T.Uint64], ["plain"])
    inner = capi.JOIN_INNER
    assert _code(lambda: ctx.hash_join([], [], inner)) == capi.ERR_INVALID_ARGUMENT
    assert _code(lambda: ctx.hash_join(p * 9, f * 9, inner)) == capi.ERR_INVALID_ARGUMENT
    assert _code(lambda: ctx.hash_join(p, f, 2)) == capi.ERR_INVALID_ARGUMENT
    assert _code(lambda: ctx.hash_join(p, fu, inner)) == capi.ERR_INVALID_ARGUMENT
    short, _ = side(rng, 99, [T.Int64], ["plain"])
    assert _code(lambda: ctx.hash_join(p + short, f + f, inner)) == capi.ERR_INVALID_ARGUMENT
    # more than 2^30 rows: refused from the view alone, before any access
    huge = Column(T.Int64, values=np.zeros(1, np.uint64), value_count=2**30 + 1)
    assert _code(lambda: ctx.hash_join([huge], f, inner)) == capi.ERR_UNSUPPORTED
    assert _code(lambda: ctx.hash_join(p, [huge], inner)) == capi.ERR_UNSUPPORTED
    # the foreign rows go through the radix sort, which takes fewer than 2^30 rows
    exact = Column(T.Int64, values=np.zeros(1, np.uint64), value_count=2**30)
    assert _code(lambda: ctx.hash_join(p, [exact], inner)) == capi.ERR_UNSUPPORTED
    s = Column(T.String, values=np.zeros(100, np.uint64))
    assert _code(lambda: ctx.hash_join([s], [s], inner)) == capi.ERR_UNSUPPORTED


def _strings(rng, n, pool):
    vals = [pool[i] for i in rng.integers(0, len(pool), n)]
    return [None if rng.random() < 0.1 else v for v in vals]


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_string_keys_through_joint_value_ids(ctx, device):
    import torch
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(23)
    fs = _strings(rng, 800, [b"", b"a", b"b", b"foreign-only", b"\x00x", b"long" * 20])
    ps = _strings(rng, 1200, [b"", b"a", b"b", b"primary-only", b"\x00x", b"long" * 20, b"lon"])
    vals = fs + ps
    heap = np.frombuffer(b"".join(v or b"" for v in vals), np.uint8).copy()
    lengths = np.asarray([len(v or b"") for v in vals], np.uint32)
    starts = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.uint64)
    nulls = np.asarray([v is None for v in vals], np.uint8)
    args = (heap, starts, lengths, nulls)
    if device:
        args = tuple(torch.from_numpy(a.view({1: np.uint8, 4: np.int32, 8: np.int64}[a.dtype.itemsize])).cuda() for a in args)
    ids, onull = ctx.string_value_ids(*args)
    F = len(fs)
    fcol = Column(T.Uint64, values=ids[:F].contiguous() if device else ids[:F].copy(), null_bitmap=M._bm(nulls[:F].astype(bool)))
    pcol = Column(T.Uint64, values=ids[F:].contiguous() if device else ids[F:].copy(), null_bitmap=M._bm(nulls[F:].astype(bool)))
    if device:
        for c in (fcol, pcol):
            c.null_bitmap = torch.from_numpy(c.null_bitmap).cuda()
    for kind in (capi.JOIN_INNER, capi.JOIN_LEFT):
        want_p, want_f = ref_join([(v,) for v in ps], [(v,) for v in fs], kind == capi.JOIN_LEFT)
        got_p, got_f = ctx.hash_join([pcol], [fcol], kind)
        np.testing.assert_array_equal(u32(got_p), want_p)
        np.testing.assert_array_equal(u32(got_f), want_f)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("kind", ENCODINGS)
def test_gpu_gather_column(ctx, kind, device):
    import torch
    rng = np.random.default_rng(29 + ENCODINGS.index(kind))
    for vtype in TYPES:
        n = 1000
        dom = np.asarray(DOMAINS[vtype], np.uint64)
        values = dom[rng.integers(0, len(dom), n)]
        col, nulls = make_column(kind, vtype, values, rng.random(n) < 0.2, rng)
        count = 777  # not a multiple of 64: the bitmap's tail bits must be zero
        rows = rng.integers(0, n, count).astype(np.uint32)
        rows[rng.random(count) < 0.1] = NO_ROW
        if device:
            col = M.to_device(col)
        r = torch.from_numpy(rows.view(np.int32)).cuda() if device else rows
        got = ctx.gather_column(col, r)
        gv, gb = on_host(got["values"]), on_host(got["null_bitmap"])
        want_null = (rows == NO_ROW) | np.where(rows == NO_ROW, True, nulls[np.minimum(rows, n - 1)])
        want_vals = np.where(want_null, np.uint64(0), values[np.minimum(rows, n - 1)])
        assert len(gb) == (count + 63) // 64 * 8
        bits = np.unpackbits(np.asarray(gb, np.uint8), bitorder="little").astype(bool)
        np.testing.assert_array_equal(bits[:count], want_null)
        assert not bits[count:].any()
        np.testing.assert_array_equal(gv, want_vals)
        assert got["null_count"] == int(want_null.sum())
    bad = rows.copy()
    bad[3] = n  # neither below the column's length nor NO_ROW
    with pytest.raises(capi.YtGpuError) as e:
        ctx.gather_column(col, torch.from_numpy(bad.view(np.int32)).cuda() if device else bad)
    assert e.value.code == capi.ERR_INVALID_ARGUMENT


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_gather_string_column(ctx, device):
    import torch
    rng = np.random.default_rng(31)
    vals = _strings(rng, 500, [b"", b"x", b"yy", b"zzz" * 9])
    heap = np.frombuffer(b"".join(v or b"" for v in vals), np.uint8).copy()
    lengths = np.asarray([len(v or b"") for v in vals], np.uint32)
    starts = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.uint64)
    nulls = np.asarray([v is None for v in vals], np.uint8)
    rows = rng.integers(0, 500, 1234).astype(np.uint32)
    rows[::7] = NO_ROW
    args = (heap, starts, lengths, nulls, rows)
    if device:
        args = tuple(torch.from_numpy(a.view({1: np.uint8, 4: np.int32, 8: np.int64}[a.dtype.itemsize])).cuda() for a in args)
    h, s, ln, nb = ctx.gather_string_column(*args)
    s, ln, nb = (on_host(x) for x in (s, ln, nb))
    hp = bytes(on_host(h))
    for i, r in enumerate(rows.tolist()):
        want = None if r == NO_ROW else vals[r]
        if want is None:
            assert nb[i] == 1 and s[i] == 0 and ln[i] == 0
        else:
            assert nb[i] == 0 and hp[s[i]:s[i] + ln[i]] == want
    bad = rows.copy()
    bad[0] = 500
    args = args[:4] + ((torch.from_numpy(bad.view(np.int32)).cuda() if device else bad),)
    with pytest.raises(capi.YtGpuError) as e:
        ctx.gather_string_column(*args)
    assert e.value.code == capi.ERR_INVALID_ARGUMENT


@pytest.mark.gpu
def test_gpu_join_timer_class(ctx):
    rng = np.random.default_rng(37)
    pcols, _ = side(rng, 5000, [T.Int64], ["plain"])
    fcols, _ = side(rng, 3000, [T.Int64], ["plain"])
    ctx.reset_timers()
    ctx.enable_timers(True)
    ctx.hash_join(pcols, fcols, capi.JOIN_LEFT)
    ms, launches = ctx.kernel_ms(capi.KC_JOIN)
    ctx.enable_timers(False)
    assert launches > 0 and ms > 0


@pytest.mark.gpu
def test_gpu_host_adapter_join_clause(ctx):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "join_ut"], stdout=subprocess.DEVNULL)
    r = subprocess.run([os.path.join(ROOT, "host", "join_ut")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    assert "join_ut: 0 failure(s)" in r.stdout
