"""The join table on the GPU (csrc/join.cu): ytgpu_join_table_build / _probe / _destroy against a plain Python dict join,
and the YQL block map join adapter over it (host/tests/map_join_ut.cpp).

The reference builds a dict from each foreign key tuple to its foreign rows in ascending order, then walks the primary rows
in order.  A tuple is (None or the 64-bit payload) per column, so doubles compare by bit pattern under both NULL rules.
Under NULLS_EQUAL a None equals a None; under NULLS_NEVER_MATCH a tuple holding a None matches nothing: it is not in the
dict, and a primary tuple holding one finds nothing.  INNER / LEFT give (primary rows, foreign rows), SEMI / ANTI the
ascending primary rows; all are compared for exact equality."""
import copy
import ctypes as C
import gc
import importlib.util
import os
import subprocess
import tempfile

import numpy as np
import pytest

from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import EValueType as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NO_ROW = capi.JOIN_NO_ROW
KINDS = [capi.JOIN_INNER, capi.JOIN_LEFT, capi.JOIN_SEMI, capi.JOIN_ANTI]
KIND_IDS = ["inner", "left", "semi", "anti"]
RULES = [capi.JOIN_NULLS_EQUAL, capi.JOIN_NULLS_NEVER_MATCH]
RULE_IDS = ["nulls_equal", "never_match"]


def _load(name):
    """A sibling test module's helpers, loaded by path so no import mode matters."""
    spec = importlib.util.spec_from_file_location("_join_table_" + name[:-3], os.path.join(os.path.dirname(os.path.abspath(__file__)), name))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


M = _load("test_groupby_kernel_matrix.py")  # encode(), to_device(), _bm()

TYPES = [T.Int64, T.Uint64, T.Double, T.Boolean]
# every encoding of test_hash_join.py: encode()'s, an Arrow validity bitmap and has_values = 0 (every row NULL); every
# column starts at start_index 3 (a window over its value vector)
ENCODINGS = ["plain", "base", "bitmap", "dict", "rle", "packed", "arrow", "novalues"]
NULLABLE = ("bitmap", "dict", "rle", "arrow")


def _dbits(x):
    import struct
    return struct.unpack("<Q", struct.pack("<d", x))[0]


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


def ref_join(primary, foreign, kind, nulls):
    """The plain dict join -> (primary rows, foreign rows) for INNER / LEFT, the primary rows for SEMI / ANTI."""
    never = nulls == capi.JOIN_NULLS_NEVER_MATCH
    table = {}
    for f, t in enumerate(foreign):
        if not (never and None in t):
            table.setdefault(t, []).append(f)
    ps, fs, rows = [], [], []
    for p, t in enumerate(primary):
        m = None if never and None in t else table.get(t)
        if kind == capi.JOIN_SEMI:
            if m:
                rows.append(p)
        elif kind == capi.JOIN_ANTI:
            if not m:
                rows.append(p)
        elif m:
            ps += [p] * len(m)
            fs += m
        elif kind == capi.JOIN_LEFT:
            ps.append(p)
            fs.append(NO_ROW)
    if kind in (capi.JOIN_SEMI, capi.JOIN_ANTI):
        return np.asarray(rows, np.uint32)
    return np.asarray(ps, np.uint32), np.asarray(fs, np.uint32)


# ------------------------------------------------------------------------------------------------- inputs (as test_hash_join.py)
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
    import torch
    if torch.is_tensor(x):
        x = x.cpu().numpy()
    x = np.asarray(x)
    return x.view({1: np.uint8, 4: np.uint32, 8: np.uint64}[x.dtype.itemsize])


def u32(x):
    return on_host(x).view(np.uint32)


def check_probe(table, pcols, pref, fref, kind, nulls, **kw):
    """One probe against the reference; -> the number of rows / pairs."""
    want = ref_join(tuples(pref), tuples(fref), kind, nulls)
    got = table.probe(pcols, kind, **kw)
    if kind in (capi.JOIN_SEMI, capi.JOIN_ANTI):
        np.testing.assert_array_equal(u32(got), want)
        n = len(want)
    else:
        np.testing.assert_array_equal(u32(got[0]), want[0])
        np.testing.assert_array_equal(u32(got[1]), want[1])
        n = len(want[0])
    assert table.probe(pcols, kind, count_only=True) == n
    return n


# ------------------------------------------------------------------------------------------------- no GPU
HEADER_PROGRAM = r"""
#include <stdio.h>
#include "include/ytgpu.h"
int main(void) {
    ytgpu_join_kind semi = YTGPU_JOIN_SEMI, anti = YTGPU_JOIN_ANTI;
    ytgpu_join_nulls eq = YTGPU_JOIN_NULLS_EQUAL, never = YTGPU_JOIN_NULLS_NEVER_MATCH;
    printf("%d %d %d %d\n", (int)semi, (int)anti, (int)eq, (int)never);
    return 0;
}
"""
DECLARATIONS = r"""
#include "include/ytgpu.h"
int build_it(ytgpu_context* c, const ytgpu_column_view* k, ytgpu_join_table** t) { return ytgpu_join_table_build(c, k, 1, YTGPU_JOIN_NULLS_EQUAL, t, 0); }
int probe_it(ytgpu_context* c, const ytgpu_join_table* t, const ytgpu_column_view* k, uint32_t* p, uint64_t* n) {
    return ytgpu_join_table_probe(c, t, k, 1, YTGPU_JOIN_SEMI, p, 0, 0, n, YTGPU_MEM_HOST, 0);
}
int destroy_it(ytgpu_join_table* t) { return ytgpu_join_table_destroy(t, 0); }
"""


def test_header_and_bindings_declare_the_table_calls():
    with tempfile.TemporaryDirectory() as d:
        src, exe, obj = os.path.join(d, "j.c"), os.path.join(d, "j"), os.path.join(d, "decl.o")
        open(src, "w").write(HEADER_PROGRAM)
        subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", ROOT, src, "-o", exe])
        out = [int(x) for x in subprocess.check_output([exe], text=True).split()]
        decl = os.path.join(d, "decl.c")
        open(decl, "w").write(DECLARATIONS)
        subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", ROOT, "-c", decl, "-o", obj])
    assert out == [capi.JOIN_SEMI, capi.JOIN_ANTI, capi.JOIN_NULLS_EQUAL, capi.JOIN_NULLS_NEVER_MATCH] == [2, 3, 0, 1]
    lib = capi.load()
    for name in ("ytgpu_join_table_build", "ytgpu_join_table_probe", "ytgpu_join_table_destroy"):
        assert name in capi.EXPORTED_SYMBOLS
        assert getattr(lib, name).argtypes is not None
    assert lib.ytgpu_join_table_destroy(None, None) == capi.OK  # destroy(NULL) is a no-op, no device needed


def test_reference_kinds_and_null_rules():
    p = [(1,), (None,), (2,), (3,)]
    f = [(2,), (1,), (None,), (2,)]
    eq, never = capi.JOIN_NULLS_EQUAL, capi.JOIN_NULLS_NEVER_MATCH
    assert [x.tolist() for x in ref_join(p, f, capi.JOIN_LEFT, eq)] == [[0, 1, 2, 2, 3], [1, 2, 0, 3, NO_ROW]]
    assert [x.tolist() for x in ref_join(p, f, capi.JOIN_LEFT, never)] == [[0, 1, 2, 2, 3], [1, NO_ROW, 0, 3, NO_ROW]]
    assert ref_join(p, f, capi.JOIN_SEMI, eq).tolist() == [0, 1, 2]
    assert ref_join(p, f, capi.JOIN_SEMI, never).tolist() == [0, 2]
    assert ref_join(p, f, capi.JOIN_ANTI, never).tolist() == [1, 3]


def test_map_join_adapter_builds_and_refuses_cpu():
    import torch
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "map_join_ut"], stdout=subprocess.DEVNULL)
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([os.path.join(ROOT, "host", "map_join_ut")], capture_output=True, text=True, timeout=120)
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
@pytest.mark.parametrize("nulls", RULES, ids=RULE_IDS)
@pytest.mark.parametrize("nk", [1, 2, 3, 8])
def test_gpu_kinds_rules_keys_and_encodings(ctx, nk, nulls):
    """Every kind under both rules, over 1, 2, 3 and 8 key columns (plain 64-bit on both sides, then every encoding on each
    side, shifted so that the sides differ), in HOST and DEVICE memory.  Small domains give duplicate foreign keys, and
    the nullable encodings put NULLs in some but not all components of a tuple."""
    rng = np.random.default_rng(1000 * nk + nulls)
    key_types = [TYPES[k % 4] for k in range(nk)]
    layouts = [(["plain"], ["plain"])] + [(ENCODINGS[t:] + ENCODINGS[:t], ENCODINGS[3 + t:] + ENCODINGS[:3 + t]) for t in range(2)]
    for trial, (pk, fk) in enumerate(layouts):
        pcols, pref = side(rng, 2500, key_types, pk)
        fcols, fref = side(rng, 1700, key_types, fk)
        if trial == 1:
            pcols = [M.to_device(copy.copy(c)) for c in pcols]
            fcols = [M.to_device(copy.copy(c)) for c in fcols]
        with ctx.join_table(fcols, nulls) as table:
            for kind in KINDS:
                check_probe(table, pcols, pref, fref, kind, nulls)
    if nk == 1:  # each encoding on key 0 of either side
        for e in ENCODINGS:
            pcols, pref = side(rng, 700, key_types, [e])
            fcols, fref = side(rng, 500, key_types, ["dict"])
            with ctx.join_table(fcols, nulls) as table:
                for kind in KINDS:
                    check_probe(table, pcols, pref, fref, kind, nulls)
            pcols, pref = side(rng, 700, key_types, ["bitmap"])
            fcols, fref = side(rng, 500, key_types, [e])
            with ctx.join_table(fcols, nulls) as table:
                for kind in KINDS:
                    check_probe(table, pcols, pref, fref, kind, nulls)


@pytest.mark.gpu
@pytest.mark.parametrize("nulls", RULES, ids=RULE_IDS)
def test_gpu_double_keys_by_bit_pattern(ctx, nulls):
    rng = np.random.default_rng(9)
    nan_a, nan_b = 0x7FF8000000000000, 0x7FF8000000000001
    pv = np.asarray([_dbits(0.0), _dbits(-0.0), nan_a, nan_b, 0, _dbits(1.0)], np.uint64)
    pn = np.asarray([0, 0, 0, 0, 1, 0], bool)
    fv = np.asarray([_dbits(-0.0), nan_a, 0, _dbits(0.0), _dbits(2.0)], np.uint64)
    fn = np.asarray([0, 0, 1, 0, 0], bool)
    p, _ = make_column("bitmap", T.Double, pv, pn, rng)
    f, _ = make_column("bitmap", T.Double, fv, fn, rng)
    with ctx.join_table([f], nulls) as table:
        got_p, got_f = table.probe([p], capi.JOIN_LEFT)
        null_match = 2 if nulls == capi.JOIN_NULLS_EQUAL else NO_ROW
        # +0.0 matches +0.0 only, -0.0 -0.0 only, the same NaN bits only; NULL the NULL under the QL rule only
        assert u32(got_p).tolist() == [0, 1, 2, 3, 4, 5]
        assert u32(got_f).tolist() == [3, 0, 1, NO_ROW, null_match, NO_ROW]
        assert u32(table.probe([p], capi.JOIN_SEMI)).tolist() == ([0, 1, 2, 4] if nulls == capi.JOIN_NULLS_EQUAL else [0, 1, 2])
        assert u32(table.probe([p], capi.JOIN_ANTI)).tolist() == ([3, 5] if nulls == capi.JOIN_NULLS_EQUAL else [3, 4, 5])


def _probe_blocks(table, values, kind, sizes):
    """values (a device int64 tensor) probed block by block; -> the results concatenated, rows shifted by the block start."""
    from ytsaurus_b200 import Column
    ps, fs, start = [], [], 0
    for size in sizes:
        got = table.probe([Column(T.Int64, values=values[start:start + size])], kind)
        if kind in (capi.JOIN_SEMI, capi.JOIN_ANTI):
            ps.append(u32(got).astype(np.int64) + start)
        else:
            ps.append(u32(got[0]).astype(np.int64) + start)
            fs.append(u32(got[1]))
        start += size
    return np.concatenate(ps), (np.concatenate(fs) if fs else None)


@pytest.mark.gpu
@pytest.mark.parametrize("nulls", RULES, ids=RULE_IDS)
def test_gpu_block_probing_equals_one_probe(ctx, nulls):
    import torch
    from ytsaurus_b200 import Column
    g = torch.Generator(device="cuda").manual_seed(77)
    fkeys = torch.randint(0, 60_000, (40_000,), device="cuda", generator=g)  # duplicates
    pkeys = torch.randint(0, 120_000, (150_001,), device="cuda", generator=g)
    sizes = [1, 31, 2049, 65537]
    sizes.append(pkeys.numel() - sum(sizes))  # the uneven remainder
    with ctx.join_table([Column(T.Int64, values=fkeys)], nulls) as table:
        for kind in KINDS:
            whole = table.probe([Column(T.Int64, values=pkeys)], kind)
            bp, bf = _probe_blocks(table, pkeys, kind, sizes)
            if kind in (capi.JOIN_SEMI, capi.JOIN_ANTI):
                np.testing.assert_array_equal(bp, u32(whole).astype(np.int64))
            else:
                np.testing.assert_array_equal(bp, u32(whole[0]).astype(np.int64))
                np.testing.assert_array_equal(bf, u32(whole[1]))
        # and the whole probe against numpy
        fk, pk = fkeys.cpu().numpy(), pkeys.cpu().numpy()
        np.testing.assert_array_equal(u32(table.probe([Column(T.Int64, values=pkeys)], capi.JOIN_SEMI)), np.flatnonzero(np.isin(pk, fk)))


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_same_pairs_as_hash_join(ctx, device):
    rng = np.random.default_rng(21)
    for nk, pk, fk in [(1, ["dict"], ["bitmap"]), (2, ["plain"], ["plain"]), (3, ENCODINGS, ENCODINGS[2:] + ENCODINGS[:2])]:
        key_types = [TYPES[k % 4] for k in range(nk)]
        pcols, _ = side(rng, 3000, key_types, pk)
        fcols, _ = side(rng, 2000, key_types, fk)
        if device:
            pcols, fcols = [M.to_device(copy.copy(c)) for c in pcols], [M.to_device(copy.copy(c)) for c in fcols]
        with ctx.join_table(fcols, capi.JOIN_NULLS_EQUAL) as table:
            for kind in (capi.JOIN_INNER, capi.JOIN_LEFT):
                a, b = table.probe(pcols, kind)
                c, d = ctx.hash_join(pcols, fcols, kind)
                np.testing.assert_array_equal(u32(a), u32(c))
                np.testing.assert_array_equal(u32(b), u32(d))


@pytest.mark.gpu
def test_gpu_string_keys_through_joint_value_ids(ctx):
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(23)
    pool = [b"", b"a", b"b", b"foreign-only", b"\x00x", b"long" * 20, b"lon"]
    vals = [None if rng.random() < 0.1 else pool[i] for i in rng.integers(0, len(pool), 2000)]
    F = 800
    heap = np.frombuffer(b"".join(v or b"" for v in vals), np.uint8).copy()
    lengths = np.asarray([len(v or b"") for v in vals], np.uint32)
    starts = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.uint64)
    nulls = np.asarray([v is None for v in vals], np.uint8)
    ids, _ = ctx.string_value_ids(heap, starts, lengths, nulls)
    fcol = Column(T.Uint64, values=ids[:F].copy(), null_bitmap=M._bm(nulls[:F].astype(bool)))
    pcol = Column(T.Uint64, values=ids[F:].copy(), null_bitmap=M._bm(nulls[F:].astype(bool)))
    with ctx.join_table([fcol]) as table:
        for kind in (capi.JOIN_INNER, capi.JOIN_LEFT):
            a, b = table.probe([pcol], kind)
            c, d = ctx.hash_join([pcol], [fcol], kind)
            np.testing.assert_array_equal(u32(a), u32(c))
            np.testing.assert_array_equal(u32(b), u32(d))


@pytest.mark.gpu
@pytest.mark.parametrize("nulls", RULES, ids=RULE_IDS)
def test_gpu_table_owns_its_keys(ctx, nulls):
    import torch
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(31)
    pcols, pref = side(rng, 3000, [T.Int64, T.Double], ["bitmap", "plain"])
    # DEVICE foreign keys, overwritten after the build
    fcols, fref = side(rng, 2000, [T.Int64, T.Double], ["plain", "arrow"])
    dcols = [M.to_device(copy.copy(c)) for c in fcols]
    table_d = ctx.join_table(dcols, nulls)
    for c in dcols:
        c.values.fill_(7)
        if torch.is_tensor(c.null_bitmap):
            c.null_bitmap.fill_(0)
    torch.cuda.synchronize()
    # HOST foreign keys: the arrays overwritten and deleted after the build
    hcols, href = side(rng, 2000, [T.Int64, T.Double], ["dict", "bitmap"])
    table_h = ctx.join_table(hcols, nulls)
    for c in hcols:
        for name in ("values", "null_bitmap", "dictionary_indexes"):
            a = getattr(c, name, None)
            if isinstance(a, np.ndarray):
                a[...] = 0xA5 if a.dtype == np.uint8 else 3
    del hcols
    gc.collect()
    for table, ref in ((table_d, fref), (table_h, href)):
        with table:
            for kind in KINDS:
                check_probe(table, pcols, pref, ref, kind, nulls)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_edge_sides(ctx, device):
    import torch
    rng = np.random.default_rng(5)
    t = [T.Int64]
    empty, empty_ref = side(rng, 0, t, ["plain"])
    pcols, pref = side(rng, 1000, t, ["bitmap"])
    all_null, all_null_ref = side(rng, 300, t, ["novalues"])
    if device:
        pcols = [M.to_device(copy.copy(c)) for c in pcols]
    for nulls in RULES:
        # an empty foreign side: INNER / SEMI give nothing, LEFT / ANTI every row
        with ctx.join_table(empty, nulls) as table:
            want = {capi.JOIN_INNER: 0, capi.JOIN_LEFT: 1000, capi.JOIN_SEMI: 0, capi.JOIN_ANTI: 1000}
            for kind in KINDS:
                assert check_probe(table, pcols, pref, empty_ref, kind, nulls) == want[kind]
            # an empty primary side
            for kind in KINDS:
                assert check_probe(table, empty, empty_ref, empty_ref, kind, nulls) == 0
        with ctx.join_table(all_null, nulls) as table:
            for kind in KINDS:
                n = check_probe(table, pcols, pref, all_null_ref, kind, nulls)
                if nulls == capi.JOIN_NULLS_NEVER_MATCH:  # behaves as the empty side
                    assert n == want[kind]
            assert check_probe(table, empty, empty_ref, all_null_ref, capi.JOIN_ANTI, nulls) == 0
    del torch


@pytest.mark.gpu
def test_gpu_large_primary_side(ctx):
    """2 * 10^7 primary rows U[0, 2 * 10^6) against 10^6 unique foreign keys, checked on a seeded sample."""
    import torch
    from ytsaurus_b200 import Column
    g = torch.Generator(device="cuda").manual_seed(11)
    D, N = 1_000_000, 20_000_000
    fkeys = torch.randperm(2 * D, device="cuda", generator=g)[:D].contiguous()
    pkeys = torch.randint(0, 2 * D, (N,), device="cuda", generator=g)
    where = torch.full((2 * D,), -1, dtype=torch.int64, device="cuda")
    where[fkeys] = torch.arange(D, device="cuda")
    hit = where[pkeys] >= 0
    rng = np.random.default_rng(12)
    sample = np.unique(rng.integers(0, N, 100_000))
    with ctx.join_table([Column(T.Int64, values=fkeys)], capi.JOIN_NULLS_NEVER_MATCH) as table:
        p = [Column(T.Int64, values=pkeys)]
        semi = u32(table.probe(p, capi.JOIN_SEMI)).astype(np.int64)
        anti = u32(table.probe(p, capi.JOIN_ANTI)).astype(np.int64)
        h = hit.cpu().numpy()
        assert len(semi) == int(h.sum()) and len(anti) == N - len(semi)
        assert np.array_equal(np.isin(sample, semi), h[sample]) and not np.isin(sample, anti)[h[sample]].any()
        op, of = table.probe(p, capi.JOIN_INNER)
        op, of = u32(op).astype(np.int64), u32(of)
        np.testing.assert_array_equal(op, semi)  # unique foreign keys: one pair per matching row
        w = where.cpu().numpy()
        pk = pkeys.cpu().numpy()
        pos = np.searchsorted(op, sample)
        ok = h[sample]
        np.testing.assert_array_equal(of[pos[ok]], w[pk[sample[ok]]])


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_out_mem_count_and_capacity(ctx, device):
    rng = np.random.default_rng(17)
    pcols, pref = side(rng, 2000, [T.Uint64], ["dict"])
    fcols, fref = side(rng, 1500, [T.Uint64], ["bitmap"])
    if device:
        pcols = [M.to_device(c) for c in pcols]
    with ctx.join_table(fcols, capi.JOIN_NULLS_NEVER_MATCH) as table:
        for out_mem in (capi.MEM_HOST, capi.MEM_DEVICE):
            for kind in KINDS:
                check_probe(table, pcols, pref, fref, kind, capi.JOIN_NULLS_NEVER_MATCH, out_mem=out_mem)
                count = table.probe(pcols, kind, count_only=True)
                assert count > 0
                with pytest.raises(capi.YtGpuError) as e:
                    table.probe(pcols, kind, capacity=count - 1, out_mem=out_mem)
                assert e.value.code == capi.ERR_INVALID_ARGUMENT and e.value.pair_count == count
                if kind in (capi.JOIN_SEMI, capi.JOIN_ANTI):  # exactly the count suffices, in one call
                    assert len(table.probe(pcols, kind, capacity=count, out_mem=out_mem)) == count


def _raw_probe(ctx, table_handle, cols, kind, out_p=None, out_f=None, capacity=0, key_count=None):
    views = (capi.ColumnView * max(len(cols), 1))(*[c.view() for c in cols])
    n, err = C.c_uint64(0), capi.Error()
    return ctx.lib.ytgpu_join_table_probe(ctx.handle, table_handle, C.cast(views, C.c_void_p), len(cols) if key_count is None else key_count,
                                          kind, out_p, out_f, capacity, C.byref(n), capi.MEM_HOST, C.byref(err))


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
    pu, _ = side(rng, 100, [T.Uint64], ["plain"])
    inv, uns = capi.ERR_INVALID_ARGUMENT, capi.ERR_UNSUPPORTED
    with ctx.join_table(f) as table:
        assert _code(lambda: table.probe(p + p, capi.JOIN_INNER)) == inv  # key count other than the table's
        assert _code(lambda: table.probe(pu, capi.JOIN_SEMI)) == inv      # key type other than the table's
        for kind in (4, -1):
            assert _code(lambda: table.probe(p, kind)) == inv
        out = np.zeros(100, np.uint32)
        assert _raw_probe(ctx, table.handle, p, capi.JOIN_SEMI, out.ctypes.data, out.ctypes.data, 100) == inv  # SEMI with foreign rows
        assert _raw_probe(ctx, table.handle, p, capi.JOIN_ANTI, out.ctypes.data, out.ctypes.data, 100) == inv
        assert _raw_probe(ctx, table.handle, p, capi.JOIN_INNER, out.ctypes.data, None, 100) == inv  # exactly one output
        assert _raw_probe(ctx, None, p, capi.JOIN_SEMI) == inv  # a null table
        # more than 2^30 primary rows: refused from the view alone, before any access
        huge = Column(T.Int64, values=np.zeros(1, np.uint64), value_count=2**30 + 1)
        assert _code(lambda: table.probe([huge], capi.JOIN_SEMI)) == uns
        assert _code(lambda: table.probe([huge], capi.JOIN_INNER)) == uns
    assert _code(lambda: ctx.join_table(f, nulls=2)) == inv
    assert _code(lambda: ctx.join_table([])) == inv
    assert _code(lambda: ctx.join_table(f * 9)) == inv
    exact = Column(T.Int64, values=np.zeros(1, np.uint64), value_count=2**30)  # the foreign side: fewer than 2^30 rows
    assert _code(lambda: ctx.join_table([exact])) == uns
    s = Column(T.String, values=np.zeros(100, np.uint64))
    assert _code(lambda: ctx.join_table([s])) == uns
    err = capi.Error()
    assert ctx.lib.ytgpu_join_table_destroy(None, C.byref(err)) == capi.OK
    # the one-shot call keeps refusing every kind but INNER and LEFT
    assert _code(lambda: ctx.hash_join(p, f, capi.JOIN_SEMI)) == inv


@pytest.mark.gpu
def test_gpu_host_adapter_map_join(ctx):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "map_join_ut"], stdout=subprocess.DEVNULL)
    r = subprocess.run([os.path.join(ROOT, "host", "map_join_ut")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    assert "map_join_ut: 0 failure(s)" in r.stdout
