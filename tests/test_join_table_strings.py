"""Join tables with string keys (csrc/join.cu, the string dictionary of csrc/string_column_writer.cu):
ytgpu_join_table_build_strings / _probe_strings against the dict join of test_join_table.py, and the YQL block map join
adapter with STRING keys (host/tests/map_join_strings_ut.cpp).

A key tuple is the numeric keys followed by the string keys.  The reference tuples hold the numeric payloads (or None)
followed by each string as bytes (or None), so string equality is byte equality and b"" is not NULL."""
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


def _load(name):
    spec = importlib.util.spec_from_file_location("_join_strings_" + name[:-3], os.path.join(os.path.dirname(os.path.abspath(__file__)), name))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


JT = _load("test_join_table.py")  # ref_join, tuples, side, u32, ENCODINGS, M
ROOT, NO_ROW, KINDS, KIND_IDS, RULES, RULE_IDS = JT.ROOT, JT.NO_ROW, JT.KINDS, JT.KIND_IDS, JT.RULES, JT.RULE_IDS
u32 = JT.u32
INV, UNS = capi.ERR_INVALID_ARGUMENT, capi.ERR_UNSUPPORTED

# prefixes of each other, "" next to NULL, embedded zeros and bytes >= 0x80
POOL = [b"", b"a", b"a\x00", b"ab", b"abc", b"\x00", b"\x00\x00", b"\xff", b"\x80a\xfe", b"b" * 40, b"b" * 41, b"host-17.example.org",
        b"k\x00k"]


# ------------------------------------------------------------------------------------------------- string columns
def strings_of(rng, n, pool=POOL, null_rate=0.1):
    return [None if rng.random() < null_rate else pool[i] for i in rng.integers(0, len(pool), n)]


def strcol(vals, layout="packed", rng=None):
    """A flat string column holding vals (bytes or None) -> (heap, starts, lengths, nulls or None), numpy.
    packed: one value after the other.  shuffled: the values placed in a random order, so the starts are unsorted, with
    unreferenced garbage between them, and half of them pointed at bytes already in the heap (another value's, or a
    part of one: overlapping starts).  odd: every value at an odd start."""
    rng = rng or np.random.default_rng(0)
    n = len(vals)
    starts = np.zeros(n, np.uint64)
    lengths = np.asarray([len(v or b"") for v in vals], np.uint32)
    heap = bytearray()
    if layout == "shuffled":
        for i in rng.permutation(n):
            v = vals[i] or b""
            pos = heap.find(v) if v and rng.random() < 0.5 else -1
            if pos < 0:
                heap += bytes(rng.integers(0, 256, int(rng.integers(0, 5)), dtype=np.uint8))  # garbage
                pos = len(heap)
                heap += v
            starts[i] = pos
    else:
        for i, v in enumerate(vals):
            if layout == "odd" and len(heap) % 2 == 0:
                heap += b"\x5a"
            starts[i] = len(heap)
            heap += v or b""
    heap += bytes(rng.integers(0, 256, 3, dtype=np.uint8))  # garbage after the last value
    nulls = np.asarray([v is None for v in vals], np.uint8) if any(v is None for v in vals) else None
    return np.frombuffer(bytes(heap), np.uint8).copy(), starts, lengths, nulls


def on_device(col):
    import torch
    heap, starts, lengths, nulls = col
    return (torch.from_numpy(heap).cuda(), torch.from_numpy(starts.view(np.int64)).cuda(), torch.from_numpy(lengths.view(np.int32)).cuda(),
            None if nulls is None else torch.from_numpy(nulls).cuda())


def rows_of(numeric_ref, string_vals, n):
    """Reference tuples: the numeric payloads (test_join_table.tuples) followed by the strings."""
    num = JT.tuples(numeric_ref) if numeric_ref else [()] * n
    return [tuple(t) + tuple(s[i] for s in string_vals) for i, t in enumerate(num)]


def check(table, pcols, pstr, prows, frows, kind, nulls, **kw):
    """One probe against the reference, and its count query; -> the number of rows / pairs."""
    want = JT.ref_join(prows, frows, kind, nulls)
    got = table.probe(pcols, kind, string_keys=pstr, **kw)
    if kind in (capi.JOIN_SEMI, capi.JOIN_ANTI):
        np.testing.assert_array_equal(u32(got), want)
        n = len(want)
    else:
        np.testing.assert_array_equal(u32(got[0]), want[0])
        np.testing.assert_array_equal(u32(got[1]), want[1])
        n = len(want[0])
    assert table.probe(pcols, kind, count_only=True, string_keys=pstr) == n
    return n


# ------------------------------------------------------------------------------------------------- no GPU
DECLARATIONS = r"""
#include "include/ytgpu.h"
int build_it(ytgpu_context* c, const ytgpu_column_view* k, const ytgpu_string_column* s, ytgpu_join_table** t) {
    return ytgpu_join_table_build_strings(c, k, 0, s, 1, YTGPU_JOIN_NULLS_NEVER_MATCH, t, 0);
}
int probe_it(ytgpu_context* c, const ytgpu_join_table* t, const ytgpu_column_view* k, const ytgpu_string_column* s, uint32_t* p,
             uint32_t* f, uint64_t* n) {
    return ytgpu_join_table_probe_strings(c, t, k, 1, s, 2, YTGPU_JOIN_INNER, p, f, 10, n, YTGPU_MEM_DEVICE, 0);
}
"""


def test_header_and_bindings_declare_the_string_calls():
    with tempfile.TemporaryDirectory() as d:
        src, obj = os.path.join(d, "decl.c"), os.path.join(d, "decl.o")
        open(src, "w").write(DECLARATIONS)
        subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", ROOT, "-c", src, "-o", obj])
    lib = capi.load()
    for name in ("ytgpu_join_table_build_strings", "ytgpu_join_table_probe_strings"):
        assert name in capi.EXPORTED_SYMBOLS
        assert getattr(lib, name).argtypes is not None


def test_string_column_layouts():
    rng = np.random.default_rng(3)
    vals = strings_of(rng, 300)
    for layout in ("packed", "shuffled", "odd"):
        heap, starts, lengths, nulls = strcol(vals, layout, rng)
        got = [None if nulls is not None and nulls[i] else heap[int(starts[i]):int(starts[i]) + int(lengths[i])].tobytes() for i in range(len(vals))]
        assert got == vals
        if layout == "odd":
            assert all(int(s) % 2 == 1 for s, v in zip(starts, vals) if v)


def test_map_join_strings_adapter_builds_and_refuses_cpu():
    import torch
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "map_join_strings_ut"], stdout=subprocess.DEVNULL)
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([os.path.join(ROOT, "host", "map_join_strings_ut")], capture_output=True, text=True, timeout=120)
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


SHAPES = {  # numeric key types, string key count
    "s": ([], 1),
    "ss": ([], 2),
    "i64_s": ([T.Int64], 1),
    "dbl_bool_s": ([T.Double, T.Boolean], 1),
    "8": ([T.Int64, T.Uint64, T.Double, T.Boolean], 4),
}
# 8 components drawn from the full domains would almost never match: two values per component instead
SMALL = {t: JT.DOMAINS[t][:2] for t in JT.DOMAINS}


def make_side(rng, n, shape, kinds, layout):
    types, ns = SHAPES[shape]
    wide = len(types) + ns == 8
    cols, ref = JT.side(rng, n, types, kinds, SMALL if wide else None, 0.02 if wide else 0.1) if types else ([], [])
    svals = [strings_of(rng, n, POOL[2:4] if wide else POOL, 0.02 if wide else 0.1) for _ in range(ns)]
    return cols, ref, svals, [strcol(v, layout, rng) for v in svals]


@pytest.mark.gpu
@pytest.mark.parametrize("nulls", RULES, ids=RULE_IDS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_gpu_kinds_rules_and_shapes(ctx, shape, nulls):
    """Every kind under both rules against the reference, with HOST and DEVICE inputs, both output memories, count
    queries and the capacity protocol."""
    rng = np.random.default_rng(100 * list(SHAPES).index(shape) + nulls)
    for trial, (pk, fk, layout) in enumerate([(["plain"], ["plain"], "packed"), (JT.ENCODINGS, JT.ENCODINGS[3:] + JT.ENCODINGS[:3], "shuffled"),
                                              (JT.ENCODINGS[1:], JT.ENCODINGS[5:] + JT.ENCODINGS[:5], "odd")]):
        pcols, pref, pvals, pstr = make_side(rng, 1500, shape, pk, layout)
        fcols, fref, fvals, fstr = make_side(rng, 900, shape, fk, "packed" if trial == 1 else layout)
        if trial >= 1:  # DEVICE inputs (trial 2: odd starts in a device heap)
            pcols = [JT.M.to_device(copy.copy(c)) for c in pcols]
            pstr = [on_device(s) for s in pstr]
        if trial == 2:
            fcols = [JT.M.to_device(copy.copy(c)) for c in fcols]
            fstr = [on_device(s) for s in fstr]
        prows, frows = rows_of(pref, pvals, 1500), rows_of(fref, fvals, 900)
        with ctx.join_table(fcols, nulls, string_keys=fstr) as table:
            for kind in KINDS:
                for out_mem in (capi.MEM_HOST, capi.MEM_DEVICE):
                    check(table, pcols, pstr, prows, frows, kind, nulls, out_mem=out_mem)
                count = table.probe(pcols, kind, count_only=True, string_keys=pstr)
                if kind == capi.JOIN_INNER and nulls == capi.JOIN_NULLS_EQUAL:
                    assert count > 0
                if count == 0:  # every primary tuple has a match (ANTI), or an all-NULL column under the SQL rule
                    continue
                with pytest.raises(capi.YtGpuError) as e:
                    table.probe(pcols, kind, capacity=count - 1, string_keys=pstr)
                assert e.value.code == INV and e.value.pair_count == count


@pytest.mark.gpu
@pytest.mark.parametrize("nulls", RULES, ids=RULE_IDS)
def test_gpu_values(ctx, nulls):
    """b"" against NULL, prefixes, embedded zeros, bytes >= 0x80, lengths 0..300, two 64 KiB values, and duplicate
    foreign keys listed in ascending foreign row order."""
    rng = np.random.default_rng(41)
    big_a = bytes(rng.integers(0, 256, 65536, dtype=np.uint8))
    big_b = big_a[:-1] + bytes([big_a[-1] ^ 1])
    lens = [bytes(rng.integers(0, 256, k, dtype=np.uint8)) for k in range(301)]
    pool = POOL + lens + [big_a, big_b]
    fvals = [pool[i] for i in rng.integers(0, len(pool), 1200)] + [b"", None, b"a", b"a", big_a] + lens
    pvals = pool + [None, b"a\x00\x00", b"zz", big_b[:-1]] + [pool[i] for i in rng.integers(0, len(pool), 2000)]
    for device in (False, True):
        pstr = [strcol(pvals, "shuffled", rng)]
        fstr = [strcol(fvals, "packed", rng)]
        if device:
            pstr, fstr = [on_device(pstr[0])], [on_device(fstr[0])]
        prows, frows = [(v,) for v in pvals], [(v,) for v in fvals]
        with ctx.join_table([], nulls, string_keys=fstr) as table:
            for kind in KINDS:
                check(table, [], pstr, prows, frows, kind, nulls)
            p, f = table.probe([], capi.JOIN_INNER, string_keys=pstr)
            p, f = u32(p), u32(f)
            i = pvals.index(b"a")
            assert f[p == i].tolist() == [k for k, v in enumerate(fvals) if v == b"a"]  # ascending duplicates
            i = pvals.index(b"")
            assert f[p == i].tolist() == [k for k, v in enumerate(fvals) if v == b""]  # "" matches "" only, never NULL


@pytest.mark.gpu
def test_gpu_fingerprint_collisions(ctx):
    """Distinct strings with one fingerprint and one start slot: both stay distinct keys in the table, and a primary value
    that collides with a foreign one but differs matches nothing."""
    E = _load("test_columnar_codec_edges.py")
    pairs = E.colliding_string_pairs(4)
    assert len(pairs) >= 3
    (a1, a2), (b1, b2), (c1, c2) = pairs[:3]
    for fvals in ([a1, a2, b1, None, a1, c1], [a2, a1, c1, b1, b1, a2, b"", b"x"]):
        pvals = [a1, a2, b1, b2, c1, c2, None, b"", a2]
        frows, prows = [(v,) for v in fvals], [(v,) for v in pvals]
        for nulls in RULES:
            with ctx.join_table([], nulls, string_keys=[strcol(fvals)]) as table:
                for kind in KINDS:
                    check(table, [], [strcol(pvals)], prows, frows, kind, nulls)


@pytest.mark.gpu
@pytest.mark.parametrize("nulls", RULES, ids=RULE_IDS)
def test_gpu_table_owns_its_strings(ctx, nulls):
    import torch
    rng = np.random.default_rng(51)
    pcols, pref, pvals, pstr = make_side(rng, 2000, "i64_s", ["bitmap"], "packed")
    prows = rows_of(pref, pvals, 2000)
    # DEVICE foreign strings, overwritten and freed after the build
    fcols, fref, fvals, fstr = make_side(rng, 1500, "i64_s", ["plain"], "shuffled")
    dstr = [on_device(s) for s in fstr]
    table_d = ctx.join_table(fcols, nulls, string_keys=dstr)
    for t in dstr[0]:
        if t is not None:
            t.fill_(1)
    del dstr
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    # HOST foreign strings, overwritten and deleted after the build
    hcols, href, hvals, hstr = make_side(rng, 1500, "i64_s", ["dict"], "odd")
    table_h = ctx.join_table(hcols, nulls, string_keys=hstr)
    for a in hstr[0]:
        if a is not None:
            a[...] = 0xA5 if a.dtype == np.uint8 else 3
    del hstr
    gc.collect()
    for table, rows in ((table_d, rows_of(fref, fvals, 1500)), (table_h, rows_of(href, hvals, 1500))):
        with table:
            for kind in KINDS:
                check(table, pcols, pstr, prows, rows, kind, nulls)


@pytest.mark.gpu
@pytest.mark.parametrize("nulls", RULES, ids=RULE_IDS)
def test_gpu_block_probing_equals_one_probe(ctx, nulls):
    rng = np.random.default_rng(61)
    pool = [b"%d" % k for k in range(60_000)]
    fvals = strings_of(rng, 40_000, pool, 0.05)
    pvals = strings_of(rng, 150_001, pool + [b"miss%d" % k for k in range(60_000)], 0.05)
    heap, starts, lengths, pnulls = on_device(strcol(pvals))
    sizes = [1, 31, 2049, 65537]
    sizes.append(len(pvals) - sum(sizes))
    with ctx.join_table([], nulls, string_keys=[on_device(strcol(fvals))]) as table:
        for kind in KINDS:
            whole = table.probe([], kind, string_keys=[(heap, starts, lengths, pnulls)])
            ps, fs, at = [], [], 0
            for size in sizes:
                block = (heap, starts[at:at + size], lengths[at:at + size], None if pnulls is None else pnulls[at:at + size])
                got = table.probe([], kind, string_keys=[block])
                if kind in (capi.JOIN_SEMI, capi.JOIN_ANTI):
                    ps.append(u32(got).astype(np.int64) + at)
                else:
                    ps.append(u32(got[0]).astype(np.int64) + at)
                    fs.append(u32(got[1]))
                at += size
            if kind in (capi.JOIN_SEMI, capi.JOIN_ANTI):
                np.testing.assert_array_equal(np.concatenate(ps), u32(whole).astype(np.int64))
            else:
                np.testing.assert_array_equal(np.concatenate(ps), u32(whole[0]).astype(np.int64))
                np.testing.assert_array_equal(np.concatenate(fs), u32(whole[1]))
        want = JT.ref_join([(v,) for v in pvals], [(v,) for v in fvals], capi.JOIN_SEMI, nulls)
        np.testing.assert_array_equal(u32(table.probe([], capi.JOIN_SEMI, string_keys=[(heap, starts, lengths, pnulls)])), want)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_same_pairs_as_joint_value_ids(ctx, device):
    """The pairs equal those of ytgpu_string_value_ids over foreign + primary followed by hash_join (NULL equals NULL)."""
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(71)
    F = 1100
    vals = strings_of(rng, 3000)
    heap, starts, lengths, nulls = strcol(vals, "shuffled", rng)
    ids, _ = ctx.string_value_ids(heap, starts, lengths, nulls)
    nm = nulls.astype(bool)
    fcol = Column(T.Uint64, values=ids[:F].copy(), null_bitmap=JT.M._bm(nm[:F]))
    pcol = Column(T.Uint64, values=ids[F:].copy(), null_bitmap=JT.M._bm(nm[F:]))
    fstr = [(heap, starts[:F].copy(), lengths[:F].copy(), nulls[:F].copy())]
    pstr = [(heap, starts[F:].copy(), lengths[F:].copy(), nulls[F:].copy())]
    if device:
        fstr, pstr = [on_device(fstr[0])], [on_device(pstr[0])]
    with ctx.join_table([], capi.JOIN_NULLS_EQUAL, string_keys=fstr) as table:
        for kind in (capi.JOIN_INNER, capi.JOIN_LEFT):
            a, b = table.probe([], kind, string_keys=pstr)
            c, d = ctx.hash_join([pcol], [fcol], kind)
            np.testing.assert_array_equal(u32(a), u32(c))
            np.testing.assert_array_equal(u32(b), u32(d))


def _decimal(keys):
    """Non-negative int64 keys (a CUDA tensor) -> their decimal renderings as a device string column: 12 digits per row,
    the leading zeros skipped through the starts."""
    import torch
    digits = 12
    pow10 = torch.tensor([10 ** (digits - 1 - i) for i in range(digits)], dtype=torch.int64, device=keys.device)
    d = (keys[:, None] // pow10) % 10
    heap = (d + 48).to(torch.uint8).reshape(-1).contiguous()
    nz = (d != 0).to(torch.int8)
    lead = torch.where(nz.any(1), nz.argmax(1), torch.full_like(keys, digits - 1))
    starts = (torch.arange(keys.numel(), device=keys.device) * digits + lead).contiguous()
    lengths = (digits - lead).to(torch.int32).contiguous()
    return heap, starts, lengths, None


@pytest.mark.gpu
def test_gpu_large_strings_equal_the_int64_join(ctx):
    """10^6 unique foreign strings against 2 * 10^7 primary rows: decimal renderings of int64 keys, so the pairs equal those
    of the int64 join over the same numbers; checked in full against it, and on a seeded sample against numpy."""
    import torch
    from ytsaurus_b200 import Column
    g = torch.Generator(device="cuda").manual_seed(13)
    D, N = 1_000_000, 20_000_000
    fkeys = torch.randperm(2 * D, device="cuda", generator=g)[:D].contiguous()
    pkeys = torch.randint(0, 2 * D, (N,), device="cuda", generator=g)
    fstr, pstr = _decimal(fkeys), _decimal(pkeys)
    first = fstr[0][:12].cpu().numpy().tobytes()
    assert first[12 - int(fstr[2][0]):] == str(int(fkeys[0])).encode()
    with ctx.join_table([], capi.JOIN_NULLS_NEVER_MATCH, string_keys=[fstr]) as st, \
            ctx.join_table([Column(T.Int64, values=fkeys)], capi.JOIN_NULLS_NEVER_MATCH) as it:
        for kind in (capi.JOIN_INNER, capi.JOIN_SEMI, capi.JOIN_ANTI):
            got = st.probe([], kind, string_keys=[pstr])
            want = it.probe([Column(T.Int64, values=pkeys)], kind)
            if kind == capi.JOIN_INNER:
                assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
                op, of = u32(got[0]).astype(np.int64), u32(got[1])
            else:
                assert torch.equal(got, want)
        where = np.full(2 * D, -1, np.int64)
        where[fkeys.cpu().numpy()] = np.arange(D)
        pk = pkeys.cpu().numpy()
        sample = np.unique(np.random.default_rng(14).integers(0, N, 100_000))
        hit = where[pk[sample]] >= 0
        pos = np.searchsorted(op, sample)
        assert np.array_equal(np.isin(sample, op), hit)
        np.testing.assert_array_equal(of[pos[hit]], where[pk[sample[hit]]])


def _sc(col, mem=None, row_count=None):
    """A capi.StringColumn over a numpy (heap, starts, lengths, nulls) tuple, with mem / row_count overridden."""
    heap, starts, lengths, nulls = col
    return capi.StringColumn(heap.ctypes.data if heap is not None else None, len(heap) if heap is not None else 0,
                             starts.ctypes.data if starts is not None else None, lengths.ctypes.data if lengths is not None else None,
                             nulls.ctypes.data if nulls is not None else None, len(starts if starts is not None else lengths) if row_count is None else row_count,
                             capi.MEM_HOST if mem is None else mem, 0)


def _raw_build(ctx, cols, strings, nulls=capi.JOIN_NULLS_EQUAL):
    views = (capi.ColumnView * max(len(cols), 1))(*[c.view() for c in cols])
    sarr = (capi.StringColumn * max(len(strings), 1))(*strings)
    h, err = C.c_void_p(), capi.Error()
    code = ctx.lib.ytgpu_join_table_build_strings(ctx.handle, C.cast(views, C.c_void_p), len(cols), C.cast(sarr, C.c_void_p), len(strings),
                                                  nulls, C.byref(h), C.byref(err))
    if h.value:
        ctx.lib.ytgpu_join_table_destroy(h, None)
    return code


def _raw_probe(ctx, table, cols, strings, kind=capi.JOIN_INNER):
    views = (capi.ColumnView * max(len(cols), 1))(*[c.view() for c in cols])
    sarr = (capi.StringColumn * max(len(strings), 1))(*strings)
    n, err = C.c_uint64(0), capi.Error()
    return ctx.lib.ytgpu_join_table_probe_strings(ctx.handle, table.handle, C.cast(views, C.c_void_p), len(cols), C.cast(sarr, C.c_void_p),
                                                  len(strings), kind, None, None, 0, C.byref(n), capi.MEM_HOST, C.byref(err))


@pytest.mark.gpu
def test_gpu_refusals(ctx):
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(81)
    i64, _ = JT.side(rng, 100, [T.Int64], ["plain"])
    u64, _ = JT.side(rng, 100, [T.Uint64], ["plain"])
    s = strcol(strings_of(rng, 100))
    s99 = strcol(strings_of(rng, 99))
    good = _sc(s)
    # key counts: 0 and 9 in all
    assert _raw_build(ctx, [], []) == INV
    assert _raw_build(ctx, i64 * 5, [good] * 4) == INV
    assert _raw_build(ctx, i64 * 4, [good] * 4) == capi.OK
    # string columns of another length, null starts / lengths, a null heap with bytes, a bad mem
    assert _raw_build(ctx, i64, [_sc(s99)]) == INV
    assert _raw_build(ctx, [], [good, _sc(s99)]) == INV
    assert _raw_build(ctx, [], [_sc((s[0], None, s[2], s[3]))]) == INV
    assert _raw_build(ctx, [], [_sc((s[0], s[1], None, s[3]))]) == INV
    bad_heap = _sc(s)
    bad_heap.heap = None
    assert _raw_build(ctx, [], [bad_heap]) == INV
    assert _raw_build(ctx, [], [_sc(s, mem=7)]) == INV
    # the foreign row limit, from the view
    assert _raw_build(ctx, [], [_sc(s, row_count=2**30)]) == UNS
    with ctx.join_table(i64, string_keys=[s]) as table:
        assert _raw_probe(ctx, table, i64, [good]) == capi.OK
        assert _raw_probe(ctx, table, i64, [good, good]) == INV   # string count other than the table's
        assert _raw_probe(ctx, table, i64 + i64, [good]) == INV   # numeric count
        assert _raw_probe(ctx, table, [], [good]) == INV
        assert _raw_probe(ctx, table, u64, [good]) == INV         # numeric type
        assert _raw_probe(ctx, table, i64, [_sc(s99)]) == INV     # another length
        assert _raw_probe(ctx, table, i64, [_sc((s[0], None, s[2], s[3]))]) == INV
        assert _raw_probe(ctx, table, i64, [bad_heap]) == INV
        assert _raw_probe(ctx, table, i64, [_sc(s, mem=-1)]) == INV
        huge = Column(T.Int64, values=np.zeros(1, np.uint64), value_count=2**30 + 1)
        assert _raw_probe(ctx, table, [huge], [_sc(s, row_count=2**30 + 1)]) == UNS
        assert _raw_probe(ctx, table, [huge], [_sc(s, row_count=2**30 + 1)], capi.JOIN_SEMI) == UNS
    with ctx.join_table([], string_keys=[s]) as table:
        assert _raw_probe(ctx, table, [], [_sc(s, row_count=2**30 + 1)]) == UNS
        assert _raw_probe(ctx, table, i64, [good]) == INV
        # a value outside its heap, on either side: INVALID_ARGUMENT, and the context probes correctly afterwards
        heap, starts, lengths, nulls = s
        out = starts.copy()
        k = int(np.flatnonzero(lengths > 0 if nulls is None else (lengths > 0) & (nulls == 0))[0])
        out[k] = len(heap) - int(lengths[k]) + 1
        for kind in (capi.JOIN_INNER, capi.JOIN_SEMI):
            assert _raw_probe(ctx, table, [], [_sc((heap, out, lengths, nulls))], kind) == INV
        dev = on_device((heap, out, lengths, nulls))
        with pytest.raises(capi.YtGpuError) as e:
            table.probe([], capi.JOIN_LEFT, string_keys=[dev])
        assert e.value.code == INV
        assert _raw_build(ctx, [], [_sc((heap, out, lengths, nulls))]) == INV
        with pytest.raises(capi.YtGpuError) as e:
            ctx.join_table([], string_keys=[dev])
        assert e.value.code == INV
        vals = [None if nulls is not None and nulls[i] else heap[int(starts[i]):int(starts[i]) + int(lengths[i])].tobytes() for i in range(100)]
        rows = [(v,) for v in vals]
        for kind in KINDS:
            check(table, [], [s], rows, rows, kind, capi.JOIN_NULLS_EQUAL)
    # the calls without strings keep refusing STRING column views
    assert _raw_build(ctx, [Column(T.String, values=np.zeros(100, np.uint64))], []) == UNS


@pytest.mark.gpu
def test_gpu_host_adapter_map_join_strings(ctx):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "map_join_strings_ut"], stdout=subprocess.DEVNULL)
    r = subprocess.run([os.path.join(ROOT, "host", "map_join_strings_ut")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    assert "map_join_strings_ut: 0 failure(s)" in r.stdout
