"""WHERE expressions on the GPU (ytgpu_evaluate_filter, csrc/filter.cu) against a Python model of their semantics.

The model restates include/ytgpu.h: a postfix program evaluated under Kleene logic; COMPARE is the built-in predicate's
comparison (INT64 signed, UINT64 unsigned, DOUBLE by IEEE — a NaN operand makes every op false except NE, -0.0 == +0.0 —
BOOLEAN 0 < 1, STRING unsigned bytes then the shorter first) and NULL when the value is NULL; IN is NULL for a NULL value
and otherwise "equal to some entry by the EQ rule"; STARTS_WITH compares the first len(prefix) bytes; IS_NULL /
IS_NOT_NULL are never NULL.  The model is computed column-wise with numpy for scalars and row by row for strings."""
import ctypes as C
import math
import os
import struct
import subprocess
import tempfile

import numpy as np
import pytest

import oracle
from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import EValueType as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CMP = [capi.CMP_LT, capi.CMP_LE, capi.CMP_GT, capi.CMP_GE, capi.CMP_EQ, capi.CMP_NE]
CMPOP, CMPCOLS, IN, SW, ISNULL, NOTNULL, AND, OR, NOT = (capi.FILTER_COMPARE, capi.FILTER_COMPARE_COLUMNS, capi.FILTER_IN,
                                                         capi.FILTER_STARTS_WITH, capi.FILTER_IS_NULL, capi.FILTER_IS_NOT_NULL,
                                                         capi.FILTER_AND, capi.FILTER_OR, capi.FILTER_NOT)
TRUE, FALSE, NULL = 1, 0, 2  # the model's truth values


# ------------------------------------------------------------------------------------------------- the model
def k_and(a, b):
    return np.where((a == FALSE) | (b == FALSE), FALSE, np.where((a == TRUE) & (b == TRUE), TRUE, NULL))


def k_or(a, b):
    return np.where((a == TRUE) | (b == TRUE), TRUE, np.where((a == FALSE) & (b == FALSE), FALSE, NULL))


def k_not(a):
    return np.where(a == NULL, NULL, 1 - a)


def _f(bits):
    return struct.unpack("<d", struct.pack("<Q", int(bits) & 0xFFFFFFFFFFFFFFFF))[0]


def _bits(x):
    return struct.unpack("<Q", struct.pack("<d", float(x)))[0]


def _typed(vtype, bits):
    bits = np.asarray(bits, dtype=np.uint64)
    if vtype == T.Double:
        return bits.view(np.float64)
    if vtype == T.Int64:
        return bits.view(np.int64)
    return bits


def scalar_cmp(op, vtype, a_bits, b_bits):
    """passes() of columnar.cuh, element-wise (b may be a scalar)."""
    a = _typed(vtype, a_bits)
    b = _typed(vtype, np.asarray(b_bits, dtype=np.uint64))
    with np.errstate(invalid="ignore"):
        return {capi.CMP_LT: a < b, capi.CMP_LE: a <= b, capi.CMP_GT: a > b, capi.CMP_GE: a >= b, capi.CMP_EQ: a == b,
                capi.CMP_NE: a != b}[op]


def str_cmp(op, a: bytes, b: bytes):
    c = (a > b) - (a < b)  # Python bytes order: unsigned bytes, then the shorter first
    return {capi.CMP_LT: c < 0, capi.CMP_LE: c <= 0, capi.CMP_GT: c > 0, capi.CMP_GE: c >= 0, capi.CMP_EQ: c == 0,
            capi.CMP_NE: c != 0}[op]


class Data:
    """Logical columns: scalars[i] = (vtype, bits, nulls); strings[j] = list of bytes or None."""

    def __init__(self, n, scalars=(), strings=()):
        self.n, self.scalars, self.strings = n, list(scalars), list(strings)


def model(data, program, list_values=(), consts=b""):
    """-> uint8 array of TRUE / FALSE / NULL per row."""
    n, ns = data.n, len(data.scalars)
    lv = [int(x) for x in list_values]
    stack = []

    def string_leaf(node, s):
        op, cmp, col, col2, const, length = node
        out = np.empty(n, np.uint8)
        for i in range(n):
            v = s[i]
            if op == ISNULL:
                out[i] = TRUE if v is None else FALSE
            elif op == NOTNULL:
                out[i] = FALSE if v is None else TRUE
            elif v is None:
                out[i] = NULL
            elif op == CMPOP:
                out[i] = str_cmp(cmp, v, consts[const:const + length])
            elif op == CMPCOLS:
                w = data.strings[col2 - ns][i]
                out[i] = NULL if w is None else str_cmp(cmp, v, w)
            elif op == SW:
                out[i] = v[:length] == consts[const:const + length] and len(v) >= length
            else:
                out[i] = any(v == consts[e >> 32:(e >> 32) + (e & 0xFFFFFFFF)] for e in lv[const:const + length])
        return out

    for node in program:
        op, cmp, col, col2, const, length = (tuple(node) + (0,) * 6)[:6]
        if op in (AND, OR):
            b, a = stack.pop(), stack.pop()
            stack.append(k_and(a, b) if op == AND else k_or(a, b))
            continue
        if op == NOT:
            stack.append(k_not(stack.pop()))
            continue
        if col >= ns:
            stack.append(string_leaf((op, cmp, col, col2, const, length), data.strings[col - ns]))
            continue
        vtype, bits, nulls = data.scalars[col]
        if op == ISNULL:
            r = np.where(nulls, TRUE, FALSE)
        elif op == NOTNULL:
            r = np.where(nulls, FALSE, TRUE)
        elif op == CMPOP:
            r = np.where(nulls, NULL, scalar_cmp(cmp, vtype, bits, const).astype(np.uint8))
        elif op == CMPCOLS:
            _, bits2, nulls2 = data.scalars[col2]
            r = np.where(nulls | nulls2, NULL, scalar_cmp(cmp, vtype, bits, bits2).astype(np.uint8))
        else:  # IN: equal to an entry by the EQ rule
            entries = np.asarray(lv[const:const + length], dtype=np.uint64)
            hit = np.zeros(n, bool)
            if vtype == T.Double:
                ev = entries.view(np.float64)
                ev = ev[~np.isnan(ev)]
                hit = np.isin(bits.view(np.float64), ev)  # == on doubles: -0.0 == +0.0, NaN equals nothing
            else:
                hit = np.isin(bits, entries)
            r = np.where(nulls, NULL, hit.astype(np.uint8))
        stack.append(r.astype(np.uint8))
    assert len(stack) == 1
    return stack[0].astype(np.uint8)


# ------------------------------------------------------------------------------------------------- CPU checks
def test_kleene_truth_tables_are_exhaustively_the_sql_ones():
    vals = [TRUE, FALSE, NULL]
    py = {TRUE: True, FALSE: False, NULL: None}
    for a in vals:
        assert int(k_not(np.array([a]))[0]) == {TRUE: FALSE, FALSE: TRUE, NULL: NULL}[a]
        for b in vals:
            x, y = py[a], py[b]
            want_and = False if (x is False or y is False) else (None if (x is None or y is None) else True)
            want_or = True if (x is True or y is True) else (None if (x is None or y is None) else False)
            inv = {True: TRUE, False: FALSE, None: NULL}
            assert int(k_and(np.array([a]), np.array([b]))[0]) == inv[want_and]
            assert int(k_or(np.array([a]), np.array([b]))[0]) == inv[want_or]


def test_model_comparison_rules():
    nan, nz = _bits(math.nan), _bits(-0.0)
    bits = np.array([nan, nz, _bits(0.0), _bits(1.0)], np.uint64)
    assert scalar_cmp(capi.CMP_NE, T.Double, bits, nan).tolist() == [True] * 4
    for op in CMP[:-1]:
        assert not scalar_cmp(op, T.Double, bits, nan).any()
    assert scalar_cmp(capi.CMP_EQ, T.Double, bits, _bits(0.0)).tolist() == [False, True, True, False]
    assert scalar_cmp(capi.CMP_LT, T.Int64, np.array([2**64 - 1], np.uint64), 0).tolist() == [True]
    assert scalar_cmp(capi.CMP_LT, T.Uint64, np.array([2**64 - 1], np.uint64), 0).tolist() == [False]
    assert str_cmp(capi.CMP_LT, b"ab", b"ab\0") and str_cmp(capi.CMP_GT, b"\xff", b"\x7f\xff")
    d = Data(4, [(T.Double, bits, np.array([0, 0, 0, 1], bool))])
    got = model(d, [(IN, 0, 0, 0, 0, 2)], [nan, _bits(0.0)])
    assert got.tolist() == [FALSE, TRUE, TRUE, NULL]


HEADER_PROGRAM = r"""
#include <stdio.h>
#include "include/ytgpu.h"
int main(void) {
    printf("%zu %d %d %d %d %u\n", sizeof(ytgpu_filter_node), YTGPU_FILTER_COMPARE, YTGPU_FILTER_NOT, YTGPU_FILTER_MAX_NODES,
           YTGPU_FILTER_MAX_IN_ENTRIES, (unsigned)YTGPU_FILTER_MAX_STRING_CONSTANT_BYTES);
    return 0;
}
"""


def test_header_compiles_as_c99_and_the_node_matches_the_binding():
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "f.c"), os.path.join(d, "f")
        open(src, "w").write(HEADER_PROGRAM)
        subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", ROOT, src, "-o", exe])
        out = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    assert out == [32, capi.FILTER_COMPARE, capi.FILTER_NOT, capi.FILTER_MAX_NODES, capi.FILTER_MAX_IN_ENTRIES,
                   capi.FILTER_MAX_STRING_CONSTANT_BYTES]
    assert C.sizeof(capi.FilterNode) == 32


def test_entry_point_is_declared_and_exported():
    lib = capi.load()
    assert "ytgpu_evaluate_filter" in capi.EXPORTED_SYMBOLS and hasattr(lib, "ytgpu_evaluate_filter")
    assert "ytgpu_evaluate_filter(" in open(os.path.join(ROOT, "include", "ytgpu.h")).read()


def random_program(rng, leaves, max_nodes=64, max_depth=16):
    """A random postfix program of at most max_nodes nodes and stack depth <= max_depth, built from `leaves` (node tuples)."""
    while True:
        target = int(rng.integers(1, max_nodes + 1))

        def build(budget):  # -> (postfix, depth)
            if budget <= 2 or rng.random() < 0.15:
                return [leaves[int(rng.integers(0, len(leaves)))]], 1
            if rng.random() < 0.2:
                p, d = build(budget - 1)
                return p + [(NOT,)], d
            left = int(rng.integers(1, budget - 1))
            a, da = build(left)
            b, db = build(budget - 1 - left)
            return a + b + [(AND if rng.random() < 0.5 else OR,)], max(da, 1 + db)
        prog, depth = build(target)
        if len(prog) <= max_nodes and depth <= max_depth:
            return prog


def stack_depth(prog):
    d = m = 0
    for node in prog:
        op = node[0]
        d += -1 if op in (AND, OR) else (0 if op == NOT else 1)
        m = max(m, d)
    return m


def test_random_programs_respect_the_limits():
    rng = np.random.default_rng(5)
    leaves = [(ISNULL, 0, 0, 0, 0, 0)]
    sizes = []
    for _ in range(300):
        p = random_program(rng, leaves)
        assert 1 <= len(p) <= 64 and stack_depth(p) <= 16
        sizes.append(len(p))
    assert max(sizes) >= 48


# ------------------------------------------------------------------------------------------------- inputs
def _bm(mask):
    return np.packbits(np.asarray(mask, dtype=np.uint8), bitorder="little")


def edge_values(rng, vtype, n):
    if vtype == T.Int64:
        v = rng.integers(-50, 50, n, dtype=np.int64)
        pick = rng.random(n)
        v[pick < 0.1] = np.iinfo(np.int64).min
        v[(pick >= 0.1) & (pick < 0.2)] = np.iinfo(np.int64).max
        v[(pick >= 0.2) & (pick < 0.3)] = rng.integers(-2**62, 2**62, int(((pick >= 0.2) & (pick < 0.3)).sum()))
        return v.view(np.uint64)
    if vtype == T.Uint64:
        v = rng.integers(0, 50, n, dtype=np.uint64)
        pick = rng.random(n)
        v[pick < 0.3] |= np.uint64(2**63)
        v[(pick >= 0.3) & (pick < 0.4)] = 2**64 - 1
        return v
    if vtype == T.Boolean:
        return rng.integers(0, 2, n, dtype=np.uint64)
    d = rng.integers(-5, 5, n).astype(np.float64)
    pick = rng.random(n)
    d[pick < 0.08] = np.nan
    d[(pick >= 0.08) & (pick < 0.16)] = -0.0
    d[(pick >= 0.16) & (pick < 0.24)] = 0.0
    d[(pick >= 0.24) & (pick < 0.28)] = np.inf
    d[(pick >= 0.28) & (pick < 0.32)] = -np.inf
    d[(pick >= 0.32) & (pick < 0.4)] = rng.integers(-3, 3, int(((pick >= 0.32) & (pick < 0.4)).sum())) * 5e-324  # subnormals
    return d.view(np.uint64).copy()


ENCODINGS = ["plain", "w8", "w16", "w32", "packed", "bitmap", "arrow", "dict", "rle", "dictrle", "allnull"]
BOOL_ENCODINGS = ["bits", "bits_nulls", "w8", "dict", "rle", "allnull"]


def make_column(kind, vtype, n, start, rng, nullp=0.15):
    """-> (Column, logical bits of rows [start, start + n), nulls).  Rows before the window hold other values."""
    from ytsaurus_b200 import Column
    m = start + n
    full = edge_values(rng, vtype, m)
    fnull = rng.random(m) < nullp
    if kind in ("w8", "w16", "w32", "packed"):
        width = {"w8": 8, "w16": 16, "w32": 32, "packed": 0}[kind]
        hi = 255 if width == 8 else (65535 if width == 16 else (2**32 - 1 if width == 32 else 1000))
        raw = rng.integers(0, hi, m, dtype=np.uint64, endpoint=True)
        if vtype == T.Boolean:
            raw, base, zz = raw & np.uint64(1), 0, False
        else:
            base = int(rng.integers(0, 2**64 - 1, dtype=np.uint64, endpoint=True)) if rng.random() < 0.5 else 0
            zz = bool(rng.random() < 0.5)
        x = raw + np.uint64(base)
        logical = (x >> np.uint64(1)) ^ (np.uint64(0) - (x & np.uint64(1))) if zz else x
        if width:
            vals = raw.astype({8: np.uint8, 16: np.uint16, 32: np.uint32}[width])
            col = Column(vtype, values=vals, bit_width=width, start_index=start, value_count=n, base_value=base, zigzag=zz)
        else:
            col = Column(vtype, values=oracle.bit_pack(raw, int(raw.max())), bit_width=0, start_index=start, value_count=n,
                         base_value=base, zigzag=zz)
        return col, logical[start:].copy(), np.zeros(n, bool)
    if kind == "plain":
        return Column(vtype, values=full, start_index=start, value_count=n), full[start:].copy(), np.zeros(n, bool)
    if kind in ("bitmap", "arrow"):
        bm = _bm(~fnull if kind == "arrow" else fnull)
        return (Column(vtype, values=full, start_index=start, value_count=n, null_bitmap=bm, arrow_validity=kind == "arrow"),
                full[start:].copy(), fnull[start:].copy())
    if kind in ("bits", "bits_nulls"):
        nulls = fnull if kind == "bits_nulls" else np.zeros(m, bool)
        col = Column(vtype, values=_bm(full.astype(bool)), bit_width=1, start_index=start, value_count=n,
                     null_bitmap=_bm(nulls) if kind == "bits_nulls" else None)
        return col, full[start:].copy(), nulls[start:].copy()
    if kind == "dict":
        uniq, inv = np.unique(full, return_inverse=True)
        idx = (inv.reshape(-1) + 1).astype(np.uint32)
        idx[fnull] = 0
        return Column(vtype, values=uniq, dictionary_indexes=idx, start_index=start, value_count=n), full[start:].copy(), fnull[start:].copy()
    if kind in ("rle", "dictrle"):
        # runs of 1..6 rows
        lens = rng.integers(1, 7, m)
        run_of = np.repeat(np.arange(m), lens)[:m]
        full, fnull = full[run_of], fnull[run_of]
        change = np.r_[True, (full[1:] != full[:-1]) | (fnull[1:] != fnull[:-1])]
        runs = np.flatnonzero(change)
        if kind == "rle":
            col = Column(vtype, values=full[runs].copy(), rle_indexes=runs.astype(np.uint64), null_bitmap=_bm(fnull[runs]),
                         start_index=start, value_count=n)
        else:
            uniq, inv = np.unique(full[runs], return_inverse=True)
            idx = (inv.reshape(-1) + 1).astype(np.uint32)
            idx[fnull[runs]] = 0
            col = Column(vtype, values=uniq, dictionary_indexes=idx, rle_indexes=runs.astype(np.uint64), start_index=start,
                         value_count=n)
        return col, full[start:].copy(), fnull[start:].copy()
    if kind == "allnull":
        return Column(vtype, values=None, start_index=start, value_count=n), np.zeros(n, np.uint64), np.ones(n, bool)
    raise ValueError(kind)


def to_device(col):
    import torch
    for attr in ("values", "null_bitmap", "dictionary_indexes", "rle_indexes"):
        a = getattr(col, attr)
        if a is not None:
            signed = {1: np.uint8, 2: np.int16, 4: np.int32, 8: np.int64}[a.dtype.itemsize]
            setattr(col, attr, torch.from_numpy(np.ascontiguousarray(a).view(signed)).cuda())
    return col


def strings_to_column(values, device=False, pad=0):
    """values: list of bytes / None -> (heap, starts, lengths, nulls); pad shifts the heap so starts are unaligned."""
    heap = bytearray(b"\xee" * pad)
    starts, lengths = [], []
    for v in values:
        starts.append(len(heap) if v is not None else 0)
        lengths.append(len(v) if v is not None else 0)
        if v is not None:
            heap += v
    h = np.frombuffer(bytes(heap), np.uint8).copy()
    s, ln = np.asarray(starts, np.uint64), np.asarray(lengths, np.uint32)
    nl = np.asarray([v is None for v in values], np.uint8)
    if device:
        import torch
        return (torch.from_numpy(h).cuda(), torch.from_numpy(s.view(np.int64)).cuda(), torch.from_numpy(ln.view(np.int32)).cuda(),
                torch.from_numpy(nl).cuda())
    return h, s, ln, nl


def host(x):
    import torch
    if x is None:
        return None
    if torch.is_tensor(x):
        x = x.cpu().numpy()
    return x


def check_outputs(got, want_truth, n):
    """bitmap / bytemap / rows / count against the model and against each other."""
    sel = want_truth == TRUE
    bitmap, bytemap, rows = host(got["bitmap"]), host(got["bytemap"]), host(got["rows"])
    assert got["count"] == int(sel.sum())
    assert len(bitmap) == 8 * ((n + 63) // 64)
    bits = np.unpackbits(bitmap, bitorder="little").astype(bool)
    assert np.array_equal(bits[:n], sel), np.flatnonzero(bits[:n] != sel)[:10]
    assert not bits[n:].any()
    assert np.array_equal(bytemap.astype(bool), sel) and set(np.unique(bytemap)) <= {0, 1}
    assert np.array_equal(rows.view(np.uint32), np.flatnonzero(sel).astype(np.uint32))


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


def run(ctx, data, cols, program, list_values=(), consts=b"", strings=(), device=False, **kw):
    if device:
        cols = [to_device(c) for c in cols]
    got = ctx.evaluate_filter(cols, strings, program, list_values, consts, **kw)
    want = model(data, program, list_values, consts)
    check_outputs(got, want, data.n)
    return got, want


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("vtype", [T.Int64, T.Uint64, T.Double, T.Boolean], ids=["i64", "u64", "f64", "bool"])
def test_gpu_every_leaf_over_every_encoding_and_window(ctx, vtype, device):
    rng = np.random.default_rng(int(vtype) * 7 + int(device))
    n = 300
    kinds = BOOL_ENCODINGS if vtype == T.Boolean else ENCODINGS
    for kind in kinds:
        for start in (0, 1, 3):
            col, bits, nulls = make_column(kind, vtype, n, start, rng)
            other, obits, onulls = make_column("bitmap" if vtype != T.Boolean else "bits_nulls", vtype, n, 0, rng)
            data = Data(n, [(vtype, bits, nulls), (vtype, obits, onulls)])
            pool = np.r_[bits[~nulls][:8], edge_values(rng, vtype, 4)] if (~nulls).any() else edge_values(rng, vtype, 8)
            lists = [int(x) for x in pool] + [_bits(math.nan), _bits(-0.0)] if vtype == T.Double else [int(x) for x in pool]
            programs = [[(CMPOP, op, 0, 0, int(pool[i % len(pool)]), 0)] for i, op in enumerate(CMP)]
            programs += [[(ISNULL, 0, 0)], [(NOTNULL, 0, 0)], [(IN, 0, 0, 0, 0, len(lists))],
                         [(CMPCOLS, capi.CMP_LT, 0, 1)], [(CMPCOLS, capi.CMP_EQ, 1, 0)], [(CMPCOLS, capi.CMP_NE, 0, 1)]]
            for prog in programs:
                cols = [col, other]
                if device:
                    import copy
                    cols = [copy.copy(c) for c in cols]
                run(ctx, data, cols, prog, lists, device=device)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_random_programs_at_every_size(ctx, device):
    import copy
    rng = np.random.default_rng(17 + int(device))
    for n in (0, 1, 31, 32, 33, 63, 64, 65, 4097):
        for rep in range(6):
            specs = [("plain", T.Int64), ("rle", T.Uint64), ("bitmap", T.Double), ("bits_nulls", T.Boolean), ("dict", T.Int64),
                     ("packed", T.Int64), ("arrow", T.Double)]
            cols, scal = [], []
            for kind, vt in specs:
                c, b, nl = make_column(kind, vt, n, int(rng.integers(1, 4)), rng)
                cols.append(c)
                scal.append((vt, b, nl))
            words = [b"", b"a", b"ab", b"ab\0", b"b", b"https://x", b"http://y"]
            svals = [None if rng.random() < 0.2 else words[int(rng.integers(0, len(words)))] for _ in range(n)]
            consts = b"ab" + b"https://" + b"b"
            head = [int(x) for x in scal[0][1][:5]]
            lists = head + [7] * (5 - len(head)) + [(0 << 32) | 2, (10 << 32) | 1]
            data = Data(n, scal, [svals])
            leaves = []
            for ci, (vt, b, _) in enumerate(scal):
                const = int(b[int(rng.integers(0, n))]) if n else 0
                leaves += [(CMPOP, int(rng.choice(CMP)), ci, 0, const, 0), (ISNULL, 0, ci), (NOTNULL, 0, ci)]
            leaves += [(IN, 0, 0, 0, 0, 5), (CMPCOLS, capi.CMP_LE, 2, 6), (CMPCOLS, capi.CMP_NE, 0, 4),
                       (SW, 0, 7, 0, 2, 8), (CMPOP, capi.CMP_GE, 7, 0, 0, 2), (IN, 0, 7, 0, 5, 2), (ISNULL, 0, 7)]
            prog = random_program(rng, leaves)
            strings = [strings_to_column(svals, device)]
            run(ctx, data, [copy.copy(c) for c in cols], prog, lists, consts, strings, device=device)


@pytest.mark.gpu
def test_gpu_random_programs_ten_million_rows(ctx):
    import copy
    rng = np.random.default_rng(29)
    n = 10**7
    cols, scal = [], []
    for kind, vt in [("plain", T.Int64), ("rle", T.Uint64), ("bitmap", T.Double), ("bits_nulls", T.Boolean), ("dict", T.Int64)]:
        c, b, nl = make_column(kind, vt, n, 1, rng)
        cols.append(c)
        scal.append((vt, b, nl))
    data = Data(n, scal)
    leaves = []
    for ci, (vt, b, _) in enumerate(scal):
        leaves += [(CMPOP, int(rng.choice(CMP)), ci, 0, int(b[int(rng.integers(0, n))]), 0), (ISNULL, 0, ci)]
    leaves += [(IN, 0, 0, 0, 0, 16), (CMPCOLS, capi.CMP_LT, 0, 4)]
    lists = [int(x) for x in scal[0][1][:16]]
    for device in (False, True):
        prog = random_program(rng, leaves)
        run(ctx, data, [copy.copy(c) for c in cols], prog, lists, device=device)


def _check_same_groupby(a, b):
    assert len(a["count"]) == len(b["count"])
    for key in ("count", "first_row"):
        assert np.array_equal(host(a[key]), host(b[key]))
    for xs, ys in ((a["keys"], b["keys"]), (a["key_null"], b["key_null"]), (a["values"], b["values"]), (a["value_null"], b["value_null"])):
        for x, y in zip(xs, ys):
            assert np.array_equal(host(x), host(y))


def bitmap_column(bitmap, n):
    from ytsaurus_b200 import Column
    return Column(T.Boolean, values=bitmap, bit_width=1, value_count=n)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_one_compare_node_equals_the_builtin_predicate(ctx, device):
    import copy
    rng = np.random.default_rng(41 + int(device))
    n = 5000
    keys, _, _ = make_column("plain", T.Int64, n, 0, rng)
    keys.values = (keys.values % np.uint64(37)).astype(np.uint64)
    for vtype in (T.Int64, T.Uint64, T.Double, T.Boolean):
        kind = "bits_nulls" if vtype == T.Boolean else "bitmap"
        col, bits, nulls = make_column(kind, vtype, n, 0, rng)
        agg_col, _, _ = make_column("bitmap", T.Int64, n, 0, rng)
        aggs = [(capi.AGG_SUM, 1), (capi.AGG_MIN, 1), (capi.AGG_MAX, 0), (capi.AGG_COUNT, 0), (capi.AGG_FIRST, 0)]
        consts = [int(bits[~nulls][0]), int(edge_values(rng, vtype, 1)[0])] + ([_bits(math.nan)] if vtype == T.Double else [])
        for op in CMP:
            for const in consts:
                kc, vc, ac = copy.copy(keys), copy.copy(col), copy.copy(agg_col)
                if device:
                    kc, vc, ac = to_device(kc), to_device(vc), to_device(ac)
                want = ctx.scan_filter_groupby_multi([kc], [vc, ac], aggs, predicate=(op, const), predicate_column=0)
                f = ctx.evaluate_filter([vc], (), [(CMPOP, op, 0, 0, const, 0)], want_bytemap=False, want_rows=False)
                truth = model(Data(n, [(vtype, bits, nulls)]), [(CMPOP, op, 0, 0, const, 0)])
                assert f["count"] == int((truth == TRUE).sum())
                got = ctx.scan_filter_groupby_multi([kc], [vc, ac, bitmap_column(f["bitmap"], n)], aggs,
                                                    predicate=(capi.CMP_EQ, 1), predicate_column=2)
                _check_same_groupby(got, want)


def _string_groups_model(keys, sel, svals, aggs_cols):
    """First-seen groups of the selected rows -> (keys, counts, first rows, per string aggregate (op) the result row / count)."""
    order, members = [], {}
    for i in np.flatnonzero(sel):
        k = int(keys[i])
        if k not in members:
            members[k] = []
            order.append(k)
        members[k].append(i)
    out = []
    for op in aggs_cols:
        col = []
        for k in order:
            rows = [i for i in members[k] if svals[i] is not None]
            if op == capi.AGG_COUNT:
                col.append(len(rows))
            elif not rows:
                col.append(None)
            elif op == capi.AGG_MIN:
                col.append(min(rows, key=lambda i: (svals[i], i)))
            elif op == capi.AGG_MAX:
                col.append(min(rows, key=lambda i: (_neg(svals[i]), i)))
            else:
                col.append(rows[0])
        out.append(col)
    return order, [len(members[k]) for k in order], [members[k][0] for k in order], out


class _neg:
    def __init__(self, b):
        self.b = b

    def __lt__(self, o):
        return self.b > o.b

    def __eq__(self, o):
        return self.b == o.b


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_groupby_through_the_bitmap_matches_the_oracle(ctx, device):
    import copy
    rng = np.random.default_rng(53 + int(device))
    n = 20011
    kcol, kbits, knull = make_column("bitmap", T.Int64, n, 0, rng)
    kbits = kbits % np.uint64(101)
    kcol.values = kcol.values % np.uint64(101)
    vals = []
    cols = []
    for kind, vt in [("plain", T.Int64), ("bitmap", T.Uint64), ("bitmap", T.Double), ("rle", T.Int64)]:
        c, b, nl = make_column(kind, vt, n, 0, rng)
        cols.append(c)
        vals.append((vt, b, nl))
    words = [b"", b"ab", b"ab\0", b"https://a", b"https://b", b"http://c", b"zz"]
    svals = [None if rng.random() < 0.1 else words[int(rng.integers(0, len(words)))] for _ in range(n)]
    consts = b"https://"
    prog = [(CMPOP, capi.CMP_GE, 0, 0, (-20) & (2**64 - 1), 0), (CMPOP, capi.CMP_LT, 0, 0, 20, 0), (AND,),
            (IN, 0, 3, 0, 0, 4), (AND,), (CMPOP, capi.CMP_LT, 2, 0, _bits(1.5), 0), (ISNULL, 0, 1), (OR,), (AND,),
            (SW, 0, 4, 0, 0, 8), (NOT,), (OR,)]
    lists = [int(x) for x in vals[3][1][:4]]
    data = Data(n, vals, [svals])
    truth = model(data, prog, lists, consts)
    sel = truth == TRUE
    strings = [strings_to_column(svals, device)]
    cdev = [copy.copy(c) for c in cols]
    kc = copy.copy(kcol)
    if device:
        cdev, kc = [to_device(c) for c in cdev], to_device(kc)
    f = ctx.evaluate_filter(cdev, strings, prog, lists, consts)
    check_outputs(f, truth, n)
    vcols = cdev + [bitmap_column(f["bitmap"], n)]
    aggs = [(capi.AGG_SUM, 0), (capi.AGG_MIN, 1), (capi.AGG_MAX, 2), (capi.AGG_COUNT, 2), (capi.AGG_FIRST, 3), (capi.AGG_SUM, 3),
            (capi.AGG_ARGMIN, 0, 1)]
    got = ctx.scan_filter_groupby_multi([kc], vcols, aggs, predicate=(capi.CMP_EQ, 1), predicate_column=4)
    want = oracle.groupby_multi([kbits], [knull.astype(np.uint8)], [v[1] for v in vals], [v[2].astype(np.uint8) for v in vals],
                                [v[0] for v in vals], aggs, filt=sel.astype(np.uint8), style=oracle.MINMAX_YQL)  # data with NaN
    assert np.array_equal(host(got["count"]), want["count"]) and np.array_equal(host(got["first_row"]), want["first_row"])
    for a in range(len(aggs)):
        assert np.array_equal(host(got["value_null"][a]), want["value_null"][a])
        gv = host(got["values"][a]).view(np.uint64)
        wv = want["values"][a].view(np.uint64)
        live = want["value_null"][a] == 0
        if aggs[a][0] == capi.AGG_MAX and vals[aggs[a][1]][0] == T.Double:
            g, w = gv[live].view(np.float64), wv[live].view(np.float64)  # NaN the largest; a ±0 result compared by value
            assert np.array_equal(np.isnan(g), np.isnan(w)) and np.array_equal(g[~np.isnan(g)], w[~np.isnan(w)]), a
        else:
            assert np.array_equal(gv[live], wv[live]), a
    assert np.array_equal(host(got["keys"][0]).view(np.uint64)[host(got["key_null"][0]) == 0],
                          want["keys"][0][want["key_null"][0] == 0])

    # string aggregates through the _strings entry point
    saggs = [(capi.AGG_MIN, 5), (capi.AGG_MAX, 5), (capi.AGG_COUNT, 5), (capi.AGG_FIRST, 5)]
    got = ctx.scan_filter_groupby_multi([kc], vcols, saggs, predicate=(capi.CMP_EQ, 1), predicate_column=4, string_columns=strings)
    eff_keys = np.where(knull, np.uint64(2**64 - 1), kbits)  # NULL key: its own group
    order, counts, firsts, res = _string_groups_model(eff_keys, sel, svals, [a[0] for a in saggs])
    assert host(got["count"]).tolist() == counts and host(got["first_row"]).tolist() == firsts
    for a in range(len(saggs)):
        gv, gn = host(got["values"][a]).view(np.uint64).tolist(), host(got["value_null"][a]).tolist()
        for g, want_v in enumerate(res[a]):
            assert (gn[g] == 1) == (want_v is None)
            if want_v is not None:
                assert gv[g] == want_v, (a, g)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_string_edges(ctx, device):
    rng = np.random.default_rng(61)
    long_a = b"x" * 1000 + b"a"
    long_b = b"x" * 1000 + b"b"
    words = [b"", b"\0", b"a\0b", b"ab", b"ab\0", b"abc", b"\xff", b"\x7f\xff", long_a, long_b, b"x" * 1000, b"https://q"]
    n = 777
    svals = [None if rng.random() < 0.1 else words[int(rng.integers(0, len(words)))] for _ in range(n)]
    svals2 = [None if rng.random() < 0.1 else words[int(rng.integers(0, len(words)))] for _ in range(n)]
    # constants: the words, then padding past the 4096-byte shared-memory stage, then the words again
    consts = b"".join(words)
    offs = np.cumsum([0] + [len(w) for w in words])
    far = len(consts) + 5000
    consts = consts + b"\0" * 5000 + b"".join(words)
    entries = [(int(offs[i]) << 32) | len(w) for i, w in enumerate(words)]
    far_entries = [((far + int(offs[i])) << 32) | len(w) for i, w in enumerate(words)]
    data = Data(n, [], [svals, svals2])
    strings = [strings_to_column(svals, device, pad=3), strings_to_column(svals2, device, pad=1)]
    ok = 0
    for i, w in enumerate(words):
        for base in (int(offs[i]), far + int(offs[i])):
            for op in CMP:
                run(ctx, data, [], [(CMPOP, op, 0, 0, base, len(w))], (), consts, strings)
            run(ctx, data, [], [(SW, 0, 0, 0, base, len(w))], (), consts, strings)  # full-length and empty prefixes included
            ok += 1
    for op in CMP:
        run(ctx, data, [], [(CMPCOLS, op, 0, 1)], (), consts, strings)
    # IN lists: duplicates, below and above the shared-memory stage (1024 entries)
    dup = entries + entries[:5] + far_entries
    run(ctx, data, [], [(IN, 0, 0, 0, 0, len(dup))], dup, consts, strings)
    big = [entries[j % len(entries)] for j in range(3000)] + far_entries
    run(ctx, data, [], [(IN, 0, 1, 0, 0, len(big))], big, consts, strings)
    run(ctx, data, [], [(IN, 0, 0, 0, 0, 0)], big, consts, strings)  # an empty list: FALSE for every non-NULL value
    run(ctx, data, [], [(ISNULL, 0, 0), (NOTNULL, 0, 1), (AND,)], (), consts, strings)
    assert ok == 2 * len(words)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_scalar_in_lists_around_the_staging_size(ctx, device):
    import copy
    rng = np.random.default_rng(67)
    n = 5000
    for vtype in (T.Int64, T.Uint64, T.Double):
        col, bits, nulls = make_column("bitmap", vtype, n, 2, rng)
        data = Data(n, [(vtype, bits, nulls)])
        for size in (1, 1023, 1024, 1025, 3000):
            lst = [int(x) for x in rng.choice(bits, size)]
            lst[: min(size, 3)] = lst[:1] * min(size, 3)  # duplicates
            run(ctx, data, [copy.copy(col)], [(IN, 0, 0, 0, 0, size)], lst, device=device)
        # the second IN list of a call lies past the staged entries
        lst = [int(x) for x in edge_values(rng, vtype, 2000)] + [int(x) for x in bits[:7]]
        run(ctx, data, [copy.copy(col)], [(IN, 0, 0, 0, 0, 5), (IN, 0, 0, 0, 2000, 7), (OR,)], lst, device=device)


def _code(fn):
    try:
        fn()
    except capi.YtGpuError as e:
        return e.code
    return capi.OK


@pytest.mark.gpu
def test_gpu_limits_and_errors(ctx):
    import copy

    import torch

    from ytsaurus_b200 import Column
    rng = np.random.default_rng(71)
    n = 100
    col, bits, nulls = make_column("bitmap", T.Int64, n, 0, rng)
    ucol, _, _ = make_column("plain", T.Uint64, n, 0, rng)
    svals = [b"abc", None] * (n // 2)
    s = strings_to_column(svals)
    inv = capi.ERR_INVALID_ARGUMENT

    def ev(prog, lists=(), consts=b"", cols=None, strings=(s,), **kw):
        return lambda: ctx.evaluate_filter([copy.copy(c) for c in (cols or [col, ucol])], strings, prog, lists, consts, **kw)
    leaf = (ISNULL, 0, 0)
    # 64 nodes / 65 nodes
    chain = [leaf] + [leaf, (AND,)] * 31 + [(NOT,)]
    assert len(chain) == 64 and _code(ev(chain)) == capi.OK
    assert _code(ev(chain + [(NOT,)])) == inv
    # depth 16 / 17
    deep = [leaf] * 16 + [(AND,)] * 15
    assert _code(ev(deep)) == capi.OK
    assert _code(ev([leaf] * 17 + [(AND,)] * 16)) == inv
    # IN entries: 65536 / 65537 over all IN nodes of a call
    lst = list(range(65537))
    assert _code(ev([(IN, 0, 0, 0, 0, 32768), (IN, 0, 0, 0, 32768, 32768), (OR,)], lst)) == capi.OK
    assert _code(ev([(IN, 0, 0, 0, 0, 32768), (IN, 0, 0, 0, 32768, 32769), (OR,)], lst)) == inv
    # string constants: 1 MiB / 1 MiB + 1
    mib = 1 << 20
    assert _code(ev([(SW, 0, 2, 0, mib - 3, 3)], (), b"\0" * (mib - 3) + b"abc")) == capi.OK
    assert _code(ev([(SW, 0, 2, 0, 0, 3)], (), b"abc" + b"\0" * (mib - 2))) == inv
    # malformed programs
    assert _code(ev([(AND,)])) == inv                                  # underflow
    assert _code(ev([leaf, (NOT,), leaf, (AND,), (AND,)])) == inv      # underflow later
    assert _code(ev([leaf, leaf])) == inv                              # two values left
    assert _code(ev([(10, 0, 0)])) == inv and _code(ev([(0, 0, 0)])) == inv   # unknown op
    assert _code(ev([(CMPOP, 0, 0, 0, 1, 0)])) == inv and _code(ev([(CMPOP, 7, 0, 0, 1, 0)])) == inv  # unknown cmp
    assert _code(ev([(CMPOP, capi.CMP_NE, 0, 0, 1, 0)])) == capi.OK
    assert _code(ev([(ISNULL, 0, 3)])) == inv and _code(ev([(ISNULL, 0, -1)])) == inv and _code(ev([(ISNULL, 0, 2)])) == capi.OK
    assert _code(ev([(CMPCOLS, capi.CMP_EQ, 0, 3)])) == inv
    # STARTS_WITH / a string constant on a scalar column; COMPARE_COLUMNS over different types
    assert _code(ev([(SW, 0, 0, 0, 0, 1)], (), b"a")) == inv
    assert _code(ev([(CMPOP, capi.CMP_EQ, 0, 0, 0, 1)], (), b"a")) == inv
    assert _code(ev([(CMPCOLS, capi.CMP_EQ, 0, 1)])) == inv
    assert _code(ev([(CMPCOLS, capi.CMP_EQ, 0, 2)])) == inv
    assert _code(ev([(CMPCOLS, capi.CMP_EQ, 0, 0)])) == capi.OK
    # constant and list ranges
    assert _code(ev([(CMPOP, capi.CMP_EQ, 2, 0, 1, 3)], (), b"abcd")) == capi.OK
    assert _code(ev([(CMPOP, capi.CMP_EQ, 2, 0, 2, 3)], (), b"abcd")) == inv
    assert _code(ev([(IN, 0, 0, 0, 1, 3)], [1, 2, 3, 4])) == capi.OK
    assert _code(ev([(IN, 0, 0, 0, 2, 3)], [1, 2, 3, 4])) == inv
    assert _code(ev([(IN, 0, 2, 0, 0, 1)], [(1 << 32) | 3], b"abcd")) == capi.OK
    assert _code(ev([(IN, 0, 2, 0, 0, 1)], [(2 << 32) | 3], b"abcd")) == inv
    # unsupported column type
    scol = Column(T.String, values=np.zeros(n, np.uint64), value_count=n)
    assert _code(ev([(ISNULL, 0, 0)], cols=[scol])) == capi.ERR_UNSUPPORTED
    # row counts: equal / different
    short, _, _ = make_column("plain", T.Int64, n - 1, 0, rng)
    assert _code(ev([leaf], cols=[col, short])) == inv
    assert _code(ev([leaf], strings=(strings_to_column(svals[:-1]),))) == inv
    # rows_capacity: the selected count / one less (the count is still reported)
    want = int((~nulls).sum())
    assert ctx.evaluate_filter([copy.copy(col)], (), [(NOTNULL, 0, 0)], rows_capacity=want)["count"] == want
    with pytest.raises(capi.YtGpuError) as e:
        ctx.evaluate_filter([copy.copy(col)], (), [(NOTNULL, 0, 0)], rows_capacity=want - 1)
    assert e.value.code == inv and e.value.selected == want
    # a string outside its heap (host and device)
    for device in (False, True):
        h, st, ln, nl = strings_to_column([b"abc"] * n)
        st = st.copy()
        st[n // 2] = len(h) - 1  # 3 bytes from the last byte: leaves the heap
        bad = (h, st, ln, nl)
        if device:
            bad = tuple(torch.from_numpy(x.view({1: np.uint8, 4: np.int32, 8: np.int64}[x.dtype.itemsize])).cuda() for x in bad)
        assert _code(ev([(NOTNULL, 0, 2)], strings=(bad,))) == inv
        st[n // 2] = len(h) - 3  # ends on the last byte
        good = (h, st, ln, nl)
        assert _code(ev([(NOTNULL, 0, 2)], strings=(good,))) == capi.OK
    # fewer than 2^32 rows: an all-NULL DEVICE column (no data) of 2^32 - 1 rows / 2^32 rows
    r = _device_all_null_filter(ctx, 2**32 - 1)
    assert r == (capi.OK, 0)
    assert _device_all_null_filter(ctx, 2**32)[0] == inv


def _device_all_null_filter(ctx, n):
    """IS_NOT_NULL over an all-NULL DEVICE column of n rows, bitmap output only -> (code, selected)."""
    import torch
    v = capi.ColumnView()
    v.value_count, v.value_type, v.has_values, v.bit_width, v.mem = n, T.Int64, 0, 64, capi.MEM_DEVICE
    words = (n + 63) // 64
    bitmap = torch.empty(words * 8 if n < 2**32 else 8, dtype=torch.uint8, device="cuda")
    node = capi.FilterNode(NOTNULL, 0, 0, 0, 0, 0, 0)
    sel = C.c_uint64(123)
    err = capi.Error()
    code = ctx.lib.ytgpu_evaluate_filter(ctx.handle, C.cast(C.pointer(v), C.c_void_p), 1, None, 0, C.cast(C.pointer(node), C.c_void_p), 1,
                                         None, 0, None, 0, bitmap.data_ptr(), None, None, 0, C.byref(sel), capi.MEM_DEVICE, C.byref(err))
    if code == capi.OK:
        torch.cuda.synchronize()
        assert int(bitmap.count_nonzero()) == 0
    return code, int(sel.value)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_launch_count(ctx, device):
    import copy
    rng = np.random.default_rng(73)
    n = 10000
    col, bits, nulls = make_column("rle", T.Int64, n, 1, rng)
    prog = [(CMPOP, capi.CMP_GT, 0, 0, 0, 0), (ISNULL, 0, 0), (OR,)]
    c = to_device(copy.copy(col)) if device else copy.copy(col)
    before = ctx.launch_count()
    got = ctx.evaluate_filter([c], (), prog, want_rows=False)
    assert ctx.launch_count() - before == 1
    assert got["rows"] is None and got["count"] == int((model(Data(n, [(T.Int64, bits, nulls)]), prog) == TRUE).sum())
    before = ctx.launch_count()
    ctx.evaluate_filter([c], (), prog, want_rows=True)
    assert ctx.launch_count() - before == 5


def test_host_adapter_builds_and_refuses_cpu():
    import torch
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "filter_ut"], stdout=subprocess.DEVNULL)
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([os.path.join(ROOT, "host", "filter_ut")], capture_output=True, text=True, timeout=120)
    assert r.returncode == 100 and "no CPU fallback" in r.stderr


@pytest.mark.gpu
def test_gpu_host_adapter_where_expression():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "filter_ut"], stdout=subprocess.DEVNULL)
    r = subprocess.run([os.path.join(ROOT, "host", "filter_ut")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
