"""Computed string columns on the GPU (ytgpu_evaluate_expression_strings, csrc/expression.cu) against a pure-Python model.

The model restates include/ytgpu.h: CONCAT joins two strings, LOWER / UPPER map ASCII letters and keep every other byte,
and refuse (UNSUPPORTED) a byte >= 0x80 in an evaluated operand; a NULL operand makes CONCAT / LOWER / UPPER NULL, IF_NULL
takes its second operand when the first is NULL; FARM_HASH(k) folds the k values' fingerprints from 0xdeadc0de with
Fingerprint(uint128) and xors k, never NULL; rows outside the selection are NULL and never evaluated.  Strings are
compared byte for byte: heap, starts, lengths and the NULL bytemap."""
import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle
from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import EValueType as T
from ytsaurus_b200.rowset import U64, make_rowset

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
(COL, CONST, ADD, MOD, BAND, IFNULL, CONCAT, LOWER, UPPER, FARM) = (
    capi.EXPR_COLUMN, capi.EXPR_CONSTANT, capi.EXPR_ADD, capi.EXPR_MOD, capi.EXPR_BIT_AND, capi.EXPR_IF_NULL, capi.EXPR_CONCAT,
    capi.EXPR_LOWER, capi.EXPR_UPPER, capi.EXPR_FARM_HASH)
I64, U64T, DBL, BOOL, STR = int(T.Int64), int(T.Uint64), int(T.Double), int(T.Boolean), int(T.String)
M64 = (1 << 64) - 1
K_MUL = 0x9DDFEA08EB382D69


# ------------------------------------------------------------------------------------------------- the model
class NonAscii(Exception):
    pass


def fp_u64(x):
    """FarmHash Fingerprint(uint64)."""
    b = (x * K_MUL) & M64
    b ^= b >> 44
    b = (b * K_MUL) & M64
    b ^= b >> 41
    return (b * K_MUL) & M64


def fp_u128(lo, hi):
    """FarmHash Fingerprint(uint128) (Hash128to64)."""
    a = ((lo ^ hi) * K_MUL) & M64
    a ^= a >> 47
    b = ((hi ^ a) * K_MUL) & M64
    b ^= b >> 44
    b = (b * K_MUL) & M64
    b ^= b >> 41
    return (b * K_MUL) & M64


_bytes_fp_cache = {}


def fp_bytes(s):
    """Fingerprint64 of a string's bytes, from the oracle's value fingerprint of a one-string row."""
    if s not in _bytes_fp_cache:
        rs = make_rowset([[s]])
        _bytes_fp_cache[s] = int(oracle.value_fingerprints(rs.values, rs.heap)[0])
    return _bytes_fp_cache[s]


def farm_hash(vals):
    """vals: (type, value) with value None for NULL, bytes for STRING, the 64-bit pattern otherwise (BOOLEAN 0 / 1)."""
    h = 0xDEADC0DE
    for t, v in vals:
        f = fp_u64(0) if v is None else (fp_bytes(v) if t == STR else fp_u64(v))
        h = fp_u128(h, f)
    return h ^ len(vals)


def case_map(s, op):
    if any(b >= 0x80 for b in s):
        raise NonAscii()
    return s.lower() if op == LOWER else s.upper()  # bytes.lower / upper map ASCII letters only


def eval_row(prog, row, consts):
    """row: per input column (type, value); -> (type, value)."""
    st = []
    for node in prog:
        op, column, vtype, constant = (tuple(node) + (0, 0, 0, 0))[:4]
        if op == COL:
            st.append(row[column])
        elif op == CONST:
            st.append((STR, consts[constant >> 32:(constant >> 32) + (constant & 0xFFFFFFFF)]) if vtype == STR else (vtype, constant))
        elif op in (LOWER, UPPER):
            t, v = st.pop()
            st.append((t, None if v is None else case_map(v, op)))
        elif op == FARM:
            vals = st[len(st) - column:]
            del st[len(st) - column:]
            st.append((U64T, farm_hash(vals)))
        else:
            (ta, a), (tb, b) = st[-2], st[-1]
            del st[-2:]
            if op == IFNULL:
                st.append((ta, b if a is None else a))
            elif a is None or b is None:
                st.append((ta, None))
            elif op == CONCAT:
                st.append((STR, a + b))
            elif op == MOD:
                st.append((ta, a % b))
            elif op == ADD:
                st.append((ta, (a + b) & M64))
            elif op == BAND:
                st.append((ta, a & b))
            else:
                raise AssertionError(op)
    assert len(st) == 1
    return st[0]


def model(prog, rows, consts, selection=None):
    """-> ('error', 'nonascii') or (type, list of values)."""
    out, t = [], None
    for i, row in enumerate(rows):
        if selection is not None and not selection[i]:
            out.append(None)
            continue
        try:
            t, v = eval_row(prog, row, consts)
        except NonAscii:
            return "error", "nonascii"
        out.append(v)
    return t, out


def flat_strings(values):
    """A result in the GPU's layout: heap, starts, lengths, null bytemap."""
    lengths = np.array([0 if v is None else len(v) for v in values], np.uint32)
    starts = np.zeros(len(values), np.uint64)
    if len(values):
        starts[1:] = np.cumsum(lengths[:-1], dtype=np.uint64)
    heap = b"".join(v for v in values if v is not None)
    return heap, starts, lengths, np.array([v is None for v in values], np.uint8)


# ------------------------------------------------------------------------------------------------- programs
def constant(consts, s):
    """Appends s to the constants buffer (a bytearray) -> the node's constant."""
    off = len(consts)
    consts += s
    return (off << 32) | len(s)


WORDS = [b"", b"/", b"x", b"Abc", b"MiXeD-Case_09", b"none", b"Z" * 40]


def random_program(rng, string_cols, numeric_cols, consts, max_nodes=64):
    """A random well-typed program over string columns (indexes in string_cols) and numeric columns (index, type) within every
    limit: at most 64 nodes, a stack of 16, 16 pieces, FARM_HASH of 1..16 operands whose strings are leaves, constants or
    IF_NULL of those.  The result is a STRING or, through FARM_HASH, a UINT64 that may be reduced further."""
    def plain(budget):  # -> (postfix, pieces)
        r = rng.random()
        if budget >= 3 and r < 0.25:
            a, pa = plain((budget - 1) // 2)
            b, pb = plain((budget - 1) // 2)
            return a + b + [(IFNULL, 0, STR)], max(pa, pb)
        if string_cols and r < 0.75:
            return [(COL, int(rng.choice(string_cols)))], 1
        return [(CONST, 0, STR, constant(consts, WORDS[int(rng.integers(0, len(WORDS)))]))], 1

    def string(budget, pieces):  # -> (postfix, pieces), pieces <= the bound
        r = rng.random()
        if budget >= 3 and pieces >= 2 and r < 0.35:
            left = int(rng.integers(1, pieces))
            a, pa = string((budget - 1) // 2, left)
            b, pb = string((budget - 1) // 2, pieces - pa)
            return a + b + [(CONCAT,)], pa + pb
        if budget >= 2 and r < 0.55:
            a, pa = string(budget - 1, pieces)
            return a + [(int(rng.choice([LOWER, UPPER])),)], pa
        if budget >= 3 and r < 0.7:
            a, pa = string((budget - 1) // 2, pieces)
            b, pb = string((budget - 1) // 2, pieces)
            return a + b + [(IFNULL, 0, STR)], max(pa, pb)
        return plain(min(budget, 3))

    if rng.random() < 0.6 or not (string_cols or numeric_cols):
        while True:
            prog, _ = string(int(rng.integers(1, max_nodes + 1)), int(rng.integers(1, 17)))
            if len(prog) <= max_nodes and stack_depth(prog) <= 16 and pieces_bound(prog, string_cols) <= 16:
                return prog
    while True:
        k = int(rng.integers(1, 17))
        prog = []
        for _ in range(k):
            if numeric_cols and rng.random() < 0.4:
                prog.append((COL, numeric_cols[int(rng.integers(0, len(numeric_cols)))][0]))
            else:
                prog += plain(3)[0]
        prog.append((FARM, k))
        if rng.random() < 0.6:
            prog += [(CONST, 0, U64T, int(rng.choice([1, 4, 64, 100, 1 << 40]))), (int(rng.choice([MOD, BAND, ADD])),)]
        if len(prog) <= max_nodes and stack_depth(prog) <= 16:
            return prog


def stack_depth(prog):
    d = m = 0
    for node in prog:
        op = node[0]
        d += 1 if op in (COL, CONST) else (0 if op in (LOWER, UPPER) else (1 - node[1] if op == FARM else -1))
        m = max(m, d)
    return m


def pieces_bound(prog, string_cols):
    """The check's piece bound: a STRING leaf or constant is 1, CONCAT sums, IF_NULL takes the larger, FARM_HASH and the
    numeric ops leave none."""
    st, m = [], 0
    for node in prog:
        op = node[0]
        if op == COL:
            st.append(1 if node[1] in string_cols else 0)
        elif op == CONST:
            st.append(1 if node[2] == STR else 0)
        elif op == FARM:
            del st[len(st) - node[1]:]
            st.append(0)
        elif op in (CONCAT, IFNULL):
            b = st.pop()
            st[-1] = st[-1] + b if op == CONCAT else max(st[-1], b)
        elif op in (MOD, ADD, BAND):
            st.pop()
            st[-1] = 0
        m = max(m, sum(st))
    return m


# ------------------------------------------------------------------------------------------------- CPU
def test_model_hand_written_cases():
    c = bytearray()
    rows = [[(STR, b"Hello"), (STR, b"World")], [(STR, None), (STR, b"x")], [(STR, b"AbC-\x7f"), (STR, None)]]
    sep = constant(c, b"/")
    none = constant(c, b"none")
    c = bytes(c)
    assert model([(COL, 0), (CONST, 0, STR, sep), (CONCAT,), (COL, 1), (CONCAT,)], rows, c)[1] == [b"Hello/World", None, None]
    assert model([(COL, 0), (LOWER,)], rows, c)[1] == [b"hello", None, b"abc-\x7f"]
    assert model([(COL, 0), (UPPER,), (LOWER,)], rows, c)[1] == [b"hello", None, b"abc-\x7f"]  # the outermost wins
    assert model([(COL, 0), (LOWER,), (UPPER,)], rows, c)[1] == [b"HELLO", None, b"ABC-\x7f"]
    assert model([(COL, 0), (CONST, 0, STR, none), (IFNULL, 0, STR)], rows, c)[1] == [b"Hello", b"none", b"AbC-\x7f"]
    assert model([(COL, 1), (COL, 0), (IFNULL, 0, STR)], rows, c)[1] == [b"World", b"x", b"AbC-\x7f"]
    assert model([(COL, 0), (LOWER,)], rows, c, selection=[True, False, False])[1] == [b"hello", None, None]
    bad = rows + [[(STR, b"Stra\xc3\x9fe"), (STR, b"")]]
    assert model([(COL, 0), (LOWER,)], bad, c) == ("error", "nonascii")
    assert model([(COL, 0), (LOWER,)], bad, c, selection=[True, True, True, False])[0] == STR  # unselected: not evaluated
    assert model([(COL, 0), (COL, 1), (CONCAT,)], bad, c)[1][3] == b"Stra\xc3\x9fe"               # CONCAT takes any byte
    h = model([(COL, 0), (COL, 1), (FARM, 2)], rows, c)[1]
    assert all(isinstance(x, int) for x in h) and len(set(h)) == 3                                  # never NULL
    assert model([(COL, 1), (FARM, 1)], rows, c)[1][2] == fp_u128(0xDEADC0DE, 0) ^ 1                # NULL hashes as 0


def _golden():
    with open(os.path.join(ROOT, "tests", "golden", "reference_vectors.json")) as f:
        return json.load(f)["farm_fingerprint"]["cases"]


def _golden_value(d):
    t, v = d["t"], d["v"]
    return {"int64": lambda: (I64, int(v) & M64), "uint64": lambda: (U64T, int(v)),
            "double": lambda: (DBL, int(np.float64(v).view(np.uint64))), "boolean": lambda: (BOOL, int(bool(v))),
            "string": lambda: (STR, v.encode())}[t]()


def _python_value(t, v):
    """(type, model value) -> the value make_rowset takes."""
    if v is None:
        return None
    return {I64: lambda: int(np.uint64(v).view(np.int64)), U64T: lambda: U64(v), DBL: lambda: float(np.uint64(v).view(np.float64)),
            BOOL: lambda: bool(v), STR: lambda: v}[t]()


def test_model_farm_hash_matches_the_oracle_and_the_reference_vectors():
    for case in _golden():
        v0, v1 = _golden_value(case["v0"]), _golden_value(case["v1"])
        assert farm_hash([v0]) ^ 1 == fp_u128(0xDEADC0DE, int(case["fp0"]))  # fp0 is the value's own fingerprint
        assert farm_hash([v0, v1]) == int(case["fp_range"])
    rng = np.random.default_rng(3)
    edge = [(DBL, int(np.float64(np.nan).view(np.uint64))), (DBL, int(np.float64(-0.0).view(np.uint64))), (BOOL, 1), (BOOL, 0),
            (STR, b""), (STR, None), (I64, None), (I64, M64), (U64T, 1 << 63), (STR, b"x" * 70), (STR, bytes(range(256)))]
    rows = []
    for _ in range(300):
        k = int(rng.integers(1, 6))
        rows.append([edge[int(rng.integers(0, len(edge)))] for _ in range(k)] + [(I64, None)] * (5 - k))
    for k in range(1, 6):
        rs = make_rowset([[_python_value(t, v) for t, v in r] for r in rows])
        want = oracle.row_fingerprints(rs.values, rs.heap, k)
        assert [farm_hash(r[:k]) for r in rows] == [int(x) for x in want]


def test_random_programs_respect_the_limits_and_are_well_typed():
    rng = np.random.default_rng(5)
    ops, sizes = set(), []
    for _ in range(400):
        consts = bytearray()
        p = random_program(rng, [2, 3], [(0, I64), (1, DBL)], consts)
        assert 1 <= len(p) <= 64 and stack_depth(p) <= 16 and pieces_bound(p, [2, 3]) <= 16
        assert len(consts) <= capi.EXPR_MAX_STRING_CONSTANT_BYTES
        row = [(I64, 5), (DBL, 0), (STR, b"Ab"), (STR, None)]
        t, _ = model(p, [row], bytes(consts))
        assert t in (STR, U64T)
        ops |= {node[0] for node in p}
        sizes.append(len(p))
    assert ops == {COL, CONST, ADD, MOD, BAND, IFNULL, CONCAT, LOWER, UPPER, FARM} and max(sizes) >= 30


HEADER_PROGRAM = r"""
#include <stdio.h>
#include "include/ytgpu.h"
int main(void) {
    int (*f)(ytgpu_context*, const ytgpu_column_view*, uint32_t, const ytgpu_string_column*, uint32_t, const uint8_t*, uint64_t,
             const ytgpu_expr_node*, uint32_t, const uint8_t*, uint64_t*, uint8_t*, uint8_t*, uint64_t, uint64_t*, uint32_t*, uint8_t*,
             uint64_t*, uint8_t*, uint64_t*, int, ytgpu_error*) = ytgpu_evaluate_expression_strings;
    printf("%d %d %d %d %d %d %d %u\n", (int)sizeof(ytgpu_expr_node), YTGPU_EXPR_CONCAT, YTGPU_EXPR_LOWER, YTGPU_EXPR_UPPER,
           YTGPU_EXPR_FARM_HASH, YTGPU_EXPR_MAX_PIECES, YTGPU_EXPR_MAX_HASH_OPERANDS, YTGPU_EXPR_MAX_STRING_CONSTANT_BYTES);
    return f == 0;
}
"""


def test_header_compiles_as_c99_and_the_symbol_is_exported():
    with tempfile.TemporaryDirectory() as d:
        src, obj = os.path.join(d, "e.c"), os.path.join(d, "e.o")
        open(src, "w").write(HEADER_PROGRAM)
        subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", ROOT, "-c", src, "-o", obj])
    lib = capi.load()
    assert "ytgpu_evaluate_expression_strings" in capi.EXPORTED_SYMBOLS and hasattr(lib, "ytgpu_evaluate_expression_strings")
    assert (capi.EXPR_CONCAT, capi.EXPR_LOWER, capi.EXPR_UPPER, capi.EXPR_FARM_HASH) == (15, 16, 17, 18)
    assert C.sizeof(capi.ExprNode) == 24


def test_host_adapter_builds_and_refuses_cpu():
    import torch
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "string_expression_ut"], stdout=subprocess.DEVNULL)
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([os.path.join(ROOT, "host", "string_expression_ut")], capture_output=True, text=True, timeout=120)
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


def host(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def string_column(values, rng, device=False, at_end=True):
    """(heap, starts, lengths, nulls) holding values (bytes or None) in a shuffled heap with gaps; with at_end the last value
    placed ends exactly at the end of the heap."""
    n = len(values)
    order = rng.permutation(n)
    heap, starts = bytearray(), np.zeros(n, np.uint64)
    for i in order:
        heap += bytes(int(rng.integers(0, 3)))
        starts[i] = len(heap)
        heap += values[i] or b""
    if not at_end:
        heap += b"\x00" * 5
    lengths = np.array([len(v or b"") for v in values], np.uint32)
    nulls = np.array([v is None for v in values], np.uint8)
    cols = [np.frombuffer(bytes(heap), np.uint8).copy(), starts, lengths.view(np.uint32), nulls]
    if device:
        import torch
        cols = [torch.from_numpy(c.view(np.int64) if c.dtype == np.uint64 else (c.view(np.int32) if c.dtype == np.uint32 else c)).cuda()
                for c in cols]
    return tuple(cols)


def numeric_column(vtype, values, device=False):
    from ytsaurus_b200 import Column
    n = len(values)
    bits = np.array([0 if v is None else v & M64 for v in values], np.uint64)
    nulls = np.array([v is None for v in values], bool)
    bm = np.zeros((n + 63) // 64 * 8, np.uint8)
    packed = np.packbits(nulls, bitorder="little")
    bm[:len(packed)] = packed
    if device:
        import torch
        return Column(vtype, values=torch.from_numpy(bits.view(np.int64)).cuda(), value_count=n,
                      null_bitmap=torch.from_numpy(bm).cuda())
    return Column(vtype, values=bits, value_count=n, null_bitmap=bm)


def check(ctx, prog, numeric, strings, rows, consts, device, selection=None):
    """Runs the program and compares it with the model, byte for byte."""
    sel = None
    n = len(rows)
    if selection is not None:
        bm = np.zeros((n + 63) // 64 * 8, np.uint8)
        packed = np.packbits(np.asarray(selection, bool), bitorder="little")
        bm[:len(packed)] = packed
        sel = bm
        if device:
            import torch
            sel = torch.from_numpy(bm).cuda()
    t, want = model(prog, rows, consts, selection)
    if t == "error":
        with pytest.raises(capi.YtGpuError) as e:
            ctx.evaluate_expression(numeric, prog, sel, string_columns=strings, string_constants=consts)
        assert e.value.code == capi.ERR_UNSUPPORTED and "0x80" in e.value.message
        return None
    got = ctx.evaluate_expression(numeric, prog, sel, string_columns=strings, string_constants=consts)
    if t is not None:  # None: no row selected, so the model typed nothing
        assert got["value_type"] == t
    assert got["null_count"] == sum(v is None for v in want)
    if got["value_type"] == STR:
        heap, starts, lengths, nulls = flat_strings(want)
        assert bytes(host(got["heap"])) == heap, prog
        assert np.array_equal(host(got["starts"]).view(np.uint64), starts)
        assert np.array_equal(host(got["lengths"]).view(np.uint32), lengths)
        assert np.array_equal(host(got["null_bytemap"]), nulls)
        if device and n:
            assert hasattr(got["heap"], "is_cuda") and got["heap"].is_cuda
    else:
        vals = host(got["values"]).view(np.uint64)
        bits = np.unpackbits(host(got["null_bitmap"]), bitorder="little")[:n].astype(bool)
        assert [None if b else int(v) for v, b in zip(vals, bits)] == want, prog
    return got


def random_strings(rng, n, null_rate=0.15, non_ascii=0.0):
    alphabet = np.frombuffer(b"abcXYZ019-_./ AZaz@[`{", np.uint8)
    out = []
    for _ in range(n):
        if rng.random() < null_rate:
            out.append(None)
            continue
        L = int(rng.choice([0, 1, 3, 7, 8, 9, 20, 47, 48, 49, 60, 100]))
        s = bytes(alphabet[rng.integers(0, len(alphabet), L)])
        if non_ascii and rng.random() < non_ascii and L:
            s = s[:-1] + b"\xc3"
        out.append(s)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_every_op(ctx, device):
    rng = np.random.default_rng(11 + int(device))
    n = 1000
    s0, s1 = random_strings(rng, n), random_strings(rng, n)
    a = [None if rng.random() < 0.1 else int(rng.integers(0, 1 << 63)) for _ in range(n)]
    d = [None if rng.random() < 0.1 else int(np.float64(x).view(np.uint64)) for x in rng.choice([0.0, -0.0, np.nan, 1.5, -3e300], n)]
    b = [None if rng.random() < 0.1 else int(rng.integers(0, 2)) for _ in range(n)]
    numeric = [numeric_column(I64, a, device), numeric_column(DBL, d, device), numeric_column(BOOL, b, device)]
    strings = [string_column(s0, rng, device), string_column(s1, rng, device)]
    rows = [[(I64, a[i]), (DBL, d[i]), (BOOL, b[i]), (STR, s0[i]), (STR, s1[i])] for i in range(n)]
    c = bytearray()
    sep, none = constant(c, b"/"), constant(c, b"None")
    consts = bytes(c)
    programs = [
        [(COL, 3), (COL, 4), (CONCAT,)], [(COL, 3), (CONST, 0, STR, sep), (CONCAT,), (COL, 4), (CONCAT,)],
        [(COL, 3), (LOWER,)], [(COL, 4), (UPPER,)], [(COL, 3), (UPPER,), (COL, 4), (CONCAT,), (LOWER,)],
        [(COL, 3), (CONST, 0, STR, none), (IFNULL, 0, STR)], [(COL, 3), (COL, 4), (IFNULL, 0, STR), (UPPER,)],
        [(COL, 3), (LOWER,), (CONST, 0, STR, none), (IFNULL, 0, STR)],
        [(COL, 3), (FARM, 1)], [(COL, 0), (COL, 3), (FARM, 2), (CONST, 0, U64T, 64), (MOD,)],
        [(COL, 0), (COL, 1), (COL, 2), (COL, 3), (COL, 4), (CONST, 0, STR, sep), (FARM, 6)],
        [(COL, 3), (COL, 4), (IFNULL, 0, STR), (CONST, 0, STR, none), (FARM, 2)],
        [(CONST, 0, STR, sep), (COL, 3), (CONCAT,)],
    ]
    for prog in programs:
        check(ctx, prog, numeric, strings, rows, consts, device)
        check(ctx, prog, numeric, strings, rows, consts, device, selection=rng.random(n) < 0.6)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_value_lengths_at_the_end_of_the_heap(ctx, device):
    rng = np.random.default_rng(23)
    c = bytearray()
    tail = constant(c, b"/Q")
    consts = bytes(c)
    for L in (0, 1, 7, 8, 9, 31, 32, 33, 64, 65, 4096, 1 << 20):
        vals = [bytes(rng.choice(np.frombuffer(b"aBcDz09", np.uint8), L)) for _ in range(3)] + [None]
        for at_end in (True, False):
            strings = [string_column(vals, rng, device, at_end)]
            rows = [[(STR, v)] for v in vals]
            for prog in ([(COL, 0), (LOWER,)], [(COL, 0), (UPPER,)], [(COL, 0), (COL, 0), (CONCAT,)],
                         [(COL, 0), (CONST, 0, STR, tail), (CONCAT,), (UPPER,)], [(COL, 0), (FARM, 1)]):
                check(ctx, prog, [], strings, rows, consts, device)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_random_programs_at_every_size(ctx, device):
    rng = np.random.default_rng(31 + int(device))
    for n in (0, 1, 31, 32, 33, 10**5):
        for rep in range(6 if n < 10**5 else 2):
            s = [random_strings(rng, n) for _ in range(2)]
            a = [None if rng.random() < 0.1 else int(rng.integers(0, 1 << 64, dtype=np.uint64)) for _ in range(n)]
            d = [None if rng.random() < 0.1 else int(np.float64(x).view(np.uint64)) for x in rng.normal(size=n)]
            numeric = [numeric_column(I64, a, device), numeric_column(DBL, d, device)]
            strings = [string_column(x, rng, device) for x in s]
            rows = [[(I64, a[i]), (DBL, d[i]), (STR, s[0][i]), (STR, s[1][i])] for i in range(n)]
            consts = bytearray()
            prog = random_program(rng, [2, 3], [(0, I64), (1, DBL)], consts)
            selection = rng.random(n) < 0.7 if rep % 2 else None
            check(ctx, prog, numeric, strings, rows, bytes(consts), device, selection)


@pytest.mark.gpu
def test_gpu_ten_million_rows(ctx):
    import torch
    rng = np.random.default_rng(37)
    n = 10**7
    pool = [bytes(x) for x in (b"Example.COM/a", b"", b"yt.TECH/Path/To/Some/Longer/Resource?q=1&r=ABC", b"x" * 70, b"MiXeD")]
    idx = rng.integers(0, len(pool) + 1, n)  # len(pool): NULL
    vals = [None if i == len(pool) else pool[i] for i in idx]
    lens = np.array([len(pool[i]) if i < len(pool) else 0 for i in range(len(pool) + 1)], np.uint32)[idx]
    starts = np.zeros(n, np.uint64)
    starts[1:] = np.cumsum(lens[:-1], dtype=np.uint64)
    heap = np.frombuffer(b"".join(v for v in vals if v is not None), np.uint8)
    nulls = (idx == len(pool)).astype(np.uint8)
    dev = (torch.from_numpy(heap.copy()).cuda(), torch.from_numpy(starts.view(np.int64)).cuda(),
           torch.from_numpy(lens.view(np.int32)).cuda(), torch.from_numpy(nulls).cuda())
    c = bytearray()
    none = constant(c, b"none")
    prog = [(COL, 0), (LOWER,), (CONST, 0, STR, none), (IFNULL, 0, STR)]
    got = ctx.evaluate_expression([], prog, string_columns=[dev], string_constants=bytes(c))
    table = [p.lower() for p in pool] + [b"none"]
    want_heap, want_starts, want_lengths, _ = flat_strings([table[i] for i in idx])
    assert bytes(host(got["heap"])) == want_heap
    assert np.array_equal(host(got["starts"]).view(np.uint64), want_starts)
    assert np.array_equal(host(got["lengths"]).view(np.uint32), want_lengths)
    assert got["null_count"] == 0
    # farm_hash(s) over the same rows against the oracle
    got = ctx.evaluate_expression([], [(COL, 0), (FARM, 1)], string_columns=[dev])
    fps = [farm_hash([(STR, p)]) for p in pool] + [farm_hash([(STR, None)])]
    assert np.array_equal(host(got["values"]).view(np.uint64), np.array(fps, np.uint64)[idx])


@pytest.mark.gpu
def test_gpu_random_programs_ten_million_rows(ctx):
    """Random mixed programs at 10^7 rows under a selection.  The rows are drawn from a pool of 4096 distinct rows, with
    short and long values and NULLs, so the model evaluates each distinct row once and its results are gathered by row."""
    import torch
    rng = np.random.default_rng(53)
    n, m = 10**7, 4096
    pool_s = [random_strings(rng, m, null_rate=0.1) for _ in range(2)]
    for s in pool_s:  # long values among them: the warp-wide copy
        for k in rng.choice(m, 200, replace=False):
            s[k] = bytes(rng.choice(np.frombuffer(b"aZ09-./Q", np.uint8), int(rng.integers(49, 600))))
    pool_a = [None if rng.random() < 0.1 else int(rng.integers(0, 1 << 63)) for _ in range(m)]
    idx = rng.integers(0, m, n)
    sel = rng.random(n) < 0.7
    strings = []
    for s in pool_s:  # one heap of the pool's values; every row points at its pool entry
        offs = np.cumsum([0] + [len(v or b"") for v in s[:-1]]).astype(np.uint64)
        heap = np.frombuffer(b"".join(v or b"" for v in s), np.uint8).copy()
        lens = np.array([len(v or b"") for v in s], np.uint32)
        nul = np.array([v is None for v in s], np.uint8)
        strings.append(tuple(torch.from_numpy(x).cuda() for x in
                             (heap, offs[idx].view(np.int64), lens[idx].view(np.int32), nul[idx])))
    a_bits = np.array([0 if v is None else v for v in pool_a], np.uint64)[idx]
    a_null = np.array([v is None for v in pool_a])[idx]
    bm = np.zeros((n + 63) // 64 * 8, np.uint8)
    bm[:(n + 7) // 8] = np.packbits(a_null, bitorder="little")
    from ytsaurus_b200 import Column
    numeric = [Column(I64, values=torch.from_numpy(a_bits.view(np.int64)).cuda(), value_count=n, null_bitmap=torch.from_numpy(bm).cuda())]
    sbm = np.zeros((n + 63) // 64 * 8, np.uint8)
    sbm[:(n + 7) // 8] = np.packbits(sel, bitorder="little")
    sel_dev = torch.from_numpy(sbm).cuda()
    rows = [[(I64, pool_a[k]), (STR, pool_s[0][k]), (STR, pool_s[1][k])] for k in range(m)]
    done = set()
    while done != {STR, U64T}:
        consts = bytearray()
        prog = random_program(rng, [1, 2], [(0, I64)], consts)
        if len(prog) < 6:
            continue
        t, want = model(prog, rows, bytes(consts))
        if t == "error" or t in done:
            continue
        done.add(t)
        got = ctx.evaluate_expression(numeric, prog, sel_dev, string_columns=strings, string_constants=bytes(consts))
        assert got["value_type"] == t
        if t == STR:
            lens = np.array([0 if v is None else len(v) for v in want], np.uint64)
            row_len = np.where(sel, lens[idx], 0)
            starts = np.zeros(n, np.uint64)
            starts[1:] = np.cumsum(row_len[:-1], dtype=np.uint64)
            assert np.array_equal(host(got["lengths"]).view(np.uint32), row_len.astype(np.uint32)), prog
            assert np.array_equal(host(got["starts"]).view(np.uint64), starts)
            pool_null = np.array([v is None for v in want])
            assert np.array_equal(host(got["null_bytemap"]).astype(bool), ~sel | pool_null[idx])
            want_heap = b"".join(want[k] for k in idx[sel] if want[k] is not None)
            assert bytes(host(got["heap"])) == want_heap, prog
        else:
            vals = np.array([0 if v is None else v for v in want], np.uint64)[idx]
            nb = np.unpackbits(host(got["null_bitmap"]), bitorder="little")[:n].astype(bool)
            assert np.array_equal(nb, ~sel)
            assert np.array_equal(host(got["values"]).view(np.uint64)[sel], vals[sel]), prog


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_farm_hash_matches_the_oracle_and_the_rowset_call(ctx, device):
    rng = np.random.default_rng(41)
    n = 2000
    choices = {I64: [0, 1, M64, 1 << 63, None], U64T: [0, M64, 12345678, None],
               DBL: [int(np.float64(x).view(np.uint64)) for x in (0.0, -0.0, np.nan, 42.0, np.inf)] + [None],
               BOOL: [0, 1, None], STR: [b"", b"0", b"abc", b"x" * 100, None]}
    types = [I64, U64T, DBL, BOOL, STR, STR]
    cols = [[choices[t][int(rng.integers(0, len(choices[t])))] for _ in range(n)] for t in types]
    numeric = [numeric_column(t, cols[j], device) for j, t in enumerate(types) if t != STR]
    strings = [string_column(cols[j], rng, device) for j, t in enumerate(types) if t == STR]
    order = [j for j, t in enumerate(types) if t != STR] + [j for j, t in enumerate(types) if t == STR]
    for k in range(1, 7):
        perm = rng.permutation(len(types))[:k]
        prog = [(COL, order.index(int(j))) for j in perm] + [(FARM, k)]
        got = host(ctx.evaluate_expression(numeric, prog, string_columns=strings)["values"]).view(np.uint64)
        rs = make_rowset([[_python_value(types[j], cols[j][i]) for j in perm] for i in range(n)])
        want = oracle.row_fingerprints(rs.values, rs.heap, k)
        assert np.array_equal(got, want)
        assert np.array_equal(host(ctx.farm_fingerprints(rs.values, rs.heap, k)).view(np.uint64), want)
    for case in _golden():
        v0, v1 = _golden_value(case["v0"]), _golden_value(case["v1"])
        c = bytearray()
        prog = [(CONST, 0, t, constant(c, v) if t == STR else v) for t, v in (v0, v1)]
        one = [numeric_column(I64, [None])]
        h0 = int(host(ctx.evaluate_expression(one, prog[:1] + [(FARM, 1)], string_constants=bytes(c))["values"])[0])
        h2 = int(host(ctx.evaluate_expression(one, prog + [(FARM, 2)], string_constants=bytes(c))["values"])[0]) & M64
        assert h0 & M64 == fp_u128(0xDEADC0DE, int(case["fp0"])) ^ 1
        assert h2 == int(case["fp_range"])


def _string_column_of(s):
    from ytsaurus_b200.runtime import _string_column
    return _string_column(*s)


def _call(ctx, strings, prog, consts=b"", heap=None, capacity=0, outs=None, mem=capi.MEM_HOST, numeric=()):
    """ytgpu_evaluate_expression_strings directly -> (code, heap bytes, message)."""
    from ytsaurus_b200.runtime import _string_column
    sarr = (capi.StringColumn * max(len(strings), 1))()
    for i, s in enumerate(strings):
        sarr[i] = _string_column(*s)
    views = [c.view() for c in numeric]
    carr = (capi.ColumnView * max(len(views), 1))(*views)
    nodes = (capi.ExprNode * max(len(prog), 1))()
    for i, node in enumerate(prog):
        op, column, vtype, constant_ = (tuple(node) + (0,) * 4)[:4]
        nodes[i].op, nodes[i].column, nodes[i].type, nodes[i].constant = op, column, vtype, constant_ & M64
    sc = np.frombuffer(consts, np.uint8) if consts else np.zeros(0, np.uint8)
    outs = outs or (None, None, None)
    heap_bytes = C.c_uint64(0)
    n = int(sarr[0].row_count) if strings else int(views[0].value_count)
    values, bm = np.zeros(max(n, 1), np.uint64), np.zeros(max(n, 1) * 8, np.uint8)
    err = capi.Error()
    ptr = lambda x: None if x is None else (x.data_ptr() if hasattr(x, "data_ptr") else x.ctypes.data)
    code = ctx.lib.ytgpu_evaluate_expression_strings(
        ctx.handle, C.cast(carr, C.c_void_p), len(views), C.cast(sarr, C.c_void_p), len(strings), sc.ctypes.data if sc.size else None,
        len(consts), C.cast(nodes, C.c_void_p), len(prog), None, values.ctypes.data, bm.ctypes.data, ptr(heap), capacity, ptr(outs[0]),
        ptr(outs[1]), ptr(outs[2]), C.byref(heap_bytes), None, None, mem, C.byref(err))
    return code, int(heap_bytes.value), err.message.decode(errors="replace")


@pytest.mark.gpu
def test_gpu_sizing_protocol_bounds_limits_and_launches(ctx):
    rng = np.random.default_rng(43)
    n = 100
    vals = random_strings(rng, n, null_rate=0.2)
    col = string_column(vals, rng)
    prog = [(COL, 0), (COL, 0), (CONCAT,)]
    need = 2 * sum(len(v) for v in vals if v is not None)
    inv, uns = capi.ERR_INVALID_ARGUMENT, capi.ERR_UNSUPPORTED
    outs = (np.zeros(n, np.uint64), np.zeros(n, np.uint32), np.zeros(n, np.uint8))
    # sizing: NULL heap -> the size; too small -> INVALID_ARGUMENT with the size; exact -> OK
    assert _call(ctx, [col], prog)[:2] == (capi.OK, need)
    small = np.zeros(need, np.uint8)
    assert _call(ctx, [col], prog, heap=small, capacity=need - 1, outs=outs)[:2] == (inv, need)
    assert _call(ctx, [col], prog, heap=small, capacity=need, outs=outs)[:2] == (capi.OK, need)
    want = flat_strings([None if v is None else v + v for v in vals])
    assert bytes(small) == want[0] and np.array_equal(outs[0], want[1]) and np.array_equal(outs[1], want[2])
    # launches: size query 4, full call 5, a numeric result 1
    before = ctx.launch_count()
    _call(ctx, [col], prog)
    assert ctx.launch_count() - before == 4
    before = ctx.launch_count()
    _call(ctx, [col], prog, heap=small, capacity=need, outs=outs)
    assert ctx.launch_count() - before == 5
    before = ctx.launch_count()
    assert _call(ctx, [col], [(COL, 0), (FARM, 1)])[0] == capi.OK
    assert ctx.launch_count() - before == 1
    # a type query (out_heap, out_values and out_null_bitmap all NULL): a numeric result is typed, not evaluated
    vtype = C.c_uint8(0)
    sarr = (capi.StringColumn * 1)(_string_column_of(col))
    nodes = (capi.ExprNode * 2)()
    nodes[0].op, nodes[1].op, nodes[1].column = COL, FARM, 1
    hb, err = C.c_uint64(0), capi.Error()
    before = ctx.launch_count()
    assert ctx.lib.ytgpu_evaluate_expression_strings(ctx.handle, None, 0, C.cast(sarr, C.c_void_p), 1, None, 0, C.cast(nodes, C.c_void_p),
                                                     2, None, None, None, None, 0, None, None, None, C.byref(hb), C.byref(vtype), None,
                                                     capi.MEM_HOST, C.byref(err)) == capi.OK
    assert ctx.launch_count() == before and vtype.value == U64T
    # ... a numeric result with only one of out_values / out_null_bitmap is still refused
    only_values = np.zeros(n, np.uint64)
    assert ctx.lib.ytgpu_evaluate_expression_strings(ctx.handle, None, 0, C.cast(sarr, C.c_void_p), 1, None, 0, C.cast(nodes, C.c_void_p),
                                                     2, None, only_values.ctypes.data, None, None, 0, None, None, None, C.byref(hb), None, None,
                                                     capi.MEM_HOST, C.byref(err)) == inv
    # non-ASCII: refused in a selected non-NULL row only
    bad = list(vals)
    bad[7] = b"Stra\xc3\x9fe"
    bcol = string_column(bad, rng)
    rows = [[(STR, v)] for v in bad]
    check(ctx, [(COL, 0), (LOWER,)], [], [bcol], rows, b"", False)                           # raises UNSUPPORTED
    sel = np.ones(n, bool)
    sel[7] = False
    check(ctx, [(COL, 0), (UPPER,)], [], [bcol], rows, b"", False, selection=sel)            # dropped by the selection
    nul = list(bcol)
    nul[3] = nul[3].copy()
    nul[3][7] = 1
    check(ctx, [(COL, 0), (LOWER,)], [], [tuple(nul)], [[(STR, None if i == 7 else v)] for i, v in enumerate(bad)], b"", False)
    assert _call(ctx, [bcol], [(COL, 0), (COL, 0), (CONCAT,)])[0] == capi.OK                  # CONCAT copies any byte
    # values outside the heap: refused on the device, also when only the size is asked
    oob = [x.copy() for x in col]
    i = next(k for k, v in enumerate(vals) if v)
    oob[1][i] = len(oob[0]) - len(vals[i]) + 1
    assert _call(ctx, [tuple(oob)], prog)[0] == inv
    oob[1][i] = len(oob[0]) - len(vals[i])  # at the very end: fine
    assert _call(ctx, [tuple(oob)], prog)[0] == capi.OK
    oob[3][i] = 1  # a NULL row's start and length are ignored
    oob[1][i] = 1 << 60
    assert _call(ctx, [tuple(oob)], prog)[0] == capi.OK
    # pieces: 16 at the bound, 17 past it
    leaf = (COL, 0)
    p16 = [leaf, leaf, (CONCAT,)] + [leaf, (CONCAT,)] * 14
    assert _call(ctx, [col], p16)[0] == capi.OK and _call(ctx, [col], p16 + [leaf, (CONCAT,)])[0] == inv
    # FARM_HASH operand counts 1..16, the operand rules
    assert _call(ctx, [col], [leaf] * 16 + [(FARM, 16)])[0] == capi.OK
    assert _call(ctx, [col], [leaf] * 16 + [(FARM, 17)])[0] == inv and _call(ctx, [col], [leaf, (FARM, 0)])[0] == inv
    assert _call(ctx, [col], [leaf, (FARM, 2)])[0] == inv                                    # underflow
    for op in (CONCAT, LOWER, UPPER):
        p = [leaf, leaf, (CONCAT,)] if op == CONCAT else [leaf, (op,)]
        assert _call(ctx, [col], p + [(FARM, 1)])[0] == uns
    assert _call(ctx, [col], [leaf, leaf, (IFNULL, 0, STR), (FARM, 1)])[0] == capi.OK
    # types: numeric ops over strings UNSUPPORTED, new ops over numbers INVALID_ARGUMENT
    num = [numeric_column(I64, [1] * n)]
    assert _call(ctx, [col], [(COL, 1), (capi.EXPR_NEG,)], numeric=num)[0] == uns
    assert _call(ctx, [col], [(COL, 1), (COL, 1), (ADD,)], numeric=num)[0] == uns
    assert _call(ctx, [col], [(COL, 1), (capi.EXPR_CAST, 0, I64)], numeric=num)[0] == uns
    assert _call(ctx, [col], [(COL, 0), (LOWER,)], numeric=num)[0] == inv
    assert _call(ctx, [col], [(COL, 0), (COL, 1), (CONCAT,)], numeric=num)[0] == inv
    assert _call(ctx, [col], [(COL, 0), (COL, 1), (IFNULL, 0, I64)], numeric=num)[0] == inv
    assert _call(ctx, [col], [(COL, 2)], numeric=num)[0] == inv                              # column out of range
    # string constants: inside the buffer, 1 MiB at most
    big = bytes(1 << 20)
    assert _call(ctx, [col], [(CONST, 0, STR, (((1 << 20) - 3) << 32) | 3)], big)[0] == capi.OK
    assert _call(ctx, [col], [(CONST, 0, STR, (((1 << 20) - 3) << 32) | 4)], big)[0] == inv
    assert _call(ctx, [col], [(CONST, 0, STR, 0)], big + b"x")[0] == inv
    # ytgpu_evaluate_expression keeps refusing strings and the new ops
    from ytsaurus_b200 import Column
    with pytest.raises(capi.YtGpuError) as e:
        ctx.evaluate_expression([Column(STR, values=np.zeros(n, np.uint64), value_count=n)], [(COL, 0)])
    assert e.value.code == uns


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_end_to_end_groupby_and_filter(ctx, device):
    """GROUP BY lower(host) and GROUP BY farm_hash(k) % 64, and a lower(agent) LIKE filter, against the same values
    computed by the model and passed as plain columns."""
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(47 + int(device))
    n = 50_000
    hosts = [None if rng.random() < 0.05 else b"Host-%d.Example.COM" % int(rng.integers(0, 50)) * int(rng.integers(1, 3)) for _ in range(n)]
    agents = [None if rng.random() < 0.05 else (b"Mozilla/5.0 " + (b"GoogleBOT" if rng.random() < 0.1 else b"Safari")) for _ in range(n)]
    k = [int(x) for x in rng.integers(0, 1000, n)]
    val = numeric_column(I64, [int(x) for x in rng.integers(-100, 100, n)], device)
    hcol, acol = string_column(hosts, rng, device), string_column(agents, rng, device)
    low = ctx.evaluate_expression([], [(COL, 0), (LOWER,)], string_columns=[hcol])
    pre = string_column([None if h is None else h.lower() for h in hosts], rng, device)
    ids_got = ctx.string_value_ids(low["heap"], low["starts"], low["lengths"], low["null_bytemap"])
    ids_want = ctx.string_value_ids(*pre)
    aggs = [(capi.AGG_COUNT, 0), (capi.AGG_SUM, 0), (capi.AGG_MIN, 1)]

    def key(ids):
        return Column(U64T, values=ids[0], value_count=n, null_bitmap=None)
    got = ctx.scan_filter_groupby_multi([key(ids_got)], [val], aggs,
                                        string_columns=[(low["heap"], low["starts"], low["lengths"], low["null_bytemap"])])
    want = ctx.scan_filter_groupby_multi([key(ids_want)], [val], aggs, string_columns=[pre])
    # keys are first rows and MIN of a string is the smallest row holding it, so equal strings give equal outputs
    assert len(host(got["count"])) > 40 and np.array_equal(host(got["count"]), host(want["count"]))
    for a, b in zip(got["keys"] + got["values"] + got["value_null"], want["keys"] + want["values"] + want["value_null"]):
        assert np.array_equal(host(a), host(b))
    # farm_hash(k) % 64 through groupby_multi
    kcol = numeric_column(I64, k, device)
    hk = ctx.evaluate_expression([kcol], [(COL, 0), (FARM, 1), (CONST, 0, U64T, 64), (MOD,)])
    hk_want = numeric_column(U64T, [farm_hash([(I64, x)]) % 64 for x in k], device)
    g1 = ctx.scan_filter_groupby_multi([hk["column"]], [val], aggs[:2])
    g2 = ctx.scan_filter_groupby_multi([hk_want], [val], aggs[:2])
    for x in ("count",):
        assert np.array_equal(host(g1[x]), host(g2[x]))
    for a, b in zip(g1["keys"] + g1["values"], g2["keys"] + g2["values"]):
        assert np.array_equal(host(a), host(b))
    # lower(agent) LIKE '%bot%'
    la = ctx.evaluate_expression([], [(COL, 0), (LOWER,)], string_columns=[acol])
    c = bytearray()
    pat = constant(c, b"%bot%")
    fprog = [(capi.FILTER_LIKE, 0, 0, -1, pat >> 32, pat & 0xFFFFFFFF)]
    f1 = ctx.evaluate_filter([], [(la["heap"], la["starts"], la["lengths"], la["null_bytemap"])], fprog, string_constants=bytes(c))
    f2 = ctx.evaluate_filter([], [string_column([None if a is None else a.lower() for a in agents], rng, device)], fprog,
                             string_constants=bytes(c))
    assert f1["count"] == f2["count"] > 0
    assert np.array_equal(host(f1["bitmap"]), host(f2["bitmap"]))


@pytest.mark.gpu
def test_gpu_host_adapter_string_expressions():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "string_expression_ut"], stdout=subprocess.DEVNULL)
    r = subprocess.run([os.path.join(ROOT, "host", "string_expression_ut")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "string_expression_ut: 0 failure(s)" in r.stdout
