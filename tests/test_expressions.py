"""Computed columns on the GPU (ytgpu_evaluate_expression, csrc/expression.cu) against a numpy model of their semantics.

The model restates include/ytgpu.h: a typed postfix program; a NULL operand makes the result NULL except in IF_NULL; integer
ADD / SUB / MUL / NEG wrap mod 2^64 (computed in uint64), DIV truncates and MOD has the dividend's sign (computed on uint64
magnitudes, so INT64_MIN is exact); a divisor of 0 and INT64_MIN / -1 in an evaluated row fail the call; doubles are IEEE
with round to nearest, one rounding per operation; DOUBLE -> integer casts truncate and saturate, NaN -> 0; rows outside
the selection are NULL and never fail.  The GPU results are compared bit for bit, except that any two NaNs of a DOUBLE result
match: IEEE leaves the sign and payload of a NaN an operation produces open, and the GPU returns a canonical NaN where the
CPU passes an operand's on."""
import ctypes as C
import importlib.util
import math
import os
import struct
import subprocess
import tempfile

import numpy as np
import pytest

from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import EValueType as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load_filter_tests():
    """The column encodings of the filter tests (make_column & co.), loaded by path so no import mode matters."""
    spec = importlib.util.spec_from_file_location("_filter_expression_helpers",
                                                  os.path.join(os.path.dirname(os.path.abspath(__file__)), "test_filter_expressions.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


F = _load_filter_tests()
make_column, edge_values, to_device, host, _bm = F.make_column, F.edge_values, F.to_device, F.host, F._bm

(COL, CONST, ADD, SUB, MUL, DIV, MOD, NEG, BAND, BOR, BXOR, BNOT, CAST, IFNULL) = (
    capi.EXPR_COLUMN, capi.EXPR_CONSTANT, capi.EXPR_ADD, capi.EXPR_SUB, capi.EXPR_MUL, capi.EXPR_DIV, capi.EXPR_MOD, capi.EXPR_NEG,
    capi.EXPR_BIT_AND, capi.EXPR_BIT_OR, capi.EXPR_BIT_XOR, capi.EXPR_BIT_NOT, capi.EXPR_CAST, capi.EXPR_IF_NULL)
I64, U64, DBL, BOOL = int(T.Int64), int(T.Uint64), int(T.Double), int(T.Boolean)
TYPES = [I64, U64, DBL, BOOL]
NUMBER, INTEGER = (I64, U64, DBL), (I64, U64)
BINARY = {ADD: NUMBER, SUB: NUMBER, MUL: NUMBER, DIV: NUMBER, MOD: INTEGER, BAND: INTEGER, BOR: INTEGER, BXOR: INTEGER,
          IFNULL: tuple(TYPES)}
UNARY = {NEG: NUMBER, BNOT: INTEGER}
INT64_MIN = 1 << 63
M64 = (1 << 64) - 1
SIGN = np.uint64(1 << 63)


def _bits(x):
    return struct.unpack("<Q", struct.pack("<d", float(x)))[0]


def _f(bits):
    return struct.unpack("<d", struct.pack("<Q", int(bits) & M64))[0]


# ------------------------------------------------------------------------------------------------- the model
class ModelError(Exception):
    pass


def _magnitude(x):
    """uint64 |x| of int64 bit patterns (|INT64_MIN| = 2^63 is exact)."""
    neg = (x & SIGN) != 0
    return np.where(neg, np.uint64(0) - x, x), neg


def _binary(op, t, a, b, live):
    """a, b: uint64 bit patterns; live: rows where both are non-NULL (only those may fail)."""
    if t == DBL:
        x, y = a.view(np.float64), b.view(np.float64)
        r = {ADD: lambda: x + y, SUB: lambda: x - y, MUL: lambda: x * y, DIV: lambda: x / y}[op]()
        return np.asarray(r, np.float64).view(np.uint64)
    if op == ADD:
        return a + b
    if op == SUB:
        return a - b
    if op == MUL:
        return a * b
    if op == BAND:
        return a & b
    if op == BOR:
        return a | b
    if op == BXOR:
        return a ^ b
    zero = live & (b == 0)
    if zero.any():
        raise ModelError("Division by zero")
    if t == I64:
        if (live & (a == np.uint64(INT64_MIN)) & (b == np.uint64(M64))).any():
            raise ModelError("Division INT_MIN by -1")
    b = np.where(b == 0, np.uint64(1), b)
    if t == U64:
        return a // b if op == DIV else a % b
    ua, na = _magnitude(a)
    ub, nb = _magnitude(b)
    if op == DIV:
        q = ua // ub
        return np.where(na ^ nb, np.uint64(0) - q, q)
    r = ua % ub
    return np.where(na, np.uint64(0) - r, r)


def _cast(frm, to, a):
    if frm == to or (frm in INTEGER and to in INTEGER) or (frm == BOOL and to in INTEGER):
        return a.copy()
    if to == DBL:
        if frm == I64:
            return a.view(np.int64).astype(np.float64).view(np.uint64)
        if frm == U64:
            return a.astype(np.float64).view(np.uint64)
        return a.astype(np.float64).view(np.uint64)  # BOOLEAN 0 / 1
    d = a.view(np.float64)
    out = np.zeros(len(a), np.uint64)
    if to == I64:
        ok = (d >= -2.0**63) & (d < 2.0**63)
        out[ok] = np.trunc(d[ok]).astype(np.int64).view(np.uint64)
        out[d >= 2.0**63] = np.uint64((1 << 63) - 1)
        out[d < -2.0**63] = np.uint64(INT64_MIN)
    else:
        ok = (d > -1.0) & (d < 2.0**64)
        out[ok] = np.trunc(d[ok]).astype(np.uint64)
        out[d >= 2.0**64] = np.uint64(M64)
    return out  # NaN stays 0


def program_types(col_types, program):
    """Result type of every node (the host check's typing) -> list; raises ValueError for a mistyped program."""
    stack, out = [], []
    for node in program:
        op, column, vtype = (tuple(node) + (0, 0, 0))[:3]
        if op == COL:
            stack.append(col_types[column])
        elif op == CONST:
            stack.append(vtype)
        elif op == CAST:
            stack[-1] = vtype
        elif op in UNARY:
            if stack[-1] not in UNARY[op]:
                raise ValueError(node)
        else:
            b, a = stack.pop(), stack[-1]
            if a != b or a not in BINARY[op]:
                raise ValueError(node)
        out.append(stack[-1])
    return out


def model(cols, program, n, selection=None):
    """cols: [(vtype, bits, nulls)]; program: (op, column, type, constant) tuples; selection: bool mask or None.
    -> (type, values uint64 (0 where NULL), nulls bool); raises ModelError for a division error."""
    sel = np.ones(n, bool) if selection is None else np.asarray(selection, bool)
    stack = []  # (type, bits, nulls)
    with np.errstate(all="ignore"):
        for node in program:
            op, column, vtype, constant = (tuple(node) + (0,) * 4)[:4]
            if op == COL:
                t, bits, nulls = cols[column]
                bits = np.asarray(bits, np.uint64)
                if t == BOOL:
                    bits = (bits != 0).astype(np.uint64)
                nl = np.asarray(nulls, bool) | ~sel
                stack.append((t, np.where(nl, np.uint64(0), bits), nl))
            elif op == CONST:
                nl = ~sel
                stack.append((vtype, np.where(nl, np.uint64(0), np.full(n, int(constant) & M64, np.uint64)), nl))
            elif op in (NEG, BNOT, CAST):
                t, a, nl = stack.pop()
                if op == NEG:
                    r = a ^ SIGN if t == DBL else np.uint64(0) - a
                elif op == BNOT:
                    r = ~a
                else:
                    r, t = _cast(t, vtype, a), vtype
                stack.append((t, np.where(nl, np.uint64(0), r), nl))
            else:
                tb, b, nb = stack.pop()
                ta, a, na = stack.pop()
                assert ta == tb, "mistyped program"
                if op == IFNULL:
                    stack.append((ta, np.where(na, b, a), na & nb))
                    continue
                nl = na | nb
                r = _binary(op, ta, a, b, ~nl)
                stack.append((ta, np.where(nl, np.uint64(0), r), nl))
    assert len(stack) == 1
    return stack[0]


def model_error(cols, program, n, selection=None):
    try:
        model(cols, program, n, selection)
    except ModelError as e:
        return str(e)
    return None


# ------------------------------------------------------------------------------------------------- CPU checks
def _one(t, x):
    return (t, np.array([x & M64], np.uint64), np.array([False]))


def _eval1(program, *cols):
    t, v, nl = model(list(cols), program, 1)
    return None if nl[0] else int(v[0])


def test_model_integer_rules():
    mn, m1 = INT64_MIN, M64  # INT64_MIN, -1 as bit patterns
    assert _eval1([(COL, 0), (COL, 1), (ADD,)], _one(I64, (1 << 63) - 1), _one(I64, 1)) == mn      # wraps
    assert _eval1([(COL, 0), (NEG,)], _one(I64, mn)) == mn                                          # NEG INT64_MIN
    assert _eval1([(COL, 0), (COL, 1), (MUL,)], _one(U64, M64), _one(U64, M64)) == 1
    assert _eval1([(COL, 0), (COL, 1), (SUB,)], _one(U64, 0), _one(U64, 1)) == M64
    assert _eval1([(COL, 0), (COL, 1), (DIV,)], _one(I64, -7), _one(I64, 2)) == (-3) & M64         # truncates
    assert _eval1([(COL, 0), (COL, 1), (MOD,)], _one(I64, -7), _one(I64, 2)) == (-1) & M64         # dividend's sign
    assert _eval1([(COL, 0), (COL, 1), (MOD,)], _one(I64, 7), _one(I64, -2)) == 1
    assert _eval1([(COL, 0), (COL, 1), (DIV,)], _one(I64, mn), _one(I64, 2)) == (-(1 << 62)) & M64
    assert _eval1([(COL, 0), (COL, 1), (MOD,)], _one(I64, mn), _one(I64, 3)) == (-(2**63 % 3)) & M64
    assert _eval1([(COL, 0), (COL, 1), (DIV,)], _one(U64, M64), _one(U64, 2)) == M64 // 2
    assert _eval1([(COL, 0), (COL, 1), (DIV,)], _one(I64, mn), _one(I64, 1)) == mn
    assert _eval1([(COL, 0), (BNOT,)], _one(I64, 0)) == M64
    assert _eval1([(COL, 0), (COL, 1), (BXOR,)], _one(U64, 0b1100), _one(U64, 0b1010)) == 0b0110
    with pytest.raises(ModelError, match="Division by zero"):
        _eval1([(COL, 0), (COL, 1), (DIV,)], _one(I64, 5), _one(I64, 0))
    with pytest.raises(ModelError, match="Division by zero"):
        _eval1([(COL, 0), (COL, 1), (MOD,)], _one(U64, 5), _one(U64, 0))
    with pytest.raises(ModelError, match="INT_MIN by -1"):
        _eval1([(COL, 0), (COL, 1), (DIV,)], _one(I64, mn), _one(I64, m1))
    with pytest.raises(ModelError, match="INT_MIN by -1"):
        _eval1([(COL, 0), (COL, 1), (MOD,)], _one(I64, mn), _one(I64, m1))
    assert _eval1([(COL, 0), (COL, 1), (DIV,)], _one(U64, mn), _one(U64, m1)) == 0  # unsigned: no such case


def test_model_double_and_cast_rules():
    nan, inf = _bits(math.nan), _bits(math.inf)
    d = lambda prog, *xs: _eval1(prog, *[_one(DBL, _bits(x)) for x in xs])  # noqa: E731
    assert _f(d([(COL, 0), (COL, 1), (DIV,)], 1.0, 0.0)) == math.inf
    assert _f(d([(COL, 0), (COL, 1), (DIV,)], 1.0, -0.0)) == -math.inf
    assert math.isnan(_f(d([(COL, 0), (COL, 1), (DIV,)], 0.0, 0.0)))
    assert d([(COL, 0), (NEG,)], 0.0) == _bits(-0.0) and d([(COL, 0), (NEG,)], -0.0) == 0
    assert _eval1([(COL, 0), (NEG,)], _one(DBL, nan)) == nan ^ INT64_MIN                           # sign bit of NaN
    assert _f(d([(COL, 0), (COL, 1), (ADD,)], 0.1, 0.2)) == 0.1 + 0.2
    assert _f(d([(COL, 0), (COL, 1), (SUB,)], math.inf, math.inf)) != _f(d([(COL, 0), (COL, 1), (SUB,)], math.inf, math.inf))
    to = lambda frm, t, x: _eval1([(COL, 0), (CAST, 0, t)], _one(frm, x))  # noqa: E731
    # integer -> double rounds to nearest
    assert to(I64, DBL, 2**53 + 1) == _bits(float(2**53)) and to(I64, DBL, 2**53 + 3) == _bits(float(2**53 + 4))
    assert to(U64, DBL, M64) == _bits(2.0**64) and to(I64, DBL, INT64_MIN) == _bits(-2.0**63)
    assert to(U64, DBL, (1 << 63) + 1025) == _bits(float((1 << 63) + 2048))
    # double -> integer truncates and saturates; NaN -> 0
    assert to(DBL, I64, _bits(-2.7)) == (-2) & M64 and to(DBL, U64, _bits(2.7)) == 2
    assert to(DBL, I64, _bits(2.0**63)) == (1 << 63) - 1 and to(DBL, I64, _bits(-2.0**63)) == INT64_MIN
    assert to(DBL, I64, _bits(-math.inf)) == INT64_MIN and to(DBL, I64, inf) == (1 << 63) - 1
    assert to(DBL, U64, _bits(2.0**63)) == 1 << 63 and to(DBL, U64, _bits(2.0**64)) == M64 and to(DBL, U64, inf) == M64
    assert to(DBL, U64, _bits(-1.0)) == 0 and to(DBL, U64, _bits(-0.5)) == 0 and to(DBL, U64, _bits(-math.inf)) == 0
    assert to(DBL, I64, nan) == 0 and to(DBL, U64, nan) == 0 and to(DBL, I64, _bits(-0.0)) == 0
    # int64 <-> uint64 keeps the bits; BOOLEAN is 0 / 1
    assert to(I64, U64, M64) == M64 and to(U64, I64, INT64_MIN) == INT64_MIN
    assert to(BOOL, DBL, 1) == _bits(1.0) and to(BOOL, I64, 1) == 1 and to(BOOL, U64, 0) == 0
    assert to(DBL, DBL, nan) == nan


def test_model_nulls_if_null_and_selection():
    a = (I64, np.array([1, 2, 0, 4], np.uint64), np.array([False, True, False, True]))
    b = (I64, np.array([10, 20, 0, 40], np.uint64), np.array([False, False, True, True]))
    t, v, nl = model([a, b], [(COL, 0), (COL, 1), (ADD,)], 4)
    assert v.tolist() == [11, 0, 0, 0] and nl.tolist() == [False, True, True, True]
    t, v, nl = model([a, b], [(COL, 0), (COL, 1), (IFNULL,)], 4)
    assert v.tolist() == [1, 20, 0, 0] and nl.tolist() == [False, False, False, True]
    # a NULL divisor never fails, a zero divisor outside the selection never fails, inside it does
    t, v, nl = model([a, b], [(COL, 0), (COL, 1), (DIV,)], 4)
    assert nl.tolist() == [False, True, True, True] and v.tolist() == [0, 0, 0, 0]
    z = (I64, np.array([5, 0, 5, 5], np.uint64), np.zeros(4, bool))
    assert model_error([a, z], [(COL, 0), (COL, 1), (DIV,)], 4) is None  # the zero sits next to a NULL dividend
    a2 = (I64, np.array([1, 2, 3, 4], np.uint64), np.zeros(4, bool))
    assert model_error([a2, z], [(COL, 0), (COL, 1), (DIV,)], 4) == "Division by zero"
    t, v, nl = model([a2, z], [(COL, 0), (COL, 1), (DIV,)], 4, selection=[True, False, True, False])
    assert nl.tolist() == [False, True, False, True] and v.tolist() == [0, 0, 0, 0]
    t, v, nl = model([a2], [(CONST, 0, I64, 7)], 4, selection=[True, False, True, True])
    assert v.tolist() == [7, 0, 7, 7] and nl.tolist() == [False, True, False, False]
    assert model([(BOOL, np.array([0, 5], np.uint64), np.zeros(2, bool))], [(COL, 0)], 2)[1].tolist() == [0, 1]


HEADER_PROGRAM = r"""
#include <stdio.h>
#include <stddef.h>
#include "include/ytgpu.h"
int main(void) {
    ytgpu_expr_node n = {YTGPU_EXPR_CAST, 0, YTGPU_TYPE_DOUBLE, {0}, 0};
    printf("%zu %zu %zu %d %d %d %d %d\n", sizeof(ytgpu_expr_node), offsetof(ytgpu_expr_node, type), offsetof(ytgpu_expr_node, constant),
           YTGPU_EXPR_COLUMN, YTGPU_EXPR_IF_NULL, YTGPU_EXPR_MAX_NODES, YTGPU_EXPR_MAX_DEPTH, n.op);
    return 0;
}
"""


def test_header_compiles_as_c99_and_the_node_matches_the_binding():
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "e.c"), os.path.join(d, "e")
        open(src, "w").write(HEADER_PROGRAM)
        subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", ROOT, src, "-o", exe])
        out = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    assert out == [C.sizeof(capi.ExprNode), capi.ExprNode.type.offset, capi.ExprNode.constant.offset, capi.EXPR_COLUMN,
                   capi.EXPR_IF_NULL, capi.EXPR_MAX_NODES, capi.EXPR_MAX_DEPTH, capi.EXPR_CAST]
    assert C.sizeof(capi.ExprNode) == 24


def test_entry_point_is_declared_and_exported():
    lib = capi.load()
    assert "ytgpu_evaluate_expression" in capi.EXPORTED_SYMBOLS and hasattr(lib, "ytgpu_evaluate_expression")
    assert "ytgpu_evaluate_expression(" in open(os.path.join(ROOT, "include", "ytgpu.h")).read()


def random_program(rng, col_types, result_type=None, max_nodes=64, max_depth=16, divisor_or_one=0.7):
    """A random well-typed postfix program of at most max_nodes nodes and stack depth <= max_depth over columns of
    col_types.  A DIV / MOD divisor is made odd (x | 1, never 0) with probability divisor_or_one."""
    def leaf(t):
        cols = [i for i, ct in enumerate(col_types) if ct == t]
        if cols and rng.random() < 0.75:
            return [(COL, int(rng.choice(cols)))]
        if t == DBL:
            c = _bits(float(rng.choice([0.0, -0.0, 1.5, -3.0, 1e300, math.inf, math.nan, 7.0])))
        elif t == BOOL:
            c = int(rng.integers(0, 2))
        else:
            c = int(rng.choice([0, 1, 2, 3, 7, 1000, M64, INT64_MIN, (1 << 63) - 1, 2**53 + 1]))
        return [(CONST, 0, t, c)]

    def build(budget, t):  # -> postfix
        if budget <= 1 or rng.random() < 0.12:
            if t != BOOL and rng.random() < 0.2 and budget >= 2:
                return build(budget - 1, TYPES[int(rng.integers(0, 4))]) + [(CAST, 0, t)]
            return leaf(t)
        r = rng.random()
        if r < 0.2 and budget >= 2:
            ops = [op for op, ts in UNARY.items() if t in ts] + ([CAST] if t != BOOL else [])
            if ops:
                op = int(rng.choice(ops))
                if op == CAST:
                    return build(budget - 1, TYPES[int(rng.integers(0, 4))]) + [(CAST, 0, t)]
                return build(budget - 1, t) + [(op,)]
        if budget < 3:
            return leaf(t)
        op = int(rng.choice([op for op, ts in BINARY.items() if t in ts]))
        left = int(rng.integers(1, budget - 1))
        a = build(left, t)
        b = build(budget - 1 - left, t)
        if op in (DIV, MOD) and t != DBL and rng.random() < divisor_or_one:
            b = b + [(CONST, 0, t, 1), (BOR,)]
        return a + b + [(op,)]

    while True:
        t = result_type if result_type is not None else TYPES[int(rng.integers(0, 4))]
        prog = build(int(rng.integers(1, max_nodes + 1)), t)
        if len(prog) <= max_nodes and stack_depth(prog) <= max_depth:
            return prog


def stack_depth(prog):
    d = m = 0
    for node in prog:
        op = node[0]
        d += 1 if op in (COL, CONST) else (0 if op in (NEG, BNOT, CAST) else -1)
        m = max(m, d)
    return m


def test_random_programs_respect_the_limits_and_are_well_typed():
    rng = np.random.default_rng(5)
    col_types = [I64, U64, DBL, BOOL]
    sizes, depths = [], []
    for _ in range(400):
        p = random_program(rng, col_types)
        assert 1 <= len(p) <= 64 and stack_depth(p) <= 16
        program_types(col_types, p)  # raises for a mistyped program
        sizes.append(len(p))
        depths.append(stack_depth(p))
    assert max(sizes) >= 48 and max(depths) >= 6
    ops = {node[0] for _ in range(50) for node in random_program(rng, col_types)}
    assert ops == set(range(COL, IFNULL + 1))


def test_host_adapter_builds_and_refuses_cpu():
    import torch
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "expression_ut"], stdout=subprocess.DEVNULL)
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([os.path.join(ROOT, "host", "expression_ut")], capture_output=True, text=True, timeout=120)
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


def _copy(cols, device):
    import copy
    cols = [copy.copy(c) for c in cols]
    return [to_device(c) for c in cols] if device else cols


def _sel_bitmap(selection, n, device):
    if selection is None:
        return None
    words = (n + 63) // 64
    bm = np.zeros(words * 8, np.uint8)
    packed = _bm(selection)
    bm[:len(packed)] = packed
    if device:
        import torch
        return torch.from_numpy(bm).cuda()
    return bm


def run(ctx, data, cols, program, n, selection=None, device=False):
    """Evaluates on the GPU and checks it against the model, bit for bit; a division error must be the model's."""
    want_err = model_error(data, program, n, selection)
    sel = _sel_bitmap(selection, n, device)
    if want_err is not None:
        with pytest.raises(capi.YtGpuError) as e:
            ctx.evaluate_expression(_copy(cols, device), program, sel)
        assert e.value.code == capi.ERR_INVALID_ARGUMENT and e.value.message == want_err, (program, e.value.message)
        return None
    t, v, nl = model(data, program, n, selection)
    got = ctx.evaluate_expression(_copy(cols, device), program, sel)
    assert got["value_type"] == t
    gv = host(got["values"]).view(np.uint64)
    bits = np.unpackbits(host(got["null_bitmap"]), bitorder="little").astype(bool)
    assert len(host(got["null_bitmap"])) == 8 * ((n + 63) // 64)
    differ = gv != v
    if t == DBL:  # the sign and payload of a NaN an operation produces are unspecified
        with np.errstate(invalid="ignore"):
            differ &= ~(np.isnan(gv.view(np.float64)) & np.isnan(v.view(np.float64)))
    bad = np.flatnonzero(differ | (bits[:n] != nl))
    assert bad.size == 0, (program, bad[:5], gv[bad[:5]], v[bad[:5]], nl[bad[:5]])
    assert not bits[n:].any()
    assert got["null_count"] == int(nl.sum())
    return got


def _nonzero_divisor(vtype, bits):
    """The same values with 0 and -1 replaced, so DIV / MOD over every encoding of the dividend never fail."""
    bits = bits.copy()
    if vtype in INTEGER:
        bits[bits == 0] = 7
        bits[bits == np.uint64(M64)] = 3
    return bits


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("vtype", TYPES, ids=["i64", "u64", "f64", "bool"])
def test_gpu_every_op_over_every_encoding_and_window(ctx, vtype, device):
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(vtype * 11 + int(device))
    n = 300
    kinds = F.BOOL_ENCODINGS if vtype == BOOL else F.ENCODINGS
    for kind in kinds:
        for start in (0, 1, 3):
            col, bits, nulls = make_column(kind, vtype, n, start, rng)
            obits = _nonzero_divisor(vtype, edge_values(rng, vtype, n))
            onulls = rng.random(n) < 0.15
            other = Column(vtype, values=obits, null_bitmap=_bm(onulls), value_count=n)
            data = [(vtype, bits, nulls), (vtype, obits, onulls)]
            const = int(edge_values(rng, vtype, 1)[0]) if vtype != BOOL else 1
            if vtype in INTEGER:
                const = const if const not in (0, M64) else 5
            programs = [[(COL, 0)], [(COL, 0), (COL, 1), (IFNULL,)], [(COL, 1), (COL, 0), (IFNULL,)],
                        [(COL, 0), (CONST, 0, vtype, const), (IFNULL,)]]
            programs += [[(COL, 0), (CAST, 0, t)] for t in NUMBER]
            programs += [[(COL, 0), (op,)] for op, ts in UNARY.items() if vtype in ts]
            for op, ts in BINARY.items():
                if vtype in ts and op != IFNULL:
                    programs += [[(COL, 0), (COL, 1), (op,)], [(COL, 0), (CONST, 0, vtype, const), (op,)]]
                    if op not in (DIV, MOD):
                        programs.append([(COL, 1), (COL, 0), (op,)])
            for prog in programs:
                run(ctx, data, [col, other], prog, n, device=device)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_random_programs_at_every_size(ctx, device):
    rng = np.random.default_rng(17 + int(device))
    specs = [("plain", I64), ("rle", U64), ("bitmap", DBL), ("bits_nulls", BOOL), ("dict", I64), ("packed", U64), ("arrow", DBL),
             ("w16", I64)]
    for n in (0, 1, 31, 32, 33, 4097):
        for rep in range(8):
            cols, data = [], []
            for kind, vt in specs:
                c, b, nl = make_column(kind, vt, n, int(rng.integers(1, 4)), rng)  # windows at 0 are in the encoding test
                cols.append(c)
                data.append((vt, b, nl))
            prog = random_program(rng, [d[0] for d in data])
            selection = rng.random(n) < 0.7 if rep % 3 == 2 else None
            run(ctx, data, cols, prog, n, selection, device=device)


@pytest.mark.gpu
def test_gpu_random_programs_ten_million_rows(ctx):
    rng = np.random.default_rng(29)
    n = 10**7
    cols, data = [], []
    for kind, vt in [("plain", I64), ("rle", U64), ("bitmap", DBL), ("bits_nulls", BOOL), ("dict", I64)]:
        c, b, nl = make_column(kind, vt, n, 1, rng)
        cols.append(c)
        data.append((vt, b, nl))
    for device in (False, True):
        prog = random_program(rng, [d[0] for d in data], result_type=I64, divisor_or_one=1.0)
        while len(prog) < 12:
            prog = random_program(rng, [d[0] for d in data], result_type=I64, divisor_or_one=1.0)
        run(ctx, data, cols, prog, n, device=device)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_selection_and_division_errors(ctx, device):
    from ytsaurus_b200 import Column
    n = 1000
    rng = np.random.default_rng(31)
    a = rng.integers(-100, 100, n, dtype=np.int64).view(np.uint64)
    b = rng.integers(1, 9, n, dtype=np.int64).view(np.uint64)
    anull = np.zeros(n, bool)
    b[[5, 700]] = 0  # two zero divisors
    anull[700] = True  # ... one of them next to a NULL dividend
    a[900], b[900] = np.uint64(INT64_MIN), np.uint64(M64)
    sel = np.ones(n, bool)
    sel[[5, 900]] = False
    cols = [Column(I64, values=a, null_bitmap=_bm(anull), value_count=n), Column(I64, values=b, value_count=n)]
    data = [(I64, a, anull), (I64, b, np.zeros(n, bool))]
    for op in (DIV, MOD):
        prog = [(COL, 0), (COL, 1), (op,)]
        got = run(ctx, data, cols, prog, n, sel, device)  # unselected rows come back NULL; rows 5 and 900 do not fail
        nb = np.unpackbits(host(got["null_bitmap"]), bitorder="little")[:n].astype(bool)
        assert nb[~sel].all() and nb[700]
        for row, msg in ((5, "Division by zero"), (900, "Division INT_MIN by -1")):
            s2 = sel.copy()
            s2[row] = True
            assert model_error(data, prog, n, s2) == msg
            run(ctx, data, cols, prog, n, s2, device)  # checks the error and its message
        assert model_error(data, prog, n) == "Division by zero"
        run(ctx, data, cols, prog, n, None, device)
    # an all-clear selection: everything NULL, nothing fails
    got = run(ctx, data, cols, [(COL, 0), (CONST, 0, I64, 0), (DIV,)], n, np.zeros(n, bool), device)
    assert got["null_count"] == n
    # doubles never fail
    run(ctx, [(DBL, np.zeros(n, np.uint64), np.zeros(n, bool))], [Column(DBL, values=np.zeros(n, np.uint64), value_count=n)],
        [(COL, 0), (COL, 0), (DIV,)], n, None, device)


def _code(fn):
    try:
        fn()
    except capi.YtGpuError as e:
        return e.code
    return capi.OK


@pytest.mark.gpu
def test_gpu_limits_and_errors(ctx):
    import torch

    from ytsaurus_b200 import Column
    rng = np.random.default_rng(71)
    n = 100
    i64, _, _ = make_column("bitmap", I64, n, 0, rng)
    u64, _, _ = make_column("plain", U64, n, 0, rng)
    f64, _, _ = make_column("bitmap", DBL, n, 0, rng)
    b1, _, _ = make_column("bits", BOOL, n, 0, rng)
    inv = capi.ERR_INVALID_ARGUMENT

    def ev(prog, cols=None):
        return lambda: ctx.evaluate_expression(_copy(cols or [i64, u64, f64, b1], False), prog)
    leaf = (COL, 0)
    chain = [leaf] + [leaf, (ADD,)] * 31 + [(NEG,)]  # 64 nodes
    assert len(chain) == 64 and _code(ev(chain)) == capi.OK
    assert _code(ev(chain + [(NEG,)])) == inv
    deep = [leaf] * 16 + [(ADD,)] * 15
    assert _code(ev(deep)) == capi.OK
    assert _code(ev([leaf] * 17 + [(ADD,)] * 16)) == inv
    assert _code(ev([])) == inv
    # malformed programs
    assert _code(ev([(ADD,)])) == inv and _code(ev([leaf, (ADD,)])) == inv and _code(ev([(NEG,)])) == inv
    assert _code(ev([leaf, leaf])) == inv
    assert _code(ev([(0, 0)])) == inv and _code(ev([(15, 0)])) == inv
    assert _code(ev([(COL, 4)])) == inv and _code(ev([(COL, -1)])) == inv
    assert _code(ev([(CONST, 0, 0x10, 0)])) == inv and _code(ev([(CONST, 0, 0x02, 0)])) == inv  # STRING / NULL constants
    assert _code(ev([(CONST, 0, BOOL, 2)])) == inv and _code(ev([(CONST, 0, BOOL, 1)])) == capi.OK
    # operand types
    assert _code(ev([(COL, 0), (COL, 1), (ADD,)])) == inv                      # int64 + uint64: no widening
    assert _code(ev([(COL, 0), (CAST, 0, U64), (COL, 1), (ADD,)])) == capi.OK
    assert _code(ev([(COL, 2), (COL, 2), (MOD,)])) == inv                      # MOD of doubles
    assert _code(ev([(COL, 2), (BNOT,)])) == inv and _code(ev([(COL, 2), (COL, 2), (BAND,)])) == inv
    for op in (ADD, SUB, MUL, DIV, MOD, BAND, BOR, BXOR):
        assert _code(ev([(COL, 3), (COL, 3), (op,)])) == inv                   # arithmetic on booleans
    assert _code(ev([(COL, 3), (NEG,)])) == inv and _code(ev([(COL, 3), (COL, 3), (IFNULL,)])) == capi.OK
    assert _code(ev([(COL, 3), (CAST, 0, BOOL)])) == inv and _code(ev([(COL, 0), (CAST, 0, 0x10)])) == inv
    assert _code(ev([(COL, 3), (CAST, 0, DBL)])) == capi.OK
    # unsupported column type; row counts
    scol = Column(T.String, values=np.zeros(n, np.uint64), value_count=n)
    assert _code(ev([(COL, 0)], cols=[u64, scol])) == capi.OK          # a column the program does not read
    assert _code(ev([(COL, 0)], cols=[scol])) == capi.ERR_UNSUPPORTED
    short, _, _ = make_column("plain", I64, n - 1, 0, rng)
    assert _code(ev([leaf], cols=[i64, short])) == inv
    # fewer than 2^32 rows: an all-NULL DEVICE column (no data) of 2^32 rows is refused before anything is read or written
    v = capi.ColumnView()
    v.value_count, v.value_type, v.has_values, v.bit_width, v.mem = 2**32, I64, 0, 64, capi.MEM_DEVICE
    nodes = (capi.ExprNode * 1)()
    nodes[0].op = COL
    values = torch.empty(1, dtype=torch.int64, device="cuda")
    nulls = torch.empty(8, dtype=torch.uint8, device="cuda")
    err = capi.Error()
    code = ctx.lib.ytgpu_evaluate_expression(ctx.handle, C.cast(C.pointer(v), C.c_void_p), 1, C.cast(nodes, C.c_void_p), 1, None,
                                             values.data_ptr(), nulls.data_ptr(), None, None, capi.MEM_DEVICE, C.byref(err))
    assert code == inv and b"2^32" in err.message
    # an all-NULL column: every row NULL, values 0
    allnull = Column(I64, values=None, value_count=n)
    got = ctx.evaluate_expression([allnull], [(COL, 0), (NEG,)])
    assert got["null_count"] == n and not host(got["values"]).any() and got["column"].null_bitmap is not None


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_launch_count(ctx, device):
    rng = np.random.default_rng(73)
    n = 10000
    col, bits, nulls = make_column("rle", I64, n, 1, rng)
    prog = [(COL, 0), (CONST, 0, I64, 1000), (MOD,), (COL, 0), (IFNULL,)]
    c = _copy([col], device)
    before = ctx.launch_count()
    got = ctx.evaluate_expression(c, prog)
    assert ctx.launch_count() - before == 1
    assert got["null_count"] == int(model([(I64, bits, nulls)], prog, n)[2].sum())
    before = ctx.launch_count()
    ctx.evaluate_expression(c, prog, _sel_bitmap(rng.random(n) < 0.5, n, device))
    assert ctx.launch_count() - before == 1


def _precomputed(vtype, values, nulls, device):
    from ytsaurus_b200 import Column
    col = Column(vtype, values=values.copy(), value_count=len(values), null_bitmap=_bm(nulls) if nulls.any() else None)
    return _copy([col], device)[0]


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_computed_column_in_groupby_and_filter(ctx, device):
    """The computed column as a GROUP BY key and as SUM / MIN / ARGMAX arguments, and under a filter, against the same values
    computed by the model and passed as a plain column."""
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(83 + int(device))
    n = 50_000
    acol, abits, anull = make_column("bitmap", I64, n, 0, rng)
    dcol, dbits, dnull = make_column("rle", DBL, n, 2, rng)
    kbits = rng.integers(0, 5, n, dtype=np.uint64)
    kcol = Column(U64, values=kbits, value_count=n)
    data = [(I64, abits, anull), (DBL, dbits, dnull)]
    key_prog = [(COL, 0), (CONST, 0, I64, 7), (MOD,)]                                     # a % 7
    val_prog = [(COL, 1), (CONST, 0, DBL, _bits(100.0)), (MUL,), (CAST, 0, I64), (COL, 0), (IFNULL,)]  # if_null(int64(d * 100), a)
    cols = _copy([acol, dcol], device)
    kc = _copy([kcol], device)[0]
    key = ctx.evaluate_expression(cols, key_prog)
    val = ctx.evaluate_expression(cols, val_prog)
    kt, kv, kn = model(data, key_prog, n)
    vt, vv, vn = model(data, val_prog, n)
    assert key["null_count"] == int(kn.sum()) and val["null_count"] == int(vn.sum())
    aggs = [(capi.AGG_SUM, 0), (capi.AGG_MIN, 0), (capi.AGG_ARGMAX, 1, 0), (capi.AGG_COUNT, 0)]
    got = ctx.scan_filter_groupby_multi([key["column"], kc], [val["column"], kc], aggs)
    want = ctx.scan_filter_groupby_multi([_precomputed(kt, kv, kn, device), kc], [_precomputed(vt, vv, vn, device), kc], aggs)
    F._check_same_groupby(got, want)
    assert len(host(got["count"])) > 20
    # with a predicate on the computed column
    got = ctx.scan_filter_groupby_multi([key["column"]], [val["column"]], aggs[:2], predicate=(capi.CMP_GT, 0), predicate_column=0)
    want = ctx.scan_filter_groupby_multi([_precomputed(kt, kv, kn, device)], [_precomputed(vt, vv, vn, device)], aggs[:2],
                                         predicate=(capi.CMP_GT, 0), predicate_column=0)
    F._check_same_groupby(got, want)
    # under a filter: a + b > 10 style, and an IS_NULL test
    fprog = [(capi.FILTER_COMPARE, capi.CMP_GT, 0, 0, 10, 0), (capi.FILTER_IS_NULL, 0, 1), (capi.FILTER_OR,)]
    got = ctx.evaluate_filter([val["column"], key["column"]], (), fprog)
    want = ctx.evaluate_filter([_precomputed(vt, vv, vn, device), _precomputed(kt, kv, kn, device)], (), fprog)
    for k in ("bitmap", "bytemap", "rows"):
        assert np.array_equal(host(got[k]), host(want[k]))
    assert got["count"] == want["count"] > 0
    # the filter's bitmap as the selection of the next expression
    sel = ctx.evaluate_expression(cols, val_prog, got["bitmap"])
    st, sv, sn = model(data, val_prog, n, host(got["bytemap"]).astype(bool))
    assert np.array_equal(host(sel["values"]).view(np.uint64), sv)
    assert np.array_equal(np.unpackbits(host(sel["null_bitmap"]), bitorder="little")[:n].astype(bool), sn)


@pytest.mark.gpu
def test_gpu_host_adapter_computed_columns():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "expression_ut"], stdout=subprocess.DEVNULL)
    r = subprocess.run([os.path.join(ROOT, "host", "expression_ut")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "expression_ut: 0 failure(s)" in r.stdout
