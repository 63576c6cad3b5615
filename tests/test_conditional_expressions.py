"""Conditional computed columns on the GPU: COMPARE, AND / OR / NOT, IS_NULL / IS_NOT_NULL and IF (csrc/expression.cu)
against a numpy model of include/ytgpu.h.

The model extends the one of test_expressions.py to every op and type, strings included.  Each stack entry carries its
rows' values, NULL flags and error bits (a division by zero, INT64_MIN / -1, a non-ASCII LOWER / UPPER operand).  Every op
passes on the union of its operands' bits, except that IF keeps the condition's and the taken branch's bits, and that
FALSE AND x and TRUE OR x drop x's; only the result's bits fail the call.  COMPARE is the filter's rule and NULL when an
operand is NULL; AND / OR / NOT are Kleene; a NULL IF condition gives NULL.  Results are compared bit for bit (strings byte
for byte); any two NaNs of a DOUBLE result match, as in test_expressions.py."""
import importlib.util
import math
import operator
import os
import subprocess
import tempfile

import numpy as np
import pytest

from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import EValueType as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name):
    """A sibling test module's helpers, loaded by path so no import mode matters."""
    spec = importlib.util.spec_from_file_location("_cond_" + name[:-3], os.path.join(os.path.dirname(os.path.abspath(__file__)), name))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


E = _load("test_expressions.py")         # the numeric model's pieces
S = _load("test_string_expressions.py")  # string columns, farm_hash
F = E.F                                  # column encodings

(COL, CONST, ADD, SUB, MUL, DIV, MOD, NEG, BAND, BOR, BXOR, BNOT, CAST, IFNULL, CONCAT, LOWER, UPPER, FARM) = range(1, 19)
(CMP, AND, OR, NOT, ISNULL, ISNOTNULL, IF) = (capi.EXPR_COMPARE, capi.EXPR_AND, capi.EXPR_OR, capi.EXPR_NOT, capi.EXPR_IS_NULL,
                                             capi.EXPR_IS_NOT_NULL, capi.EXPR_IF)
LT, LE, GT, GE, EQ, NE = capi.CMP_LT, capi.CMP_LE, capi.CMP_GT, capi.CMP_GE, capi.CMP_EQ, capi.CMP_NE
CMPS = (LT, LE, GT, GE, EQ, NE)
I64, U64, DBL, BOOL, STR = int(T.Int64), int(T.Uint64), int(T.Double), int(T.Boolean), int(T.String)
TYPES = [I64, U64, DBL, BOOL]
M64 = (1 << 64) - 1
INT64_MIN = 1 << 63
ERR_DIV0, ERR_INTMIN, ERR_ASCII = 1, 2, 4
_bits, _f = E._bits, E._f


# ------------------------------------------------------------------------------------------------- the model
class ModelError(Exception):
    """A failed call: code and message (UNSUPPORTED for non-ASCII, INVALID_ARGUMENT for a division error)."""

    def __init__(self, code, message):
        super().__init__(message)
        self.code, self.message = code, message


_PY_CMP = {LT: operator.lt, LE: operator.le, GT: operator.gt, GE: operator.ge, EQ: operator.eq, NE: operator.ne}


def _compare(cmp, t, a, b, nl):
    """COMPARE over non-NULL rows (nl: either operand NULL) -> bool array."""
    if t == STR:
        return np.array([not z and _PY_CMP[cmp](x, y) for x, y, z in zip(a, b, nl)], bool)
    return F.scalar_cmp(cmp, t, a, b) & ~nl


def _strings(values):
    return np.array([v is None for v in values], bool)


def _zero(t, v, nl):
    """The entry invariant: a NULL row holds 0 (None for a STRING)."""
    if t == STR:
        return [None if z else x for x, z in zip(v, nl)]
    return np.where(nl, np.uint64(0), v)


def _binary(op, t, a, b, nl):
    """Arithmetic / bitwise over non-NULL rows -> (values, error bits)."""
    r = E._binary(op, t, a, b, np.zeros(len(a), bool))  # no row counts as evaluated: the model's errors are masks here
    e = np.zeros(len(a), np.uint8)
    if op in (DIV, MOD) and t != DBL:
        e[~nl & (b == 0)] |= ERR_DIV0
        if t == I64:
            e[~nl & (a == np.uint64(INT64_MIN)) & (b == np.uint64(M64))] |= ERR_INTMIN
    return r, e


def evaluate(cols, program, n, selection=None, consts=b""):
    """cols: per input column (type, values, nulls): uint64 bits for a scalar, a list of bytes / None for a STRING (nulls
    unused).  -> (type, values, nulls, error bits per row); rows outside the selection are NULL and error-free."""
    sel = np.ones(n, bool) if selection is None else np.asarray(selection, bool)
    st = []  # (type, values, nulls, errors)
    with np.errstate(all="ignore"):
        for node in program:
            op, column, vtype, constant = (tuple(node) + (0,) * 4)[:4]
            z8 = np.zeros(n, np.uint8)
            if op in (COL, CONST):
                if op == COL:
                    t, vals, nulls = cols[column]
                else:
                    t = vtype
                    if t == STR:
                        s = consts[constant >> 32:(constant >> 32) + (constant & 0xFFFFFFFF)]
                        vals = [s] * n
                    else:
                        vals, nulls = np.full(n, int(constant) & M64, np.uint64), np.zeros(n, bool)
                if t == STR:
                    v = [x if k else None for x, k in zip(vals, sel)]
                    st.append((STR, v, _strings(v), z8))
                else:
                    bits = np.asarray(vals, np.uint64)
                    if t == BOOL:
                        bits = (bits != 0).astype(np.uint64)
                    nl = np.asarray(nulls, bool) | ~sel
                    st.append((t, _zero(t, bits, nl), nl, z8))
            elif op in (NEG, BNOT, CAST):
                t, a, nl, e = st.pop()
                if op == NEG:
                    r = a ^ E.SIGN if t == DBL else np.uint64(0) - a
                elif op == BNOT:
                    r = ~a
                else:
                    r, t = E._cast(t, vtype, a), vtype
                st.append((t, _zero(t, r, nl), nl, e))
            elif op in (LOWER, UPPER):
                t, a, nl, e = st.pop()
                bad = np.array([x is not None and any(ch >= 0x80 for ch in x) for x in a], bool)
                r = [x if (x is None or b) else (x.lower() if op == LOWER else x.upper()) for x, b in zip(a, bad)]
                st.append((STR, r, nl, e | np.where(bad, ERR_ASCII, 0).astype(np.uint8)))
            elif op == FARM:
                ops = st[len(st) - column:]
                del st[len(st) - column:]
                h = [S.farm_hash([(t, None if nl[i] else (v[i] if t == STR else int(v[i]))) for t, v, nl, _ in ops]) for i in range(n)]
                e = z8
                for *_, oe in ops:
                    e = e | oe
                st.append((U64, np.array(h, np.uint64), np.zeros(n, bool), e))
            elif op == NOT:
                t, a, nl, e = st.pop()
                st.append((BOOL, _zero(BOOL, a ^ np.uint64(1), nl), nl, e))
            elif op in (ISNULL, ISNOTNULL):
                t, a, nl, e = st.pop()
                st.append((BOOL, (nl if op == ISNULL else ~nl).astype(np.uint64), np.zeros(n, bool), e))
            elif op == IF:
                tb, b, nb, eb = st.pop()
                ta, a, na, ea = st.pop()
                tc, c, nc, ec = st.pop()
                ct, cf = ~nc & (c == 1), ~nc & (c == 0)
                nl = nc | (ct & na) | (cf & nb)
                if ta == STR:
                    v = [x if t_ else (y if f_ else None) for x, y, t_, f_ in zip(a, b, ct, cf)]
                else:
                    v = _zero(ta, np.where(ct, a, b), nl)
                st.append((ta, v, nl, ec | np.where(ct, ea, np.where(cf, eb, 0)).astype(np.uint8)))
            else:
                tb, b, nb, eb = st.pop()
                ta, a, na, ea = st.pop()
                assert ta == tb, "mistyped program"
                e = ea | eb
                if op == IFNULL:
                    nl = na & nb
                    v = [y if x is None else x for x, y in zip(a, b)] if ta == STR else np.where(na, b, a)
                    st.append((ta, v, nl, e))
                elif op == CONCAT:
                    nl = na | nb
                    st.append((STR, [None if z else x + y for x, y, z in zip(a, b, nl)], nl, e))
                elif op == CMP:
                    nl = na | nb
                    st.append((BOOL, _compare(column, ta, a, b, nl).astype(np.uint64), nl, e))
                elif op in (AND, OR):
                    left = (~na & (a == 0)) if op == AND else (a == 1)  # the left operand decides
                    decided = left | ((~nb & (b == 0)) if op == AND else (b == 1))
                    nl = ~decided & (na | nb)
                    v = (a & b) if op == AND else (a | b)
                    st.append((BOOL, _zero(BOOL, v, nl), nl, np.where(left, ea, e).astype(np.uint8)))
                else:
                    nl = na | nb
                    r, e2 = _binary(op, ta, a, b, nl)
                    st.append((ta, _zero(ta, r, nl), nl, e | e2))
    assert len(st) == 1
    t, v, nl, e = st[0]
    nl = nl | ~sel  # FARM_HASH, IS_NULL and IS_NOT_NULL are never NULL, but an unselected row is
    return t, _zero(t, v, nl), nl, e


def model(cols, program, n, selection=None, consts=b""):
    """-> (type, values, nulls); raises ModelError when a row's result carries an error, in the library's order."""
    t, v, nl, e = evaluate(cols, program, n, selection, consts)
    bits = int(np.bitwise_or.reduce(e)) if n else 0
    if bits & ERR_ASCII:
        raise ModelError(capi.ERR_UNSUPPORTED, "0x80")
    if bits & ERR_DIV0:
        raise ModelError(capi.ERR_INVALID_ARGUMENT, "Division by zero")
    if bits & ERR_INTMIN:
        raise ModelError(capi.ERR_INVALID_ARGUMENT, "Division INT_MIN by -1")
    return t, v, nl


def _one(t, x):
    if t == STR:
        return (STR, [x], None)
    return (t, np.array([0 if x is None else x & M64], np.uint64), np.array([x is None]))


def ev1(program, *cols, consts=b""):
    """One row: the result value (None for NULL)."""
    t, v, nl = model(list(cols), program, 1, consts=consts)
    return None if nl[0] else (v[0] if t == STR else int(v[0]))


# ------------------------------------------------------------------------------------------------- CPU: hand-written cases
def test_kleene_tables():
    vals = {True: 1, False: 0, None: None}
    sql_and = lambda a, b: False if (a is False or b is False) else (None if (a is None or b is None) else True)  # noqa: E731
    sql_or = lambda a, b: True if (a is True or b is True) else (None if (a is None or b is None) else False)  # noqa: E731
    for a in (True, False, None):
        for b in (True, False, None):
            for op, f in ((AND, sql_and), (OR, sql_or)):
                got = ev1([(COL, 0), (COL, 1), (op,)], _one(BOOL, vals[a]), _one(BOOL, vals[b]))
                want = f(a, b)
                assert got == (None if want is None else int(want)), (op, a, b)
        got = ev1([(COL, 0), (NOT,)], _one(BOOL, vals[a]))
        assert got == (None if a is None else int(not a))
        assert ev1([(COL, 0), (ISNULL,)], _one(BOOL, vals[a])) == int(a is None)
        assert ev1([(COL, 0), (ISNOTNULL,)], _one(BOOL, vals[a])) == int(a is not None)


def test_comparison_rules():
    def c(t, cmp, a, b):
        return ev1([(COL, 0), (COL, 1), (CMP, cmp)], _one(t, a), _one(t, b))
    mn, m1 = INT64_MIN, M64
    assert c(I64, LT, mn, m1) == 1 and c(I64, LT, m1, 0) == 1 and c(I64, GT, 0, mn) == 1    # signed
    assert c(U64, GT, m1, 0) == 1 and c(U64, GT, 1 << 63, (1 << 63) - 1) == 1 and c(U64, LT, 0, m1) == 1  # unsigned
    nan, inf = _bits(math.nan), _bits(math.inf)
    for cmp in CMPS:
        assert c(DBL, cmp, nan, _bits(1.0)) == int(cmp == NE) and c(DBL, cmp, nan, nan) == int(cmp == NE)
    assert c(DBL, EQ, _bits(-0.0), _bits(0.0)) == 1 and c(DBL, LT, _bits(-0.0), _bits(0.0)) == 0
    assert c(DBL, LT, _bits(-math.inf), inf) == 1 and c(DBL, GE, inf, inf) == 1 and c(DBL, LT, _bits(-1e308), _bits(5e-324)) == 1
    assert c(BOOL, LT, 0, 1) == 1 and c(BOOL, EQ, 1, 1) == 1
    assert c(I64, EQ, None, 5) is None and c(STR, NE, b"x", None) is None   # NULL, the filter's rule
    assert c(STR, LT, b"abc", b"abd") == 1 and c(STR, LT, b"ab", b"abc") == 1 and c(STR, GT, b"ab\x00", b"ab") == 1
    assert c(STR, LT, b"", b"\x00") == 1 and c(STR, EQ, b"", b"") == 1 and c(STR, GT, b"\xff", b"\x7f\xff") == 1
    assert c(STR, LT, b"a\x00b", b"a\x01") == 1
    # piece lists: lower(x) against a constant, concat against a value
    k = bytearray()
    ex = S.constant(k, b"example.com")
    assert ev1([(COL, 0), (LOWER,), (CONST, 0, STR, ex), (CMP, EQ)], _one(STR, b"Example.COM"), consts=bytes(k)) == 1
    assert ev1([(COL, 0), (COL, 1), (CONCAT,), (COL, 2), (CMP, EQ)], _one(STR, b"ab"), _one(STR, b"c"), _one(STR, b"abc")) == 1


def test_if_rules():
    k = bytearray()
    a, b = S.constant(k, b"slow"), S.constant(k, b"fast")
    prog = [(COL, 0), (CONST, 0, STR, a), (CONST, 0, STR, b), (IF,)]
    assert ev1(prog, _one(BOOL, 1), consts=bytes(k)) == b"slow" and ev1(prog, _one(BOOL, 0), consts=bytes(k)) == b"fast"
    assert ev1(prog, _one(BOOL, None), consts=bytes(k)) is None                      # a NULL condition gives NULL
    num = [(COL, 0), (COL, 1), (COL, 2), (IF,)]
    assert ev1(num, _one(BOOL, 1), _one(I64, None), _one(I64, 7)) is None           # the taken branch's NULL
    assert ev1(num, _one(BOOL, 0), _one(I64, None), _one(I64, 7)) == 7
    assert ev1(num, _one(BOOL, None), _one(I64, 3), _one(I64, 7)) is None


def test_errors_follow_the_data():
    zero, two = _one(I64, 0), _one(I64, 2)
    eq0 = [(COL, 1), (CONST, 0, I64, 0), (CMP, EQ)]
    div = [(COL, 0), (COL, 1), (DIV,)]
    assert ev1(eq0 + [(CONST, 0, I64, 0)] + div + [(IF,)], two, zero) == 0                       # if(b = 0, 0, a / b)
    with pytest.raises(ModelError, match="Division by zero"):
        ev1(eq0 + div + [(CONST, 0, I64, 0), (IF,)], two, zero)                                  # if(b = 0, a / b, 0)
    gt1 = div + [(CONST, 0, I64, 1), (CMP, GT)]
    assert ev1([(CONST, 0, BOOL, 0)] + gt1 + [(AND,)], two, zero) == 0                           # FALSE AND (a / 0 > 1)
    with pytest.raises(ModelError, match="Division by zero"):
        ev1([(COL, 2)] + gt1 + [(AND,)], two, zero, _one(BOOL, None))                            # NULL AND (a / 0 > 1)
    assert ev1([(CONST, 0, BOOL, 1)] + gt1 + [(OR,)], two, zero) == 1                            # TRUE OR (a / 0 > 1)
    with pytest.raises(ModelError, match="Division by zero"):
        ev1(gt1 + [(CONST, 0, BOOL, 0), (AND,)], two, zero)                                      # the left operand is evaluated
    with pytest.raises(ModelError, match="Division by zero"):                                    # a NULL condition keeps its own
        ev1([(COL, 0), (COL, 1), (DIV,), (CONST, 0, I64, 1), (CMP, EQ), (CONST, 0, I64, 1), (CONST, 0, I64, 2), (IF,)], two, zero)
    assert ev1([(COL, 2), (COL, 0), (COL, 1), (DIV,), (CONST, 0, I64, 0), (IF,)], two, zero, _one(BOOL, None)) is None
    with pytest.raises(ModelError, match="Division by zero"):                                    # IF_NULL stays eager
        ev1([(COL, 0), (COL, 0), (COL, 1), (DIV,), (IFNULL,)], two, zero)
    with pytest.raises(ModelError, match="INT_MIN"):
        ev1([(CONST, 0, BOOL, 1), (COL, 0), (COL, 1), (DIV,), (CONST, 0, I64, 0), (IF,)], _one(I64, INT64_MIN), _one(I64, M64))
    # non-ASCII under LOWER: refused in the taken branch only
    k = bytearray()
    x = S.constant(k, b"x")
    lw = [(COL, 1), (LOWER,)]
    assert ev1([(COL, 0)] + [(CONST, 0, STR, x)] + lw + [(IF,)], _one(BOOL, 1), _one(STR, b"Stra\xc3\x9fe"), consts=bytes(k)) == b"x"
    with pytest.raises(ModelError, match="0x80"):
        ev1([(COL, 0)] + lw + [(CONST, 0, STR, x), (IF,)], _one(BOOL, 1), _one(STR, b"Stra\xc3\x9fe"), consts=bytes(k))


HEADER_PROGRAM = r"""
#include <stdio.h>
#include "include/ytgpu.h"
int main(void) {
    ytgpu_expr_node n = {YTGPU_EXPR_COMPARE, YTGPU_CMP_GE, 0, {0}, 0};
    printf("%d %d %d %d %d %d %d %d\n", n.op, YTGPU_EXPR_AND, YTGPU_EXPR_OR, YTGPU_EXPR_NOT, YTGPU_EXPR_IS_NULL,
           YTGPU_EXPR_IS_NOT_NULL, YTGPU_EXPR_IF, n.column);
    return 0;
}
"""


def test_header_compiles_as_c99_with_the_new_ops():
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "e.c"), os.path.join(d, "e")
        open(src, "w").write(HEADER_PROGRAM)
        subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", ROOT, src, "-o", exe])
        out = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    assert out == [CMP, AND, OR, NOT, ISNULL, ISNOTNULL, IF, GE] == [19, 20, 21, 22, 23, 24, 25, capi.CMP_GE]
    assert capi.EXPR_STRING_OPS == (CONCAT, LOWER, UPPER, FARM)


# ------------------------------------------------------------------------------------------------- random programs
_CONSTS = {I64: [0, 1, 2, 7, 1000, M64, INT64_MIN, (1 << 63) - 1], U64: [0, 1, 3, 1 << 63, M64],
           DBL: [_bits(x) for x in (0.0, -0.0, 1.5, -3.0, math.inf, math.nan)], BOOL: [0, 1]}
WORDS = [b"", b"a", b"AbC", b"ab\x00", b"https://www.site5", b"Z" * 40]


def limits(prog, str_cols):
    """(stack depth, the check's piece bound) of a program; str_cols: the column indexes that are STRINGs."""
    st, depth, top = [], 0, 0
    for node in prog:
        op = node[0]
        if op in (COL, CONST):
            st.append(1 if (op == COL and node[1] in str_cols) or (op == CONST and node[2] == STR) else 0)
        elif op in (CONCAT, IFNULL):
            b = st.pop()
            st[-1] = st[-1] + b if op == CONCAT else max(st[-1], b)
        elif op == IF:
            b, a = st.pop(), st.pop()
            st[-1] = max(a, b)
        elif op in (NOT, ISNULL, ISNOTNULL, NEG, BNOT, CAST, LOWER, UPPER):
            st[-1] = st[-1] if op in (LOWER, UPPER) else 0
        else:
            st.pop()
            st[-1] = 0
        depth, top = max(depth, len(st)), max(top, sum(st))
    return depth, top


def random_program(rng, col_types, consts=None, result_type=None, max_nodes=64):
    """A random well-typed program over columns of col_types, old and new ops mixed, within every limit.  With consts (a
    bytearray) STRING leaves, constants and ops take part.  A DIV / MOD divisor is guarded by an IF on it being 0, made
    odd, or left as it is."""
    types = TYPES + ([STR] if consts is not None else [])

    def leaf(t):
        cols = [i for i, ct in enumerate(col_types) if ct == t]
        if cols and rng.random() < 0.75:
            return [(COL, int(rng.choice(cols)))]
        if t == STR:
            return [(CONST, 0, STR, S.constant(consts, WORDS[int(rng.integers(0, len(WORDS)))]))]
        pool = _CONSTS[t]
        return [(CONST, 0, t, int(pool[int(rng.integers(0, len(pool)))]))]

    def pick(xs):
        return xs[int(rng.integers(0, len(xs)))]

    def build(budget, t):
        if budget <= 1 or rng.random() < 0.1:
            return leaf(t)
        r = rng.random()
        third = max(1, (budget - 1) // 3)
        half = max(1, (budget - 1) // 2)
        if budget >= 4 and r < 0.22:
            return build(third, BOOL) + build(third, t) + build(third, t) + [(IF,)]
        if t == BOOL and budget >= 3:
            k = rng.random()
            if k < 0.45:
                ot = pick(types)
                return build(half, ot) + build(half, ot) + [(CMP, pick(CMPS))]
            if k < 0.75:
                return build(half, BOOL) + build(half, BOOL) + [(pick([AND, OR]),)]
            if k < 0.85:
                return build(budget - 1, BOOL) + [(NOT,)]
            return build(budget - 1, pick(types)) + [(pick([ISNULL, ISNOTNULL]),)]
        if t == STR and budget >= 3:
            k = rng.random()
            if k < 0.4:
                return build(half, STR) + build(half, STR) + [(CONCAT,)]
            if k < 0.6:
                return build(budget - 1, STR) + [(pick([LOWER, UPPER]),)]
            if k < 0.8:
                return build(half, STR) + build(half, STR) + [(IFNULL,)]
            return leaf(t)
        if t in (I64, U64, DBL) and budget >= 3 and r < 0.7:
            op = pick([o for o, ts in E.BINARY.items() if t in ts])
            a, b = build(half, t), build(half, t)
            if op in (DIV, MOD) and t != DBL:
                g = rng.random()
                if g < 0.45:  # if(b = 0, 0, a / b)
                    return b + [(CONST, 0, t, 0), (CMP, EQ), (CONST, 0, t, 0)] + a + b + [(op,), (IF,)]
                if g < 0.9:
                    b = b + [(CONST, 0, t, 1), (BOR,)]
            return a + b + [(op,)]
        if t in (I64, U64, DBL) and r < 0.85:
            return build(budget - 1, pick(TYPES)) + [(CAST, 0, t)]
        if t in (I64, DBL) and r < 0.92:
            return build(budget - 1, t) + [(NEG,)]
        return leaf(t)

    str_cols = {i for i, t in enumerate(col_types) if t == STR}
    while True:
        t = result_type if result_type is not None else pick(types)
        prog = build(int(rng.integers(1, max_nodes + 1)), t)
        depth, pieces = limits(prog, str_cols)
        if len(prog) <= max_nodes and depth <= 16 and pieces <= 16:
            return prog


def test_random_programs_respect_the_limits_and_are_well_typed():
    rng = np.random.default_rng(7)
    col_types = [I64, U64, DBL, BOOL, STR]
    ops, sizes = set(), []
    n = 3
    cols = [(I64, np.array([1, 0, 5], np.uint64), np.array([False, False, True])),
            (U64, np.array([0, 2, 3], np.uint64), np.zeros(3, bool)),
            (DBL, np.array([_bits(1.0), _bits(math.nan), 0], np.uint64), np.zeros(3, bool)),
            (BOOL, np.array([1, 0, 0], np.uint64), np.array([False, False, True])),
            (STR, [b"Ab", None, b""], None)]
    for _ in range(300):
        consts = bytearray()
        p = random_program(rng, col_types, consts)
        assert 1 <= len(p) <= 64
        depth, pieces = limits(p, {4})
        assert depth <= 16 and pieces <= 16
        try:
            model(cols, p, n, consts=bytes(consts))
        except ModelError:
            pass
        ops |= {node[0] for node in p}
        sizes.append(len(p))
    assert ops >= {COL, CONST, CMP, AND, OR, NOT, ISNULL, ISNOTNULL, IF, DIV, MOD, CONCAT, LOWER, UPPER, IFNULL, CAST}
    assert max(sizes) >= 40


def test_host_adapter_builds_and_refuses_cpu():
    import torch
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "conditional_expression_ut"], stdout=subprocess.DEVNULL)
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([os.path.join(ROOT, "host", "conditional_expression_ut")], capture_output=True, text=True, timeout=120)
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


host = F.host


def _sel_bitmap(selection, n, device):
    return E._sel_bitmap(selection, n, device)


def _device_strings(s):
    import torch
    h, st, ln, nl = s
    return (torch.from_numpy(np.ascontiguousarray(h)).cuda(), torch.from_numpy(np.ascontiguousarray(st).view(np.int64)).cuda(),
            torch.from_numpy(np.ascontiguousarray(ln).view(np.int32)).cuda(), torch.from_numpy(np.ascontiguousarray(nl)).cuda())


def run(ctx, data, numeric, strings, program, n, selection=None, device=False, consts=b""):
    """Evaluates on the GPU and checks it against the model.  numeric: Column objects (node columns 0..), strings: host
    (heap, starts, lengths, nulls) tuples (the node columns after them); with device every input, the selection and the
    outputs are on the device."""
    sel = _sel_bitmap(selection, n, device)
    cols = E._copy(numeric, device)
    scols = [_device_strings(s) for s in strings] if device else list(strings)
    try:
        t, v, nl = model(data, program, n, selection, consts)
    except ModelError as want:
        with pytest.raises(capi.YtGpuError) as e:
            ctx.evaluate_expression(cols, program, sel, string_columns=scols, string_constants=consts)
        assert e.value.code == want.code and want.message in e.value.message, (program, e.value.message)
        return None
    got = ctx.evaluate_expression(cols, program, sel, string_columns=scols, string_constants=consts)
    assert got["value_type"] == t, program
    assert got["null_count"] == int(nl.sum()), program
    if t == STR:
        heap, starts, lengths, nulls = S.flat_strings(v)
        assert bytes(host(got["heap"])) == heap, program
        assert np.array_equal(host(got["starts"]).view(np.uint64), starts)
        assert np.array_equal(host(got["lengths"]).view(np.uint32), lengths)
        assert np.array_equal(host(got["null_bytemap"]), nulls)
        if device and n:
            assert got["heap"].is_cuda
        return got
    gv = host(got["values"]).view(np.uint64)
    bits = np.unpackbits(host(got["null_bitmap"]), bitorder="little").astype(bool)
    differ = gv != v
    if t == DBL:
        with np.errstate(invalid="ignore"):
            differ &= ~(np.isnan(gv.view(np.float64)) & np.isnan(v.view(np.float64)))
    bad = np.flatnonzero(differ | (bits[:n] != nl))
    assert bad.size == 0, (program, bad[:5], gv[bad[:5]], v[bad[:5]], nl[bad[:5]])
    assert not bits[n:].any()
    return got


def _other(vtype, n, rng):
    """A second operand column: plain values with NULLs (edge values; booleans 0 / 1)."""
    from ytsaurus_b200 import Column
    bits = F.edge_values(rng, vtype, n)
    nulls = rng.random(n) < 0.15
    return Column(vtype, values=bits, null_bitmap=F._bm(nulls), value_count=n), bits, nulls


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("vtype", TYPES, ids=["i64", "u64", "f64", "bool"])
def test_gpu_every_new_op_over_every_encoding_and_window(ctx, vtype, device):
    rng = np.random.default_rng(vtype * 13 + int(device))
    n = 300
    kinds = F.BOOL_ENCODINGS if vtype == BOOL else F.ENCODINGS
    for kind in kinds:
        for start in (0, 1, 3):
            col, bits, nulls = F.make_column(kind, vtype, n, start, rng)
            other, obits, onulls = _other(vtype, n, rng)
            cond, cbits, cnulls = _other(BOOL, n, rng)
            data = [(vtype, bits, nulls), (vtype, obits, onulls), (BOOL, cbits, cnulls)]
            const = int(F.edge_values(rng, vtype, 1)[0])
            programs = []
            for cmp in CMPS:
                programs += [[(COL, 0), (COL, 1), (CMP, cmp)], [(COL, 1), (COL, 0), (CMP, cmp)], [(COL, 0), (CONST, 0, vtype, const), (CMP, cmp)]]
            programs += [[(COL, 0), (ISNULL,)], [(COL, 0), (ISNOTNULL,)]]
            programs += [[(COL, 2), (COL, 0), (COL, 1), (IF,)], [(COL, 2), (COL, 1), (COL, 0), (IF,)],
                         [(COL, 0), (COL, 1), (CMP, LT), (COL, 0), (COL, 1), (IF,)]]
            if vtype == BOOL:
                programs += [[(COL, 0), (NOT,)], [(COL, 0), (COL, 1), (AND,)], [(COL, 1), (COL, 0), (OR,)],
                             [(COL, 0), (COL, 2), (OR,)], [(COL, 0), (COL, 1), (COL, 2), (IF,)]]
            for prog in programs:
                run(ctx, data, [col, other, cond], [], prog, n, device=device)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_compare_equals_the_filter_and_its_nulls_are_the_operands(ctx, device):
    """COMPARE's TRUE rows are ytgpu_evaluate_filter's bitmap for the same comparison; its NULL rows are IS_NULL of either
    operand."""
    rng = np.random.default_rng(61 + int(device))
    n = 2000
    for vtype in TYPES + [STR]:
        if vtype == STR:
            a, b = S.random_strings(rng, n), S.random_strings(rng, n)
            for k in rng.choice(n, 200, replace=False):  # shared prefixes
                if a[k] is not None and b[k] is not None:
                    b[k] = a[k] + (b"\x00" if rng.random() < 0.5 else b"")
            cols, strings = [], [S.string_column(a, rng), S.string_column(b, rng)]
            na, nb = _strings(a), _strings(b)
            data = [(STR, a, None), (STR, b, None)]
        else:
            c0, a_bits, na = _other(vtype, n, rng)
            c1, b_bits, nb = _other(vtype, n, rng)
            cols, strings = [c0, c1], []
            data = [(vtype, a_bits, na), (vtype, b_bits, nb)]
        fcols = E._copy(cols, device)
        fstrings = [_device_strings(s) for s in strings] if device else strings
        for cmp in CMPS:
            got = run(ctx, data, cols, strings, [(COL, 0), (COL, 1), (CMP, cmp)], n, device=device)
            vals = host(got["values"]).view(np.uint64).astype(bool)
            nbits = np.unpackbits(host(got["null_bitmap"]), bitorder="little")[:n].astype(bool)
            f = ctx.evaluate_filter(fcols, fstrings, [(capi.FILTER_COMPARE_COLUMNS, cmp, 0, 1)])
            fbits = np.unpackbits(host(f["bitmap"]), bitorder="little")[:n].astype(bool)
            assert np.array_equal(vals & ~nbits, fbits), (vtype, cmp)
            assert np.array_equal(nbits, na | nb)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_string_if_and_compare_over_piece_lists(ctx, device):
    rng = np.random.default_rng(67 + int(device))
    n = 1000
    s0, s1 = S.random_strings(rng, n), S.random_strings(rng, n)
    c = S.random_strings(rng, n)
    flag, fbits, fnulls = _other(BOOL, n, rng)
    x, xbits, xnulls = _other(I64, n, rng)
    strings = [S.string_column(s0, rng), S.string_column(s1, rng), S.string_column(c, rng)]
    data = [(BOOL, fbits, fnulls), (I64, xbits, xnulls), (STR, s0, None), (STR, s1, None), (STR, c, None)]
    k = bytearray()
    slow, fast, sep, other = (S.constant(k, w) for w in (b"slow", b"fast", b"/", b"OTHER"))
    consts = bytes(k)
    cat = [(COL, 2), (CONST, 0, STR, sep), (CONCAT,), (COL, 3), (CONCAT,)]
    programs = [
        [(COL, 1), (CONST, 0, I64, 0), (CMP, GT), (CONST, 0, STR, slow), (CONST, 0, STR, fast), (IF,)],
        [(COL, 0), (COL, 2), (COL, 3), (IF,)],
        [(COL, 0)] + cat + [(COL, 4), (LOWER,), (IF,)],                             # a concat branch against a lower one
        [(COL, 0), (COL, 4), (UPPER,)] + cat + [(IF,)],                             # b's 3 pieces move over a's 1
        [(COL, 0), (COL, 2), (LOWER,), (COL, 3), (CONCAT,), (CONST, 0, STR, other), (IF,), (LOWER,)],
        [(COL, 2), (LOWER,), (COL, 3), (UPPER,), (CMP, LT)],
        cat + [(COL, 4), (CMP, GE)],
        [(COL, 2), (COL, 3), (CONCAT,), (COL, 3), (COL, 2), (CONCAT,), (CMP, EQ)],
        [(COL, 0), (COL, 2), (COL, 3), (IF,), (COL, 4), (CMP, NE)],
        [(COL, 2), (ISNULL,), (COL, 3), (ISNOTNULL,), (AND,)],
        [(COL, 2), (LOWER,), (ISNULL,)],
        [(COL, 0), (COL, 2), (COL, 3), (IF,), (COL, 1), (FARM, 2)],                # IF of leaves is one piece
        [(COL, 0), (COL, 2), (CONST, 0, STR, slow), (IF,), (COL, 3), (IFNULL,), (COL, 4), (CONCAT,)],
    ]
    for prog in programs:
        run(ctx, data, [flag, x], strings, prog, n, device=device, consts=consts)
        run(ctx, data, [flag, x], strings, prog, n, selection=rng.random(n) < 0.6, device=device, consts=consts)
    # 16 pieces at the bound through IF, 17 past it
    leaf = (COL, 2)
    p8 = [leaf] + [leaf, (CONCAT,)] * 7
    p7 = [leaf] + [leaf, (CONCAT,)] * 6
    for p16 in ([(COL, 0)] + p8 + p7 + [(CONCAT,), leaf, (IF,)],    # a: 15 pieces, b: 1
                [(COL, 0), leaf] + p8 + p7 + [(CONCAT,), (IF,)]):   # b: 15 pieces that move down over a's 1
        assert limits(p16, {2, 3, 4})[1] == 16
        run(ctx, data, [flag, x], strings, p16, n, device=device)
    p17 = [(COL, 0)] + p8 + p8 + [(CONCAT,), leaf, (IF,)]
    assert limits(p17, {2, 3, 4})[1] == 17
    with pytest.raises(capi.YtGpuError) as e:
        ctx.evaluate_expression(E._copy([flag, x], False), p17, string_columns=strings)
    assert e.value.code == capi.ERR_INVALID_ARGUMENT and "pieces" in e.value.message
    # non-ASCII refused in the taken branch only
    bad = list(s0)
    rows = [i for i in range(n) if bad[i] is not None][:5]
    for i in rows:
        bad[i] = b"Stra\xc3\x9fe"
    bstrings = [S.string_column(bad, rng)] + strings[1:]
    bdata = data[:2] + [(STR, bad, None)] + data[3:]
    taken = np.array([i in rows for i in range(n)])
    cond = [(COL, 1), (CONST, 0, I64, 0), (CMP, GE)]
    for prog in (cond + [(COL, 3), (COL, 2), (LOWER,), (IF,)], cond + [(COL, 2), (LOWER,), (COL, 3), (IF,)],
                 [(COL, 2), (UPPER,), (COL, 3), (CMP, EQ), (CONST, 0, BOOL, 0), (AND,)]):
        run(ctx, bdata, [flag, x], bstrings, prog, n, device=device)
        run(ctx, bdata, [flag, x], bstrings, prog, n, selection=~taken, device=device)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_empty_string_constants_without_string_columns(ctx, device):
    """`if(c, '', '')` and `'' = ''` name no string bytes and no string column: the binding still takes the string entry."""
    from ytsaurus_b200 import Column
    n = 100
    bits = (np.arange(n) % 3 == 0).astype(np.uint64)
    nulls = np.arange(n) % 7 == 0
    flag = Column(BOOL, values=bits, null_bitmap=F._bm(nulls), value_count=n)
    data = [(BOOL, bits, nulls)]
    empty = (CONST, 0, STR, 0)
    got = run(ctx, data, [flag], [], [(COL, 0), empty, empty, (IF,)], n, device=device)
    assert got["value_type"] == STR and got["null_count"] == int(nulls.sum())
    got = run(ctx, data, [flag], [], [empty, empty, (CMP, EQ), (COL, 0), (AND,)], n, device=device)
    assert got["value_type"] == BOOL


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_errors_follow_the_data(ctx, device):
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(71)
    n = 1000
    a = rng.integers(-100, 100, n, dtype=np.int64).view(np.uint64)
    b = rng.integers(-3, 4, n, dtype=np.int64).view(np.uint64)  # zeros among them
    a[[9, 500]] = np.uint64(INT64_MIN)
    b[[9, 500]] = np.uint64(M64)
    cols = [Column(I64, values=a, value_count=n), Column(I64, values=b, value_count=n), Column(BOOL, values=None, value_count=n)]
    data = [(I64, a, np.zeros(n, bool)), (I64, b, np.zeros(n, bool)), (BOOL, np.zeros(n, np.uint64), np.ones(n, bool))]
    eq0 = [(COL, 1), (CONST, 0, I64, 0), (CMP, EQ)]
    div = [(COL, 0), (COL, 1), (DIV,)]
    guard = [(COL, 1), (CONST, 0, I64, -1 & M64), (CMP, EQ), (CONST, 0, I64, 0)] + div + [(IF,)]
    cases = [
        (eq0 + [(CONST, 0, I64, 0)] + guard + [(IF,)], None),                            # if(b = 0, 0, if(b = -1, 0, a / b))
        (eq0 + div + [(CONST, 0, I64, 0), (IF,)], "Division by zero"),                   # if(b = 0, a / b, 0)
        ([(CONST, 0, BOOL, 0)] + div + [(CONST, 0, I64, 1), (CMP, GT), (AND,)], None),   # FALSE AND (a / b > 1)
        ([(COL, 2)] + div + [(CONST, 0, I64, 1), (CMP, GT), (AND,)], "Division by zero"),  # NULL AND (a / b > 1)
        ([(CONST, 0, BOOL, 1)] + div + [(CONST, 0, I64, 1), (CMP, GT), (OR,)], None),    # TRUE OR (a / b > 1)
        (eq0 + [(CONST, 0, I64, 0)] + div + [(IF,)], "Division INT_MIN by -1"),          # if(b = 0, 0, a / b)
        ([(COL, 2)] + div + [(CONST, 0, I64, 0), (IF,)], None),                          # a NULL condition takes no branch
        (eq0 + [(NOT,)] + div + [(CONST, 0, I64, 7), (IF,), (COL, 0), (IFNULL,)], "Division INT_MIN by -1"),
        ([(COL, 0), (COL, 1), (MOD,), (ISNULL,)], "Division by zero"),                   # IS_NULL keeps its operand's errors
    ]
    for prog, msg in cases:
        try:
            model(data, prog, n)
            got = None
        except ModelError as e:
            got = e.message
        assert got == msg, (prog, got)
        run(ctx, data, cols, [], prog, n, device=device)
    # under a selection that drops the erroring rows, every case passes
    sel = (b != 0) & (b != np.uint64(M64))
    for prog, _ in cases:
        run(ctx, data, cols, [], prog, n, selection=sel, device=device)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_random_programs_at_every_size(ctx, device):
    rng = np.random.default_rng(79 + int(device))
    specs = [("plain", I64), ("rle", U64), ("bitmap", DBL), ("bits_nulls", BOOL), ("dict", I64), ("arrow", BOOL)]
    for n in (0, 1, 31, 32, 33, 4097):
        for rep in range(8):
            cols, data = [], []
            for kind, vt in specs:
                c, bits, nl = F.make_column(kind, vt, n, int(rng.integers(1, 4)), rng)  # windows at 0: the encoding test
                cols.append(c)
                data.append((vt, bits, nl))
            svals = [S.random_strings(rng, n) for _ in range(2)]
            strings = [S.string_column(v, rng) for v in svals]
            data += [(STR, v, None) for v in svals]
            consts = bytearray()
            col_types = [d[0] for d in data]
            prog = random_program(rng, col_types, consts if rep % 2 else None)
            selection = rng.random(n) < 0.7 if rep % 3 == 2 else None
            run(ctx, data, cols, strings, prog, n, selection, device=device, consts=bytes(consts))


@pytest.mark.gpu
def test_gpu_random_programs_ten_million_rows(ctx):
    rng = np.random.default_rng(83)
    n = 10**7
    cols, data = [], []
    for kind, vt in [("plain", I64), ("rle", U64), ("bitmap", DBL), ("bits_nulls", BOOL), ("dict", I64)]:
        c, bits, nl = F.make_column(kind, vt, n, 1, rng)
        cols.append(c)
        data.append((vt, bits, nl))
    done = 0
    for device in (False, True, True):
        while True:
            prog = random_program(rng, [d[0] for d in data], result_type=[I64, BOOL, DBL][done])
            if len(prog) >= 12 and any(node[0] in (CMP, IF, AND, OR) for node in prog):
                break
        run(ctx, data, cols, [], prog, n, selection=(rng.random(n) < 0.7) if done == 2 else None, device=device)
        done += 1


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_launch_counts(ctx, device):
    rng = np.random.default_rng(89)
    n = 10000
    from ytsaurus_b200 import Column
    a, abits, an = F.make_column("rle", I64, n, 1, rng)
    b = Column(I64, values=rng.integers(0, 5, n, dtype=np.int64).view(np.uint64), value_count=n)  # zeros, never -1
    prog = [(COL, 1), (CONST, 0, I64, 0), (CMP, EQ), (CONST, 0, I64, 0), (COL, 0), (COL, 1), (DIV,), (IF,)]
    c = E._copy([a, b], device)
    before = ctx.launch_count()
    ctx.evaluate_expression(c, prog)
    assert ctx.launch_count() - before == 1
    s = [S.string_column(S.random_strings(rng, n), rng)]
    s = [_device_strings(x) for x in s] if device else s
    k = bytearray()
    lo, hi = S.constant(k, b"lo"), S.constant(k, b"hi")
    sprog = [(COL, 0), (CONST, 0, I64, 0), (CMP, GT), (COL, 1), (CONST, 0, STR, lo), (IF,), (CONST, 0, STR, hi), (CONCAT,)]
    before = ctx.launch_count()
    got = ctx.evaluate_expression(c[:1], sprog, string_columns=s, string_constants=bytes(k))
    assert got["value_type"] == STR
    # the Python binding asks for the type and size first (the size pass and the scan), then fills: 4 + 5
    assert ctx.launch_count() - before == 9


def _precomputed(vtype, values, nulls, device):
    from ytsaurus_b200 import Column
    col = Column(vtype, values=np.asarray(values, np.uint64).copy(), value_count=len(values),
                 null_bitmap=F._bm(nulls) if nulls.any() else None)
    return E._copy([col], device)[0]


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_conditional_columns_in_groupby(ctx, device):
    """sum(if(status = 200, 1, 0)), sum(if(b = 0, 0, a / b)), a BOOLEAN key and group by if(x > c, 'a', 'b') give the GROUP BY
    results of the same columns precomputed by the model."""
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(97 + int(device))
    n = 50_000
    status = rng.choice(np.array([200, 404, 500], np.uint64), n)
    snull = rng.random(n) < 0.05
    a, abits, anull = F.make_column("bitmap", I64, n, 0, rng)
    bbits = rng.choice(np.array([-2, 0, 1, 2, 3], np.int64), n).view(np.uint64)  # zeros, never -1 (a holds INT64_MIN)
    kbits = rng.integers(0, 7, n, dtype=np.uint64)
    cols = [Column(I64, values=status.copy(), null_bitmap=F._bm(snull), value_count=n), a, Column(I64, values=bbits, value_count=n),
            Column(U64, values=kbits, value_count=n)]
    data = [(I64, status, snull), (I64, abits, anull), (I64, bbits, np.zeros(n, bool)), (U64, kbits, np.zeros(n, bool))]
    dc = E._copy(cols, device)
    kc = dc[3]
    ok = [(COL, 0), (CONST, 0, I64, 200), (CMP, EQ), (CONST, 0, I64, 1), (CONST, 0, I64, 0), (IF,)]
    guarded = [(COL, 2), (CONST, 0, I64, 0), (CMP, EQ), (CONST, 0, I64, 0), (COL, 1), (COL, 2), (DIV,), (IF,)]
    boolkey = [(COL, 1), (CONST, 0, I64, 0), (CMP, GT)]
    aggs = [(capi.AGG_SUM, 0), (capi.AGG_SUM, 1), (capi.AGG_COUNT, 0), (capi.AGG_MIN, 1)]
    vals = [ctx.evaluate_expression(dc, p)["column"] for p in (ok, guarded)]
    want_vals = [_precomputed(*model(data, p, n), device) for p in (ok, guarded)]
    got = ctx.scan_filter_groupby_multi([kc], vals, aggs)
    want = ctx.scan_filter_groupby_multi([kc], want_vals, aggs)
    F._check_same_groupby(got, want)
    key = ctx.evaluate_expression(dc, boolkey)
    got = ctx.scan_filter_groupby_multi([key["column"], kc], vals, aggs)
    want = ctx.scan_filter_groupby_multi([_precomputed(*model(data, boolkey, n), device), kc], want_vals, aggs)
    F._check_same_groupby(got, want)
    assert len(host(got["count"])) == 3 * 7
    # group by if(a > 0, 'a', 'b') through the string ids, against the strings precomputed
    k = bytearray()
    ca, cb = S.constant(k, b"a"), S.constant(k, b"b")
    sprog = boolkey + [(CONST, 0, STR, ca), (CONST, 0, STR, cb), (IF,)]
    s = ctx.evaluate_expression(dc, sprog, string_constants=bytes(k))
    _, svals, _ = model(data, sprog, n, consts=bytes(k))
    pre = F.strings_to_column(svals, device)
    ids_got = ctx.string_value_ids(s["heap"], s["starts"], s["lengths"], s["null_bytemap"])
    ids_want = ctx.string_value_ids(*pre)
    skey = lambda ids: Column(U64, values=ids[0], value_count=n)  # noqa: E731
    got = ctx.scan_filter_groupby_multi([skey(ids_got)], vals, aggs, string_columns=[(s["heap"], s["starts"], s["lengths"], s["null_bytemap"])])
    want = ctx.scan_filter_groupby_multi([skey(ids_want)], want_vals, aggs, string_columns=[pre])
    assert len(host(got["count"])) >= 2 and np.array_equal(host(got["count"]), host(want["count"]))
    for x, y in zip(got["keys"] + got["values"] + got["value_null"], want["keys"] + want["values"] + want["value_null"]):
        assert np.array_equal(host(x), host(y))


@pytest.mark.gpu
def test_gpu_host_adapter_conditional_expressions():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "conditional_expression_ut"], stdout=subprocess.DEVNULL)
    r = subprocess.run([os.path.join(ROOT, "host", "conditional_expression_ut")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "conditional_expression_ut: 0 failure(s)" in r.stdout
