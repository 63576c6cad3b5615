"""Predicates inside expressions on the GPU: IN, STARTS_WITH, CONTAINS and LIKE as expression ops (csrc/expression.cu)
against a numpy model of include/ytgpu.h.

The model extends the one of test_conditional_expressions.py with the four ops.  Each takes the value on top of the stack
and gives a BOOLEAN, NULL for a NULL operand, and passes on its operand's error bits.  IN is COMPARE's EQ rule against
every entry (NaN never matches, -0.0 = +0.0); LIKE is test_filter_patterns.py's byte-regex model.  A STRING operand may be
any string result, matched as the bytes it would be written as."""
import importlib.util
import math
import os
import struct
import subprocess
import tempfile

import numpy as np
import pytest

from ytsaurus_b200 import capi
from ytsaurus_b200.capi import ExprConstants

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _load(name):
    """A sibling test module's helpers, loaded by path so no import mode matters."""
    spec = importlib.util.spec_from_file_location("_pred_" + name[:-3], os.path.join(os.path.dirname(os.path.abspath(__file__)), name))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


C = _load("test_conditional_expressions.py")  # the conditional model and its helpers
FP = _load("test_filter_patterns.py")          # the LIKE byte-regex model
E, S, F = C.E, C.S, C.F

(COL, CONST, ADD, SUB, MUL, DIV, MOD, NEG, BAND, BOR, BXOR, BNOT, CAST, IFNULL, CONCAT, LOWER, UPPER, FARM) = range(1, 19)
CMP, AND, OR, NOT, ISNULL, ISNOTNULL, IF = range(19, 26)
IN, SW, CONTAINS, LIKE = capi.EXPR_IN, capi.EXPR_STARTS_WITH, capi.EXPR_CONTAINS, capi.EXPR_LIKE
PREDS = (IN, SW, CONTAINS, LIKE)
EQ, NE, LT, GT = capi.CMP_EQ, capi.CMP_NE, capi.CMP_LT, capi.CMP_GT
I64, U64, DBL, BOOL, STR = C.I64, C.U64, C.DBL, C.BOOL, C.STR
TYPES = C.TYPES
M64, INT64_MIN = C.M64, C.INT64_MIN
ERR_DIV0, ERR_INTMIN, ERR_ASCII = C.ERR_DIV0, C.ERR_INTMIN, C.ERR_ASCII
ModelError = C.ModelError
_bits = C._bits


# ------------------------------------------------------------------------------------------------- the model
def in_entries(consts, constant, t):
    """The entries of an IN node's list: bytes for a STRING operand, else the uint64 bit patterns."""
    off, count = constant >> 32, constant & 0xFFFFFFFF
    raw = struct.unpack_from(f"<{count}Q", consts, off)
    if t == STR:
        return [bytes(consts[e >> 32:(e >> 32) + (e & 0xFFFFFFFF)]) for e in raw]
    return list(raw)


def predicate(node, t, a, nl, consts):
    """One of the four ops over an operand of type t (values a, NULL flags nl) -> 0 / 1 per row (0 where NULL)."""
    op, column, _, constant = (tuple(node) + (0,) * 4)[:4]
    if op == IN:
        ent = in_entries(consts, constant, t)
        if t == STR:
            s = set(ent)
            return np.array([not z and x in s for x, z in zip(a, nl)], np.uint64)
        ent = np.array(ent, np.uint64)
        hit = np.isin(a.view(np.float64), ent.view(np.float64)) if t == DBL else np.isin(a, ent)  # NaN never, -0.0 == +0.0
        return (hit & ~nl).astype(np.uint64)
    arg = bytes(consts[constant >> 32:(constant >> 32) + (constant & 0xFFFFFFFF)])
    if op == SW:
        f = lambda x: x.startswith(arg)  # noqa: E731
    elif op == CONTAINS:
        f = lambda x: arg in x  # noqa: E731
    else:
        rx = FP.like_regex(arg, column)
        f = lambda x: rx.fullmatch(x) is not None  # noqa: E731
    return np.array([not z and f(x) for x, z in zip(a, nl)], np.uint64)


def evaluate(cols, program, n, selection=None, consts=b""):
    """test_conditional_expressions.evaluate with the four ops: each operand is the value of the subprogram below the
    node, evaluated by the conditional model (recursively, so predicates nest), and the predicate's result stands in
    for it as a column that carries the operand's NULLs and error bits."""
    k = next((i for i, node in enumerate(program) if node[0] in PREDS), None)
    if k is None:
        return C.evaluate(cols, program, n, selection, consts)
    s = operand_start(program, k)
    t, a, nl, e = evaluate(cols, program[s:k], n, selection, consts)
    r = predicate(program[k], t, a, nl, consts)
    if not e.any():  # the result as a BOOLEAN leaf
        cols = list(cols) + [(BOOL, r, nl)]
        return evaluate(cols, program[:s] + [(COL, len(cols) - 1)] + program[k + 1:], n, selection, consts)
    return evaluate_with_errors(cols, program, s, k, (BOOL, r, nl, e), n, selection, consts)


def evaluate_with_errors(cols, program, s, k, entry, n, selection, consts):
    """The rest of the program with `entry` (type, values, NULLs, error bits) in place of program[s:k + 1].  The entry
    becomes if(c, x, x) over a column x of its values: IF keeps c's errors and the taken branch's.  c is TRUE in every
    row and carries the entry's bits: per error kind, `ISNULL(d) OR TRUE`, where d is a DIV (a LOWER for the non-ASCII
    kind) that fails where the kind is set and is NULL elsewhere, so OR keeps its bits exactly there; the kinds are joined
    with AND, which keeps both sides' bits of TRUE operands."""
    t, r, nl, e = entry
    cols = list(cols) + [(BOOL, r, nl)]
    vi = len(cols) - 1
    cond = []
    for bit, (num, den) in ((ERR_DIV0, (1, 0)), (ERR_INTMIN, (INT64_MIN, M64)), (ERR_ASCII, (0, 0))):
        rows = (e & bit) != 0
        if not rows.any():
            continue
        if bit == ERR_ASCII:
            cols.append((STR, [b"\xc3\x9f" if x else None for x in rows], None))
            d = [(COL, len(cols) - 1), (LOWER,)]
        else:
            cols.append((I64, np.where(rows, np.uint64(num), np.uint64(0)), ~rows))
            cols.append((I64, np.where(rows, np.uint64(den), np.uint64(1)), ~rows))
            d = [(COL, len(cols) - 2), (COL, len(cols) - 1), (DIV,)]
        cond += d + [(ISNULL,), (CONST, 0, BOOL, 1), (OR,)] + ([(AND,)] if cond else [])
    return evaluate(cols, program[:s] + cond + [(COL, vi), (COL, vi), (IF,)] + program[k + 1:], n, selection, consts)


def operand_start(program, k):
    """The first node of the subprogram that pushes node k's single operand (postfix)."""
    need, i = 1, k
    while need:
        i -= 1
        need += arity(program[i]) - 1
    return i


def arity(node):
    op = node[0]
    if op in (COL, CONST):
        return 0
    if op in (NEG, BNOT, CAST, LOWER, UPPER, NOT, ISNULL, ISNOTNULL) or op in PREDS:
        return 1
    if op == IF:
        return 3
    if op == FARM:
        return node[1]
    return 2


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


_one = C._one


def ev1(program, *cols, consts=b""):
    t, v, nl = model(list(cols), program, 1, consts=bytes(consts))
    return None if nl[0] else (v[0] if t == STR else int(v[0]))


# ------------------------------------------------------------------------------------------------- CPU: hand-written cases
def test_in_over_numbers():
    k = ExprConstants()
    big = k.in_list([INT64_MIN, M64, 0, 7, 7])                     # duplicates are fine
    empty = k.in_list([])
    zeros = k.in_list([-0.0, math.nan, 2.5])
    nan_only = k.in_list([math.nan])
    bools = k.in_list([1])
    c = bytes(k)

    def isin(t, x, lst):
        return ev1([(COL, 0), (IN, 0, 0, lst)], _one(t, x), consts=c)
    assert isin(I64, INT64_MIN, big) == 1 and isin(I64, M64, big) == 1 and isin(I64, 7, big) == 1 and isin(I64, 8, big) == 0
    assert isin(U64, M64, big) == 1 and isin(U64, 1 << 63, big) == 1 and isin(U64, 1, big) == 0
    assert isin(I64, 0, empty) == 0 and isin(I64, None, empty) is None and isin(I64, None, big) is None
    assert isin(DBL, _bits(0.0), zeros) == 1 and isin(DBL, _bits(-0.0), zeros) == 1 and isin(DBL, _bits(2.5), zeros) == 1
    assert isin(DBL, _bits(math.nan), zeros) == 0 and isin(DBL, _bits(math.nan), nan_only) == 0
    assert isin(DBL, _bits(2.4999999999999996), zeros) == 0
    assert isin(BOOL, 1, bools) == 1 and isin(BOOL, 0, bools) == 0
    # the packing: 8-aligned entries, strings before them
    k2 = ExprConstants()
    k2.string(b"abc")
    lst = k2.in_list([b"x", b""])
    assert (lst >> 32) % 8 == 0 and lst & 0xFFFFFFFF == 2
    assert in_entries(bytes(k2), lst, STR) == [b"x", b""]


def test_string_predicates():
    k = ExprConstants()
    lst = k.in_list([b"", b"a\x00", b"ab", b"abc"])
    pre, needle, pat = k.string(b"ab"), k.string(b"\x00b"), k.string(b"a%c")
    empty = k.string(b"")
    c = bytes(k)

    def p(op, x, const, esc=-1):
        return ev1([(COL, 0), (op, esc, 0, const)], _one(STR, x), consts=c)
    assert p(IN, b"", lst) == 1 and p(IN, b"a\x00", lst) == 1 and p(IN, b"a", lst) == 0 and p(IN, b"abcd", lst) == 0
    assert p(IN, None, lst) is None
    assert p(SW, b"abc", pre) == 1 and p(SW, b"a", pre) == 0 and p(SW, b"", empty) == 1 and p(SW, b"xab", pre) == 0
    assert p(CONTAINS, b"a\x00b", needle) == 1 and p(CONTAINS, b"ab", needle) == 0 and p(CONTAINS, b"", empty) == 1
    assert p(LIKE, b"abc", pat) == 1 and p(LIKE, b"a\x00c", pat) == 1 and p(LIKE, b"abd", pat) == 0 and p(LIKE, b"", empty) == 1
    # over piece lists: lower(concat(a, '/', b)) like 'x%', a prefix across the piece boundary
    k = ExprConstants()
    sep, px, sw = k.string(b"/"), k.string(b"ab/c%"), k.string(b"ab/c")
    cat = [(COL, 0), (CONST, 0, STR, sep), (CONCAT,), (COL, 1), (CONCAT,), (LOWER,)]
    assert ev1(cat + [(LIKE, -1, 0, px)], _one(STR, b"AB"), _one(STR, b"Cd"), consts=bytes(k)) == 1
    assert ev1(cat + [(SW, 0, 0, sw)], _one(STR, b"AB"), _one(STR, b"Cd"), consts=bytes(k)) == 1
    assert ev1(cat + [(SW, 0, 0, sw)], _one(STR, b"A"), _one(STR, b"BCd"), consts=bytes(k)) == 0


def test_errors_follow_the_data():
    k = ExprConstants()
    lst = k.in_list([1, 2])
    c = bytes(k)
    zero, two = _one(I64, 0), _one(I64, 2)
    div = [(COL, 0), (COL, 1), (DIV,)]
    guarded = [(COL, 1), (CONST, 0, I64, 0), (CMP, EQ), (CONST, 0, I64, 0)] + div + [(IF,)]
    assert ev1(guarded + [(IN, 0, 0, lst)], two, zero, consts=c) == 0                  # if(b = 0, 0, a / b) in (1, 2)
    with pytest.raises(ModelError, match="Division by zero"):
        ev1(div + [(IN, 0, 0, lst)], two, zero, consts=c)                               # (a / b) in (1, 2)
    assert ev1([(CONST, 0, BOOL, 0)] + div + [(IN, 0, 0, lst), (AND,)], two, zero, consts=c) == 0   # FALSE AND ...
    with pytest.raises(ModelError, match="0x80"):                                       # a non-ASCII LOWER operand
        ev1([(COL, 0), (LOWER,), (CONTAINS, 0, 0, k.string(b"x"))], _one(STR, b"\xc3\x9f"), consts=bytes(k))
    with pytest.raises(ModelError, match="Division by zero"):                           # nested: the errors ride on
        ev1(div + [(IN, 0, 0, lst), (NOT,), (CONST, 0, I64, 1), (CONST, 0, I64, 2), (IF,), (IN, 0, 0, lst)], two, zero, consts=c)


def test_like_over_pieces_agrees_with_the_filter_model():
    """LIKE of a concatenation of random pieces, with and without the escape, against the byte-regex model and the
    port of the matcher (segment_match) over the joined bytes."""
    rng = np.random.default_rng(113)
    palpha = FP.RANDOM_ALPHABET[:-1] + FP.PATTERN_EXTRA
    for _ in range(2000):
        parts = [FP.random_bytes(rng, FP.RANDOM_ALPHABET, 3) for _ in range(int(rng.integers(1, 4)))]
        value = b"".join(parts)
        pattern = FP.random_bytes(rng, palpha, 5)
        esc = 0x5C if rng.random() < 0.5 else -1
        try:
            want = FP.like_model(value, pattern, esc)
        except ValueError:
            continue
        assert FP.segment_match(value, pattern, esc) == want
        k = ExprConstants()
        pat = k.string(pattern)
        prog = [(COL, 0)] + [x for j in range(1, len(parts)) for x in ((COL, j), (CONCAT,))] + [(LIKE, esc, 0, pat)]
        assert ev1(prog, *[_one(STR, x) for x in parts], consts=bytes(k)) == int(want)


HEADER_PROGRAM = r"""
#include <stdio.h>
#include "include/ytgpu.h"
int main(void) {
    ytgpu_expr_node n = {YTGPU_EXPR_LIKE, -1, 0, {0}, 0};
    printf("%d %d %d %d %d\n", YTGPU_EXPR_IN, YTGPU_EXPR_STARTS_WITH, YTGPU_EXPR_CONTAINS, n.op, n.column);
    return 0;
}
"""


def test_header_compiles_as_c99_with_the_predicates():
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "e.c"), os.path.join(d, "e")
        open(src, "w").write(HEADER_PROGRAM)
        subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", ROOT, src, "-o", exe])
        out = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    assert out == [IN, SW, CONTAINS, LIKE, -1] == [26, 27, 28, 29, -1]
    assert capi.EXPR_PREDICATE_OPS == (IN, SW, CONTAINS, LIKE)


# ------------------------------------------------------------------------------------------------- random programs
NUM_LISTS = {I64: [0, 1, 7, M64, INT64_MIN, 1000], U64: [0, 3, 1 << 63, M64], DBL: [0.0, -0.0, 1.5, math.nan, math.inf],
             BOOL: [1]}
STR_LIST = [b"", b"a", b"ab\x00", b"AbC", b"abc", b"https://www.site5"]
PATTERNS = [b"%", b"a%", b"%b%", b"_b%", b"%\x00", b"https://%", b""]


def limits(prog, str_cols):
    """(stack depth, pieces bound) with the four ops consuming their operand's pieces."""
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
        elif arity(node) == 1:
            st[-1] = st[-1] if op in (LOWER, UPPER) else 0
        else:
            del st[len(st) - arity(node) + 1:]
            st[-1] = 0
        depth, top = max(depth, len(st)), max(top, sum(st))
    return depth, top


def random_program(rng, col_types, k, result_type=None, max_nodes=64, strings=True):
    """A well-typed program that mixes the conditional model's random programs with the four ops: a predicate over a
    random operand, used as a condition, a value or the result."""
    str_cols = {i for i, t in enumerate(col_types) if t == STR}
    types = TYPES + ([STR] if strings else [])

    def pred(budget):
        t = types[int(rng.integers(0, len(types)))]
        operand = C.random_program(rng, col_types, k.data if strings else None, result_type=t, max_nodes=max(1, budget))
        if t != STR or rng.random() < 0.3:
            vals = STR_LIST if t == STR else NUM_LISTS[t]
            m = int(rng.integers(0, len(vals) + 1))
            return operand + [(IN, 0, 0, k.in_list([vals[int(i)] for i in rng.choice(len(vals), m, replace=False)]))]
        op = [SW, CONTAINS, LIKE][int(rng.integers(0, 3))]
        pat = PATTERNS[int(rng.integers(0, len(PATTERNS)))]
        return operand + [(op, -1 if op == LIKE else 0, 0, k.string(pat[:-1] if op != LIKE and pat.endswith(b"%") else pat))]

    while True:
        budget = int(rng.integers(2, max_nodes // 3 + 2))
        shape = rng.random()
        if shape < 0.4:
            prog = pred(budget)
        elif shape < 0.7:
            prog = pred(budget) + [(NOT,)] + pred(budget) + [(AND if rng.random() < 0.5 else OR,)]
        else:
            t = result_type if result_type is not None else types[int(rng.integers(0, len(types)))]
            kd = k.data if strings else None
            prog = (pred(budget) + C.random_program(rng, col_types, kd, result_type=t, max_nodes=budget) +
                    C.random_program(rng, col_types, kd, result_type=t, max_nodes=budget) + [(IF,)])
        depth, pieces = limits(prog, str_cols)
        if len(prog) <= max_nodes and depth <= 16 and pieces <= 16:
            return prog


def test_random_programs_are_well_typed():
    rng = np.random.default_rng(131)
    col_types = [I64, U64, DBL, BOOL, STR]
    cols = [(I64, np.array([1, 0, 5], np.uint64), np.array([False, False, True])),
            (U64, np.array([0, 2, 3], np.uint64), np.zeros(3, bool)),
            (DBL, np.array([_bits(1.0), _bits(math.nan), 0], np.uint64), np.zeros(3, bool)),
            (BOOL, np.array([1, 0, 0], np.uint64), np.array([False, False, True])),
            (STR, [b"Ab", None, b""], None)]
    ops = set()
    for _ in range(200):
        k = ExprConstants()
        p = random_program(rng, col_types, k)
        try:
            model(cols, p, 3, consts=bytes(k))
        except ModelError:
            pass
        ops |= {node[0] for node in p}
    assert ops >= {IN, SW, CONTAINS, LIKE, IF, AND, OR, NOT, CMP}


def test_host_adapter_builds_and_refuses_cpu():
    import torch
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "expression_predicates_ut"], stdout=subprocess.DEVNULL)
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    r = subprocess.run([os.path.join(ROOT, "host", "expression_predicates_ut")], capture_output=True, text=True, timeout=120)
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
_device_strings = C._device_strings


def run(ctx, data, numeric, strings, program, n, selection=None, device=False, consts=b""):
    """C.run against this model."""
    saved = C.model
    C.model = model
    try:
        return C.run(ctx, data, numeric, strings, program, n, selection, device, bytes(consts))
    finally:
        C.model = saved


def _strs(rng, n, pool=None):
    """Random values with NULLs, \\0 bytes, shared prefixes and empty strings."""
    pool = pool or [b"", b"a", b"ab", b"ab\x00", b"abc", b"AbC", b"https://www.site5.example.com/x", b"\x00", b"b%_"]
    vals = [pool[int(i)] + (S.random_strings(rng, 1)[0] or b"" if rng.random() < 0.3 else b"") for i in rng.integers(0, len(pool), n)]
    return [None if rng.random() < 0.1 else v for v in vals]


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("vtype", TYPES, ids=["i64", "u64", "f64", "bool"])
def test_gpu_in_over_every_encoding_and_window(ctx, vtype, device):
    rng = np.random.default_rng(vtype * 17 + int(device))
    n = 300
    kinds = F.BOOL_ENCODINGS if vtype == BOOL else F.ENCODINGS
    for kind in kinds:
        for start in (0, 1, 3):
            col, bits, nulls = F.make_column(kind, vtype, n, start, rng)
            data = [(vtype, bits, nulls)]
            k = ExprConstants()
            sample = [int(x) for x in bits[rng.choice(n, 5)]] + [int(x) for x in F.edge_values(rng, vtype, 3)]
            if vtype == BOOL:
                sample = [x & 1 for x in sample]
            lists = [k.in_list(sample), k.in_list([]), k.in_list(sample[:1] * 3)]
            for lst in lists:
                for prog in ([(COL, 0), (IN, 0, 0, lst)], [(COL, 0), (IN, 0, 0, lst), (NOT,)],
                             [(COL, 0), (IN, 0, 0, lst), (COL, 0), (COL, 0), (IF,)]):
                    run(ctx, data, [col], [], prog, n, device=device, consts=bytes(k))


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_string_predicates_over_leaves_and_piece_lists(ctx, device):
    rng = np.random.default_rng(137 + int(device))
    n = 2000
    a, b = _strs(rng, n), _strs(rng, n)
    strings = [S.string_column(a, rng), S.string_column(b, rng)]
    x, xbits, xnulls = C._other(I64, n, rng)
    data = [(I64, xbits, xnulls), (STR, a, None), (STR, b, None)]
    k = ExprConstants()
    sep = k.string(b"/")
    lst = k.in_list([b"", b"ab", b"ab\x00", b"abc/ab", b"a/abc"] + [v for v in a[:20] if v is not None])
    args = {SW: [k.string(w) for w in (b"", b"ab", b"ab\x00", b"abc/a", b"https://www.site")],
            CONTAINS: [k.string(w) for w in (b"", b"\x00", b"c/a", b"site5", b"b%_")],
            LIKE: [k.string(w) for w in (b"", b"%", b"ab%", b"%c/a%", b"_b%", b"%\\%%", b"https://www.site_.example.com/%x%")]}
    operands = [[(COL, 1)], [(COL, 1), (LOWER,)], [(COL, 1), (CONST, 0, STR, sep), (CONCAT,), (COL, 2), (CONCAT,)],
                [(COL, 1), (CONST, 0, STR, sep), (CONCAT,), (COL, 2), (CONCAT,), (UPPER,)],
                [(COL, 0), (CONST, 0, I64, 0), (CMP, GT), (COL, 1), (COL, 2), (IF,)], [(CONST, 0, STR, sep)]]
    for operand in operands:
        progs = [operand + [(IN, 0, 0, lst)]]
        for op, consts in args.items():
            for cst in consts:
                progs.append(operand + [(op, 0x5C if op == LIKE else 0, 0, cst)])
        for prog in progs:
            run(ctx, data, [x], strings, prog, n, device=device, consts=bytes(k))
        run(ctx, data, [x], strings, progs[-1], n, selection=rng.random(n) < 0.5, device=device, consts=bytes(k))
        # a STRING result of a predicate: if(is_substr('/api/', url), 'api', 'web')
        run(ctx, data, [x], strings, progs[3] + [(CONST, 0, STR, sep), (COL, 2), (IF,)], n, device=device, consts=bytes(k))


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_agrees_with_the_filter(ctx, device):
    """TRUE rows of `x OP` are ytgpu_evaluate_filter's bitmap for the same leaf; TRUE rows of `NOT (x OP)` its NOT bitmap."""
    rng = np.random.default_rng(139 + int(device))
    n = 3000
    s = _strs(rng, n)
    strings = [S.string_column(s, rng)]
    num, nbits, nnull = C._other(I64, n, rng)
    fcols = E._copy([num], device)
    fstrings = [_device_strings(x) for x in strings] if device else strings
    k = ExprConstants()
    words = [b"", b"ab", b"ab\x00", b"https://www.site5.example.com/x"]
    cases = []  # (expression program, filter program, list_values)
    ilist = [int(v) for v in nbits[:40]] + [0, M64]
    cases.append(([(COL, 0), (IN, 0, 0, k.in_list(ilist))], [(capi.FILTER_IN, 0, 0, 0, 0, len(ilist))], ilist))
    slist_c = [k.string(w) for w in words]
    slist = k.in_list(words)
    cases.append(([(COL, 1), (IN, 0, 0, slist)], [(capi.FILTER_IN, 0, 1, 0, 0, len(words))], slist_c))
    for w in (b"ab", b"https://"):
        c = k.string(w)
        cases.append(([(COL, 1), (SW, 0, 0, c)], [(capi.FILTER_STARTS_WITH, 0, 1, 0, c >> 32, len(w))], []))
        cases.append(([(COL, 1), (CONTAINS, 0, 0, c)], [(capi.FILTER_CONTAINS, 0, 1, 0, c >> 32, len(w))], []))
    for w in (b"ab%", b"%site_%", b"%\x00"):
        c = k.string(w)
        cases.append(([(COL, 1), (LIKE, -1, 0, c)], [(capi.FILTER_LIKE, 0, 1, -1, c >> 32, len(w))], []))
    consts = bytes(k)
    data = [(I64, nbits, nnull), (STR, s, None)]
    for expr, filt, lv in cases:
        for negate in (False, True):
            prog = expr + ([(NOT,)] if negate else [])
            got = run(ctx, data, [num], strings, prog, n, device=device, consts=consts)
            vals = host(got["values"]).view(np.uint64).astype(bool)
            nb = np.unpackbits(host(got["null_bitmap"]), bitorder="little")[:n].astype(bool)
            f = ctx.evaluate_filter(fcols, fstrings, filt + ([(capi.FILTER_NOT,)] if negate else []), list_values=lv,
                                    string_constants=consts)
            fb = np.unpackbits(host(f["bitmap"]), bitorder="little")[:n].astype(bool)
            assert np.array_equal(vals & ~nb, fb), (expr, negate)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_agrees_with_materialisation(ctx, device):
    """OP over lower(concat(a, '/', b)) equals OP over that STRING result written out by the existing call; 16-piece
    operands and 1 MiB values included."""
    rng = np.random.default_rng(149 + int(device))
    n = 1500
    a = _strs(rng, n, [b"AB", b"Ab/", b"x", b"", b"HTTPS://WWW.SITE4.EXAMPLE.COM"])
    b = _strs(rng, n, [b"C", b"/api/", b"", b"site4"])
    big = [None] * n
    for i in (3, 700):
        big[i] = (b"Q" * (1 << 20 - 1)) + b"/API/" + b"q" * ((1 << 20) - 1 - (1 << 19) - 5)
    strings = [S.string_column(a, rng), S.string_column(b, rng), S.string_column(big, rng)]
    data = [(STR, a, None), (STR, b, None), (STR, big, None)]
    k = ExprConstants()
    sep = k.string(b"/")
    cat = [(COL, 0), (CONST, 0, STR, sep), (CONCAT,), (COL, 1), (CONCAT,), (LOWER,)]
    cat16 = [(COL, 0)] + [(COL, 1), (CONCAT,), (CONST, 0, STR, sep), (CONCAT,)] * 7 + [(COL, 0), (CONCAT,)]
    assert limits(cat16, {0, 1, 2})[1] == 16
    wide = [(COL, 2), (COL, 1), (IFNULL,), (COL, 0), (CONCAT,), (LOWER,)]
    ops = [(IN, 0, 0, k.in_list([b"ab/c", b"x/", b"/", b"ab//api/"])), (SW, 0, 0, k.string(b"ab/")),
           (SW, 0, 0, k.string(b"ab//a")), (CONTAINS, 0, 0, k.string(b"b/c")), (CONTAINS, 0, 0, k.string(b"/api/")),
           (LIKE, -1, 0, k.string(b"%/_p%")), (LIKE, -1, 0, k.string(b"https://www.site_.example.com/%"))]
    consts = bytes(k)
    for operand in (cat, cat16, wide):
        written = ctx.evaluate_expression([], operand, string_columns=strings, string_constants=consts)
        wcol = (host(written["heap"]), host(written["starts"]).view(np.uint64), host(written["lengths"]).view(np.uint32),
                host(written["null_bytemap"]))
        for op in ops:
            got = run(ctx, data, [], strings, operand + [op], n, device=device, consts=consts)
            want = ctx.evaluate_expression([], [(COL, 0), op], string_columns=[wcol], string_constants=consts)
            assert np.array_equal(host(got["values"]), host(want["values"])), (operand, op)
            assert np.array_equal(host(got["null_bitmap"]), host(want["null_bitmap"]))


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_long_lists_cross_the_staged_head(ctx, device):
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(151 + int(device))
    n = 20000
    v = rng.integers(0, 200_000, n, dtype=np.int64).view(np.uint64)
    col = Column(I64, values=v, value_count=n)
    sv = [b"k%06d" % int(x) for x in rng.integers(0, 100_000, n)]
    strings = [S.string_column(sv, rng)]
    data = [(I64, v, np.zeros(n, bool)), (STR, sv, None)]
    for m in (1024, 1025, 65536):
        k = ExprConstants()
        ent = rng.choice(200_000, m, replace=False)
        lst = k.in_list([int(x) for x in ent])
        run(ctx, data, [col], strings, [(COL, 0), (IN, 0, 0, lst)], n, device=device, consts=bytes(k))
        if m < 65536:  # the 65536 entries of a call are the numeric list's
            k = ExprConstants()
            lst = k.in_list([b"k%06d" % int(x) for x in ent[:m] % 100_000])
            run(ctx, data, [col], strings, [(COL, 1), (IN, 0, 0, lst)], n, device=device, consts=bytes(k))


def _code(fn):
    with pytest.raises(capi.YtGpuError) as e:
        fn()
    return e.value.code, e.value.message


@pytest.mark.gpu
def test_gpu_limits_and_errors(ctx):
    from ytsaurus_b200 import Column
    n = 64
    v = np.arange(n, dtype=np.uint64)
    col = [Column(I64, values=v, value_count=n)]
    s = [S.string_column([b"abc"] * n, np.random.default_rng(1))]

    def ev(prog, consts, strings=s):
        return ctx.evaluate_expression(col, prog, string_columns=strings, string_constants=bytes(consts))
    # IN entries: 65536 over a call, 65537 past it
    k = ExprConstants()
    a, b = k.in_list(range(65535)), k.in_list([1])
    ev([(COL, 0), (IN, 0, 0, a), (COL, 0), (IN, 0, 0, b), (AND,)], k)
    k2 = ExprConstants()
    a, b = k2.in_list(range(65536)), k2.in_list([1])
    code, msg = _code(lambda: ev([(COL, 0), (IN, 0, 0, a), (COL, 0), (IN, 0, 0, b), (AND,)], k2))
    assert code == capi.ERR_INVALID_ARGUMENT and "IN entries" in msg
    # 256 positions per pattern, 257 past it
    k = ExprConstants()
    p256, p257 = k.string(b"a" * 256), k.string(b"a" * 257)
    ev([(COL, 1), (LIKE, -1, 0, p256)], k)
    ev([(COL, 1), (CONTAINS, 0, 0, p256)], k)
    for op in (LIKE, CONTAINS):
        code, msg = _code(lambda: ev([(COL, 1), (op, -1, 0, p257)], k))
        assert code == capi.ERR_INVALID_ARGUMENT and "POSITIONS" in msg
    # 32 KiB of compiled patterns at the bound and past it, within 64 nodes: a 256-byte needle over c distinct bytes below
    # 0x80 compiles to 272 + 8 + 8 * 4 * (c + 3) bytes; 7 of c = 120 and one of c = 90 make 32768, c = 91 makes 32800
    def needle(c):
        return (bytes(range(1, c + 1)) * 3)[:256]

    def patterns_program(last):
        kk = ExprConstants()
        prog = []
        for j, c in enumerate([120] * 7 + [last]):
            prog += [(COL, 1), (CONTAINS, 0, 0, kk.string(needle(c)))] + ([(OR,)] if j else [])
        return prog, kk
    assert sum(FP.compiled_size(needle(c), like=False) for c in [120] * 7 + [90]) == 32768
    prog, kk = patterns_program(90)
    assert len(prog) <= 64
    ev(prog, kk)
    prog, kk = patterns_program(91)
    code, msg = _code(lambda: ev(prog, kk))
    assert code == capi.ERR_INVALID_ARGUMENT and "compile to more than 32768" in msg
    # malformed lists and patterns
    k = ExprConstants()
    k.string(b"abc")
    good = k.in_list([1, 2])
    bad_cases = [
        ([(COL, 0), (IN, 0, 0, good + (1 << 32))], "IN list"),                        # misaligned
        ([(COL, 0), (IN, 0, 0, good + 1)], "IN list"),                                # one entry past the constants
        ([(COL, 1), (LIKE, -1, 0, (20 << 32) | 10)], "pattern outside"),
        ([(COL, 1), (SW, 0, 0, (0 << 32) | 99)], "prefix outside"),
        ([(COL, 1), (LIKE, 300, 0, 0 << 32 | 1)], "escape"),
        ([(COL, 0), (SW, 0, 0, 0 << 32 | 1)], "takes a STRING"),
        ([(COL, 0), (CONTAINS, 0, 0, 0 << 32 | 1)], "takes a STRING"),
    ]
    for prog, want in bad_cases:
        code, msg = _code(lambda: ev(prog, k))
        assert code == capi.ERR_INVALID_ARGUMENT and want in msg, (prog, msg)
    k = ExprConstants()
    lst = k.in_list([(50 << 32) | 1])
    code, msg = _code(lambda: ev([(COL, 1), (IN, 0, 0, lst)], k))
    assert code == capi.ERR_INVALID_ARGUMENT and "entry 0 outside" in msg
    k = ExprConstants()
    lone = k.string(b"ab\\")
    code, msg = _code(lambda: ev([(COL, 1), (LIKE, 0x5C, 0, lone)], k))
    assert code == capi.ERR_INVALID_ARGUMENT and "lone escape" in msg
    k = ExprConstants()
    bl = k.in_list([2])
    bcol = [Column(BOOL, values=v & np.uint64(1), value_count=n)]
    code, msg = _code(lambda: ctx.evaluate_expression(bcol, [(COL, 0), (IN, 0, 0, bl)], string_constants=bytes(k)))
    assert code == capi.ERR_INVALID_ARGUMENT and "BOOLEAN" in msg
    # ytgpu_evaluate_expression refuses the new ops
    import ctypes as Ct
    nodes = (capi.ExprNode * 2)()
    nodes[0].op, nodes[0].column = COL, 0
    nodes[1].op = IN
    views = (capi.ColumnView * 1)(col[0].view())
    out = np.zeros(n, np.uint64)
    nb = np.zeros(8 * ((n + 63) // 64), np.uint8)
    err = capi.Error()
    rc = ctx.lib.ytgpu_evaluate_expression(ctx.handle, Ct.cast(views, Ct.c_void_p), 1, Ct.cast(nodes, Ct.c_void_p), 2, None,
                                           out.ctypes.data, nb.ctypes.data, None, None, capi.MEM_HOST, Ct.byref(err))
    assert rc == capi.ERR_INVALID_ARGUMENT and b"unknown op" in err.message


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_launch_counts_and_selection(ctx, device):
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(157)
    n = 10000
    v = rng.integers(0, 10, n, dtype=np.int64).view(np.uint64)
    c = E._copy([Column(I64, values=v, value_count=n)], device)
    k = ExprConstants()
    lst = k.in_list([1, 2, 3])
    prog = [(COL, 0), (IN, 0, 0, lst), (COL, 0), (CONST, 0, I64, 0), (IF,)]   # if(k in (1, 2, 3), k, 0)
    before = ctx.launch_count()
    ctx.evaluate_expression(c, prog, string_constants=bytes(k))
    assert ctx.launch_count() - before == 1      # the type query launches nothing
    s = S.random_strings(rng, n)
    st = [S.string_column(s, rng)]
    st = [_device_strings(x) for x in st] if device else st
    api, web = k.string(b"api"), k.string(b"web")
    needle = k.string(b"a")
    sprog = [(COL, 1), (CONTAINS, 0, 0, needle), (CONST, 0, STR, api), (CONST, 0, STR, web), (IF,)]
    before = ctx.launch_count()
    got = ctx.evaluate_expression(c, sprog, string_columns=st, string_constants=bytes(k))
    assert got["value_type"] == STR and ctx.launch_count() - before == 9   # size pass + scan, then 5
    # selection: unselected rows are NULL and raise nothing
    zero = np.zeros(n, np.uint64)
    data = [(I64, v, np.zeros(n, bool)), (I64, zero, np.zeros(n, bool))]
    hz = [Column(I64, values=v, value_count=n), Column(I64, values=zero, value_count=n)]
    cz = E._copy(hz, device)
    div = [(COL, 0), (COL, 1), (DIV,), (IN, 0, 0, lst)]
    run(ctx, data, hz, [], div, n, selection=np.zeros(n, bool), device=device, consts=bytes(k))
    with pytest.raises(capi.YtGpuError):
        ctx.evaluate_expression(cz, div, string_constants=bytes(k))


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_random_programs_at_every_size(ctx, device):
    rng = np.random.default_rng(163 + int(device))
    specs = [("plain", I64), ("rle", U64), ("bitmap", DBL), ("bits_nulls", BOOL), ("dict", I64)]
    for n in (0, 1, 31, 32, 33, 4097):
        for rep in range(8):
            cols, data = [], []
            for kind, vt in specs:
                c, bits, nl = F.make_column(kind, vt, n, int(rng.integers(1, 4)), rng)  # windows at 0: the encoding test
                cols.append(c)
                data.append((vt, bits, nl))
            svals = [_strs(rng, n) for _ in range(2)]
            strings = [S.string_column(v, rng) for v in svals]
            data += [(STR, v, None) for v in svals]
            k = ExprConstants()
            prog = random_program(rng, [d[0] for d in data], k)
            selection = rng.random(n) < 0.7 if rep % 3 == 2 else None
            run(ctx, data, cols, strings, prog, n, selection, device=device, consts=bytes(k))


@pytest.mark.gpu
def test_gpu_random_programs_ten_million_rows(ctx):
    rng = np.random.default_rng(167)
    n = 10**7
    cols, data = [], []
    for kind, vt in [("plain", I64), ("rle", U64), ("bitmap", DBL), ("dict", I64)]:
        c, bits, nl = F.make_column(kind, vt, n, 1, rng)
        cols.append(c)
        data.append((vt, bits, nl))
    for device, rt in ((False, I64), (True, BOOL)):
        k = ExprConstants()
        while True:
            prog = random_program(rng, [d[0] for d in data], k, result_type=rt, strings=False)
            if len(prog) >= 8:
                break
            k = ExprConstants()
        run(ctx, data, cols, [], prog, n, device=device, consts=bytes(k))


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_predicates_in_groupby(ctx, device):
    """sum(if(k in (...), v, 0)) and group by if(url like ..., 'a', 'b') give the GROUP BY results of the same columns
    precomputed by the model."""
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(173 + int(device))
    n = 50_000
    kk = rng.integers(0, 40, n, dtype=np.int64).view(np.uint64)
    vv = rng.integers(-1000, 1000, n, dtype=np.int64).view(np.uint64)
    g = rng.integers(0, 5, n, dtype=np.uint64)
    url = _strs(rng, n, [b"https://a/", b"http://b/api/", b"https://www.site5.example.com/q"])
    cols = [Column(I64, values=kk, value_count=n), Column(I64, values=vv, value_count=n), Column(U64, values=g, value_count=n)]
    data = [(I64, kk, np.zeros(n, bool)), (I64, vv, np.zeros(n, bool)), (U64, g, np.zeros(n, bool)), (STR, url, None)]
    strings = [S.string_column(url, rng)]
    dc = E._copy(cols, device)
    ds = [_device_strings(x) for x in strings] if device else strings
    k = ExprConstants()
    lst = k.in_list(range(0, 40, 3))
    cond = [(COL, 0), (IN, 0, 0, lst), (COL, 1), (CONST, 0, I64, 0), (IF,)]
    aggs = [(capi.AGG_SUM, 0), (capi.AGG_COUNT, 0)]
    got_v = ctx.evaluate_expression(dc, cond, string_constants=bytes(k))["column"]
    want_v = C._precomputed(*model(data, cond, n, consts=bytes(k)), device)
    F._check_same_groupby(ctx.scan_filter_groupby_multi([dc[2]], [got_v], aggs), ctx.scan_filter_groupby_multi([dc[2]], [want_v], aggs))
    ca, cb = k.string(b"a"), k.string(b"b")
    key = [(COL, 3), (LIKE, -1, 0, k.string(b"https://%")), (CONST, 0, STR, ca), (CONST, 0, STR, cb), (IF,)]
    s = ctx.evaluate_expression(dc, key, string_columns=ds, string_constants=bytes(k))
    _, svals, _ = model(data, key, n, consts=bytes(k))
    pre = F.strings_to_column(svals, device)
    ids_got = ctx.string_value_ids(s["heap"], s["starts"], s["lengths"], s["null_bytemap"])
    ids_want = ctx.string_value_ids(*pre)
    assert np.array_equal(host(ids_got[0]), host(ids_want[0]))
    skey = lambda ids: Column(U64, values=ids[0], value_count=n)  # noqa: E731
    got = ctx.scan_filter_groupby_multi([skey(ids_got)], [got_v], aggs)
    want = ctx.scan_filter_groupby_multi([skey(ids_want)], [want_v], aggs)
    assert np.array_equal(host(got["count"]), host(want["count"])) and len(host(got["count"])) >= 2


@pytest.mark.gpu
def test_gpu_host_adapter_predicates():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "expression_predicates_ut"], stdout=subprocess.DEVNULL)
    r = subprocess.run([os.path.join(ROOT, "host", "expression_predicates_ut")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "expression_predicates_ut: 0 failure(s)" in r.stdout
