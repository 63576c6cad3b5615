"""CONTAINS and LIKE leaves of the WHERE evaluator (ytgpu_evaluate_filter, csrc/filter.cu, strings.cuh).

The model restates include/ytgpu.h: LIKE is a full match of the byte regular expression in which % is [\\x00-\\xff]*, _ is
[^\\x80-\\xbf][\\x80-\\xbf]* and every other byte (an escaped one included) is itself; CONTAINS is "the needle is a
contiguous byte sequence of the value"; both are NULL for a NULL value.  On the CPU the model is pinned by hand-written
cases, compared with a code-point reference on valid UTF-8, and compared with a Python port of the kernel's algorithm (split
at %, Shift-And per segment, the earliest end of every middle segment).  On the GPU every output is compared with the model
bit for bit."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

import oracle
from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import EValueType as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CMPOP, SW, ISNULL, AND, OR, NOT = (capi.FILTER_COMPARE, capi.FILTER_STARTS_WITH, capi.FILTER_IS_NULL, capi.FILTER_AND,
                                   capi.FILTER_OR, capi.FILTER_NOT)
CONTAINS, LIKE = capi.FILTER_CONTAINS, capi.FILTER_LIKE
TRUE, FALSE, NULL = 1, 0, 2
STAR, ANY = -1, -2


# ------------------------------------------------------------------------------------------------- the model
def pattern_tokens(pattern: bytes, escape: int = -1):
    """-> literal bytes, STAR and ANY; ValueError for a trailing lone escape."""
    out, k = [], 0
    while k < len(pattern):
        b = pattern[k]
        if b == escape:
            k += 1
            if k == len(pattern):
                raise ValueError("lone escape")
            out.append(pattern[k])
        else:
            out.append(STAR if b == 0x25 else (ANY if b == 0x5F else b))
        k += 1
    return out


def like_regex(pattern: bytes, escape: int = -1):
    parts = [rb"[\x00-\xff]*" if t == STAR else (rb"[^\x80-\xbf][\x80-\xbf]*" if t == ANY else re.escape(bytes([t])))
             for t in pattern_tokens(pattern, escape)]
    return re.compile(b"".join(parts), re.DOTALL)


def like_model(value: bytes, pattern: bytes, escape: int = -1) -> bool:
    return like_regex(pattern, escape).fullmatch(value) is not None


def codepoint_like(value: bytes, pattern: bytes, escape: int = -1) -> bool:
    """The code-point rule: decode both, _ is one code point, % any code-point sequence (escape: an ASCII byte)."""
    s, p = value.decode(), pattern.decode()
    esc = chr(escape) if escape >= 0 else None
    parts, k = [], 0
    while k < len(p):
        ch = p[k]
        if ch == esc:
            k += 1
            parts.append(re.escape(p[k]))
        else:
            parts.append(".*" if ch == "%" else ("." if ch == "_" else re.escape(ch)))
        k += 1
    return re.fullmatch("".join(parts), s, re.DOTALL) is not None


def is_cont(b):
    return 0x80 <= b <= 0xBF


def segment_match(value: bytes, pattern: bytes, escape: int = -1, like: bool = True) -> bool:
    """Port of strings.cuh's pattern_match: segments split at %, Shift-And, earliest end of every non-final segment."""
    tok = pattern_tokens(pattern, escape) if like else [STAR] + list(pattern) + [STAR]
    segs, cur = [], []
    for t in tok + [STAR]:
        if t == STAR:
            if cur:
                segs.append(cur)
            cur = []
        else:
            cur.append(t)
    anchor_start = not tok or tok[0] != STAR
    anchor_end = not tok or tok[-1] != STAR
    if not segs:
        return not anchor_start or len(value) == 0
    pos = 0
    for g, seg in enumerate(segs):
        L = len(seg)
        any1 = sum(1 << i for i, t in enumerate(seg) if t == ANY)
        anchored = g == 0 and anchor_start
        to_end = g == len(segs) - 1 and anchor_end
        D, j, accept = 0, pos, False
        while j < len(value):
            b = value[j]
            enter = sum(1 << i for i, t in enumerate(seg) if t == b or (t == ANY and not is_cont(b)))
            sh = (D << 1) | (1 if (not anchored or j == pos) else 0)
            D = ((sh & enter) | (D & any1 if is_cont(b) else 0)) & ((1 << L) - 1)
            j += 1
            accept = bool((D >> (L - 1)) & 1)
            if accept and not to_end:
                break
            if anchored and D == 0:
                return False
        if not accept:
            return False
        if to_end:
            return j == len(value)
        pos = j
    return True


def compiled_size(pattern: bytes, escape: int = -1, like: bool = True) -> int:
    """The size ytgpu.h states: 272 + 8 * segments + 8 * words * (classes + 1)."""
    tok = pattern_tokens(pattern, escape) if like else list(pattern)
    positions = [t for t in tok if t != STAR]
    segs = len([s for s in re.split(b"\x00", bytes(0 if t == STAR else 1 for t in tok)) if s])
    words = max(1, (len(positions) + 63) // 64)
    lits = {t for t in positions if t >= 0}
    classes = len(lits) + any(not is_cont(b) and b not in lits for b in range(256)) + any(is_cont(b) and b not in lits
                                                                                          for b in range(256))
    return 272 + 8 * segs + 8 * words * (classes + 1)


def escape_literal(x: bytes, esc: int = 0x5C) -> bytes:
    out = bytearray()
    for b in x:
        if b in (0x25, 0x5F, esc):
            out.append(esc)
        out.append(b)
    return bytes(out)


# ------------------------------------------------------------------------------------------------- CPU checks
E = "é".encode()           # 2 bytes
NIHON = "日本".encode()    # 2 x 3 bytes
FOUR = "😀".encode()       # 4 bytes

HAND_CASES = [  # (value, pattern, escape, expected)
    (b"abc", b"abc", -1, True), (b"abc", b"ab", -1, False), (b"abc", b"a%", -1, True), (b"abc", b"%c", -1, True),
    (b"abc", b"%b%", -1, True), (b"abc", b"a_c", -1, True), (b"abc", b"a__c", -1, False), (b"ABC", b"abc", -1, False),
    (E, b"_", -1, True), (E, b"__", -1, False), (E, E, -1, True), (b"caf" + E, b"caf_", -1, True),
    (NIHON, b"__", -1, True), (NIHON, b"_", -1, False), (NIHON, b"___", -1, False), (NIHON, "日_".encode(), -1, True),
    (FOUR, b"_", -1, True), (b"a", b"_", -1, True), (b"x" + FOUR + b"y", b"x_y", -1, True),
    (b"x" + FOUR + b"y", b"x__y", -1, False),
    # stray continuation bytes: a _ eats the ones that follow a lead byte; a value may start with one
    (b"a\x80\x80", b"_", -1, True), (b"\x80", b"_", -1, False), (b"\x80", b"%", -1, True), (b"\x80a", b"_a", -1, False),
    (b"\x80a", b"%a", -1, True), (b"\x80a", b"\x80_", -1, True), (b"a\xbf", b"a_", -1, False),
    # newlines are ordinary bytes
    (b"a\nb", b"a_b", -1, True), (b"a\nb", b"a%b", -1, True), (b"\n", b"%", -1, True),
    # empty value, empty pattern
    (b"", b"", -1, True), (b"a", b"", -1, False), (b"", b"%", -1, True), (b"", b"_", -1, False), (b"", b"%%", -1, True),
    (b"abc", b"%%", -1, True), (b"a", b"_%_", -1, False), (b"ab", b"_%_", -1, True), (E + E, b"_%_", -1, True),
    # escapes: %, _ and the escape byte itself
    (b"100%", b"100\\%", 0x5C, True), (b"1000", b"100\\%", 0x5C, False), (b"a_b", b"a\\_b", 0x5C, True),
    (b"axb", b"a\\_b", 0x5C, False), (b"a\\b", b"a\\\\b", 0x5C, True), (b"a%b", b"a!%b", 0x21, True),
    (b"a!b", b"a!!b", 0x21, True), (b"ab", b"a\\b", 0x5C, True),  # an escaped ordinary byte is itself
    # all wildcards
    (b"abc", b"%_%", -1, True), (b"", b"%_%", -1, False), (b"ab", b"___", -1, False), (b"abc", b"___", -1, True),
    (b"abc", b"%___%", -1, True), (b"abc", b"____%", -1, False),
]


@pytest.mark.parametrize("value,pattern,escape,want", HAND_CASES)
def test_model_hand_cases(value, pattern, escape, want):
    assert like_model(value, pattern, escape) == want
    assert segment_match(value, pattern, escape) == want


def test_model_refuses_a_lone_trailing_escape():
    with pytest.raises(ValueError):
        pattern_tokens(b"ab\\", 0x5C)
    assert pattern_tokens(b"ab\\\\", 0x5C) == [0x61, 0x62, 0x5C]


RANDOM_ALPHABET = [b"a", b"b", b"\n", b"\x80", b"\xbf", b"\xc3", E, NIHON[:3], FOUR, b"\\"]
PATTERN_EXTRA = [b"%", b"_", b"\\%", b"\\_", b"\\\\"]


def random_bytes(rng, alphabet, max_tokens):
    return b"".join(alphabet[int(i)] for i in rng.integers(0, len(alphabet), int(rng.integers(0, max_tokens + 1))))


def test_kernel_algorithm_equals_the_byte_regex_model():
    """The earliest-end segment algorithm against the model on 10^5 random values and patterns with stray continuation
    bytes; LIKE with and without the escape, and CONTAINS against `in`."""
    rng = np.random.default_rng(101)
    palpha = RANDOM_ALPHABET[:-1] + PATTERN_EXTRA
    for _ in range(100_000):
        v = random_bytes(rng, RANDOM_ALPHABET, 8)
        p = random_bytes(rng, palpha, 6)
        esc = 0x5C if rng.random() < 0.5 else -1
        if esc < 0 and b"\\" in p:
            p = p.replace(b"\\", b"")
        assert segment_match(v, p, esc) == like_model(v, p, esc), (v, p, esc)
    for _ in range(20_000):
        v = random_bytes(rng, RANDOM_ALPHABET, 8)
        x = random_bytes(rng, RANDOM_ALPHABET, 3)
        assert segment_match(v, x, like=False) == (x in v)
        assert like_model(v, b"%" + escape_literal(x) + b"%", 0x5C) == (x in v)


def test_model_equals_the_codepoint_rule_on_valid_utf8():
    hyp = pytest.importorskip("hypothesis")
    st = hyp.strategies
    chars = st.sampled_from(["a", "b", "\n", "é", "ß", "日", "本", "😀", "%", "_", "!"])

    @hyp.settings(max_examples=2000, deadline=None, derandomize=True)
    @hyp.given(st.lists(chars.filter(lambda c: c not in "%_!"), max_size=8), st.lists(chars, max_size=6), st.booleans())
    def prop(value, pattern, use_escape):
        v = "".join(value).encode()
        p = "".join(pattern)
        esc = 0x21 if use_escape else -1
        if use_escape and p.endswith("!") and (len(p) - len(p.rstrip("!"))) % 2:
            p = p[:-1]
        p = p.encode()
        assert like_model(v, p, esc) == codepoint_like(v, p, esc)
        assert segment_match(v, p, esc) == codepoint_like(v, p, esc)
    prop()


def test_compiled_size_formula_examples():
    assert compiled_size(b"a") == 272 + 8 + 8 * 1 * 4            # one literal: classes {a, other, other continuation}
    assert compiled_size(b"%") == 272 + 8 * 1 * 3                 # no position: one word, two classes
    assert compiled_size(b"a" * 65) == 272 + 8 + 8 * 2 * 4
    assert compiled_size(b"a%b%c") == 272 + 24 + 8 * 5 * 1 + 8
    assert compiled_size(b"abc", like=False) == compiled_size(b"%abc%")


HEADER_PROGRAM = r"""
#include <stdio.h>
#include "include/ytgpu.h"
int main(void) {
    printf("%d %d %d %d\n", YTGPU_FILTER_CONTAINS, YTGPU_FILTER_LIKE, YTGPU_FILTER_MAX_PATTERN_POSITIONS,
           YTGPU_FILTER_MAX_PATTERN_BYTES);
    return 0;
}
"""


def test_header_compiles_as_c99_and_the_constants_match_the_binding():
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "f.c"), os.path.join(d, "f")
        open(src, "w").write(HEADER_PROGRAM)
        subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", ROOT, src, "-o", exe])
        out = [int(x) for x in subprocess.check_output([exe], text=True).split()]
    assert out == [capi.FILTER_CONTAINS, capi.FILTER_LIKE, capi.FILTER_MAX_PATTERN_POSITIONS, capi.FILTER_MAX_PATTERN_BYTES]
    assert out == [10, 11, 256, 32768]
    lib = capi.load()
    assert "ytgpu_evaluate_filter" in capi.EXPORTED_SYMBOLS and hasattr(lib, "ytgpu_evaluate_filter")


def test_host_adapters_build_and_refuse_cpu():
    import torch
    for target in ("filter_ut", "like_ut"):
        subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), target], stdout=subprocess.DEVNULL)
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    for target in ("filter_ut", "like_ut"):
        r = subprocess.run([os.path.join(ROOT, "host", target)], capture_output=True, text=True, timeout=120)
        assert r.returncode == 100 and "no CPU fallback" in r.stderr


# ------------------------------------------------------------------------------------------------- GPU helpers
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
        return tuple(_dev(x) for x in (h, s, ln, nl))
    return h, s, ln, nl


def _dev(x):
    import torch
    x = np.ascontiguousarray(x)
    return torch.from_numpy(x.view({1: np.uint8, 4: np.int32, 8: np.int64}[x.dtype.itemsize])).cuda()


def host(x):
    import torch
    if x is None:
        return None
    if torch.is_tensor(x):
        x = x.cpu().numpy()
    return x


def check_outputs(got, truth, n):
    sel = truth == TRUE
    bitmap, bytemap, rows = host(got["bitmap"]), host(got["bytemap"]), host(got["rows"])
    assert got["count"] == int(sel.sum())
    assert len(bitmap) == 8 * ((n + 63) // 64)
    bits = np.unpackbits(bitmap, bitorder="little").astype(bool)
    assert np.array_equal(bits[:n], sel), np.flatnonzero(bits[:n] != sel)[:10]
    assert not bits[n:].any()
    assert np.array_equal(bytemap.astype(bool), sel) and set(np.unique(bytemap)) <= {0, 1}
    assert np.array_equal(rows.view(np.uint32), np.flatnonzero(sel).astype(np.uint32))


def leaf_truth(values, fn):
    return np.array([NULL if v is None else (TRUE if fn(v) else FALSE) for v in values], np.uint8)


def string_truth(values, node, consts):
    if node[0] == ISNULL:
        return np.array([TRUE if v is None else FALSE for v in values], np.uint8)
    return leaf_truth(values, string_leaf_fn(node, consts))


def k_and(a, b):
    return np.where((a == FALSE) | (b == FALSE), FALSE, np.where((a == TRUE) & (b == TRUE), TRUE, NULL)).astype(np.uint8)


def k_or(a, b):
    return np.where((a == TRUE) | (b == TRUE), TRUE, np.where((a == FALSE) & (b == FALSE), FALSE, NULL)).astype(np.uint8)


def k_not(a):
    return np.where(a == NULL, NULL, 1 - a).astype(np.uint8)


def run_program(program, leaf):
    """Kleene evaluation of a postfix program; leaf(node) -> truth array."""
    stack = []
    for node in program:
        if node[0] in (AND, OR):
            b, a = stack.pop(), stack.pop()
            stack.append(k_and(a, b) if node[0] == AND else k_or(a, b))
        elif node[0] == NOT:
            stack.append(k_not(stack.pop()))
        else:
            stack.append(leaf(node))
    assert len(stack) == 1
    return stack[0]


def string_leaf_fn(node, consts):
    op, _, _, col2, off, length = node
    c = consts[off:off + length]
    if op == CONTAINS:
        return lambda v: c in v
    if op == LIKE:
        return lambda v: like_model(v, c, col2)
    if op == SW:
        return lambda v: v[:length] == c
    if op == CMPOP:
        return lambda v: v == c
    raise ValueError(op)


@pytest.fixture(scope="module")
def ctx():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from ytsaurus_b200 import GpuContext
    c = GpuContext(0)
    yield c
    c.close()


def _code(fn):
    try:
        fn()
    except capi.YtGpuError as e:
        return e.code
    return capi.OK


GPU_ALPHABET = [b"a", b"b", b"/", b"\n", E, NIHON[:3], NIHON[3:], FOUR, b"\x80", b"\xbf", b"%", b"_", b"\\"]


def exact_bytes(rng, tokens):
    return b"".join(GPU_ALPHABET[int(i)] for i in rng.integers(0, len(GPU_ALPHABET), tokens))


def random_values(rng, n, max_tokens, nullp=0.1):
    return [None if rng.random() < nullp else random_bytes(rng, GPU_ALPHABET, int(rng.integers(0, max_tokens + 1)))
            for _ in range(n)]


def random_patterns(rng, count):
    """-> [(op, escape, bytes)] over the value alphabet plus %, _ and escaped bytes."""
    palpha = [x for x in GPU_ALPHABET if x not in (b"%", b"_", b"\\")] + [b"%", b"%", b"_", b"\\%", b"\\_", b"\\\\"]
    out = []
    for k in range(count):
        if k % 4 == 0:
            out.append((CONTAINS, -1, random_bytes(rng, GPU_ALPHABET, 3)))
        elif k % 4 == 1:
            out.append((LIKE, -1, random_bytes(rng, [x for x in palpha if not x.startswith(b"\\")], 6)))
        else:
            out.append((LIKE, 0x5C, random_bytes(rng, palpha, 6)))
    return out


def pattern_nodes(col, pats):
    """-> (nodes, consts) with one leaf per pattern."""
    consts, nodes = b"", []
    for op, esc, p in pats:
        nodes.append((op, 0, col, esc if op == LIKE else 0, len(consts), len(p)))
        consts += p
    return nodes, consts


# ------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_every_pattern_op_against_the_model(ctx, device):
    rng = np.random.default_rng(211 + int(device))
    for n in (0, 1, 31, 32, 33, 4097):
        values = random_values(rng, n, 12)
        if n >= 33:  # a few values past the staged constants and up to several KB
            for i in rng.choice(n, 3, replace=False):
                values[int(i)] = exact_bytes(rng, int(rng.integers(1000, 3000)))
        pats = random_patterns(rng, 24) + [(LIKE, -1, b""), (LIKE, -1, b"%"), (CONTAINS, -1, b""), (LIKE, -1, b"_%_")]
        nodes, consts = pattern_nodes(0, pats)
        col = strings_to_column(values, device, pad=int(rng.integers(0, 8)))
        for node in nodes:
            got = ctx.evaluate_filter([], [col], [node], (), consts)
            check_outputs(got, leaf_truth(values, string_leaf_fn(node, consts)), n)
            neg = ctx.evaluate_filter([], [col], [node, (NOT,)], (), consts)  # NOT LIKE keeps NULL rows out
            check_outputs(neg, k_not(leaf_truth(values, string_leaf_fn(node, consts))), n)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_cross_checks_with_starts_with(ctx, device):
    rng = np.random.default_rng(223 + int(device))
    n = 4097
    values = random_values(rng, n, 10)
    col = strings_to_column(values, device, pad=3)
    for _ in range(30):
        x = random_bytes(rng, GPU_ALPHABET, 3)
        esc = escape_literal(x)
        consts = x + esc + b"%" + b"%" + esc + b"%"
        sw = ctx.evaluate_filter([], [col], [(SW, 0, 0, 0, 0, len(x))], (), consts)
        like_prefix = ctx.evaluate_filter([], [col], [(LIKE, 0, 0, 0x5C, len(x), len(esc) + 1)], (), consts)
        contains = ctx.evaluate_filter([], [col], [(CONTAINS, 0, 0, 0, 0, len(x))], (), consts)
        like_sub = ctx.evaluate_filter([], [col], [(LIKE, 0, 0, 0x5C, len(x) + len(esc) + 1, len(esc) + 2)], (), consts)
        for a, b in ((sw, like_prefix), (contains, like_sub)):
            assert a["count"] == b["count"]
            assert np.array_equal(host(a["bitmap"]), host(b["bitmap"]))
        check_outputs(contains, leaf_truth(values, lambda v: x in v), n)


def _random_program(rng, leaves, max_nodes=64, max_depth=16):
    while True:
        target = int(rng.integers(1, max_nodes + 1))

        def build(budget):
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


def _mixed_leaves(rng, pats, int_bits):
    nodes, consts = pattern_nodes(1, pats)
    consts_sw = consts + b"a" + b"ab\n"
    base = len(consts)
    nodes += [(SW, 0, 1, 0, base, 1), (CMPOP, capi.CMP_EQ, 1, 0, base + 1, 3), (ISNULL, 0, 1), (ISNULL, 0, 0),
              (CMPOP, capi.CMP_GT, 0, 0, int(int_bits[0]) if len(int_bits) else 0, 0), (CMPOP, capi.CMP_LE, 0, 0, 3, 0)]
    return nodes, consts_sw


def _mixed_truth(prog, consts, ivals, inull, leaf_of_string):
    def leaf(node):
        op, cmp, col = node[0], node[1], node[2]
        if col == 0:
            if op == ISNULL:
                return np.where(inull, TRUE, FALSE).astype(np.uint8)
            c = np.uint64(node[4]).view(np.int64)
            r = ivals > c if cmp == capi.CMP_GT else ivals <= c
            return np.where(inull, NULL, r).astype(np.uint8)
        return leaf_of_string(node)
    return run_program(prog, leaf)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_random_programs_mixing_patterns_with_other_leaves(ctx, device):
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(227 + int(device))
    for n in (1, 31, 33, 4097):
        for _ in range(4):
            values = random_values(rng, n, 10)
            ivals = rng.integers(-5, 6, n, dtype=np.int64)
            inull = rng.random(n) < 0.1
            icol = Column(T.Int64, values=ivals.view(np.uint64).copy(), null_bitmap=np.packbits(inull, bitorder="little"),
                          value_count=n)
            if device:
                icol.values, icol.null_bitmap = _dev(icol.values), _dev(icol.null_bitmap)
            nodes, consts = _mixed_leaves(rng, random_patterns(rng, 8), ivals.view(np.uint64))
            prog = _random_program(rng, nodes)
            want = _mixed_truth(prog, consts, ivals, inull,
                                lambda node: string_truth(values, node, consts))
            got = ctx.evaluate_filter([icol], [strings_to_column(values, device, pad=1)], prog, (), consts)
            check_outputs(got, want, n)


@pytest.mark.gpu
def test_gpu_random_programs_ten_million_rows(ctx):
    """10^7 rows over a pool of distinct values (the model is computed per pool value and gathered)."""
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(229)
    n = 10**7
    pool = list(dict.fromkeys([random_bytes(rng, GPU_ALPHABET, int(rng.integers(0, 14))) for _ in range(400)]))
    heap = b"".join(pool)
    offs = np.cumsum([0] + [len(p) for p in pool])[:-1].astype(np.uint64)
    lens = np.array([len(p) for p in pool], np.uint32)
    idx = rng.integers(0, len(pool), n)
    snull = rng.random(n) < 0.1
    h, st, ln, nl = np.frombuffer(heap, np.uint8).copy(), offs[idx], lens[idx], snull.astype(np.uint8)
    ivals = rng.integers(-5, 6, n, dtype=np.int64)
    inull = rng.random(n) < 0.1
    for device in (False, True):
        nodes, consts = _mixed_leaves(rng, random_patterns(rng, 8), ivals.view(np.uint64))
        prog = _random_program(rng, nodes)

        def string_leaf(node):
            if node[0] == ISNULL:
                return np.where(snull, TRUE, FALSE).astype(np.uint8)
            per = string_truth(pool, node, consts)
            return np.where(snull, NULL, per[idx]).astype(np.uint8)
        want = _mixed_truth(prog, consts, ivals, inull, string_leaf)
        icol = Column(T.Int64, values=ivals.view(np.uint64).copy(), null_bitmap=np.packbits(inull, bitorder="little"),
                      value_count=n)
        scol = (h, st, ln, nl)
        if device:
            icol.values, icol.null_bitmap = _dev(icol.values), _dev(icol.null_bitmap)
            scol = tuple(_dev(x) for x in scol)
        got = ctx.evaluate_filter([icol], [scol], prog, (), consts)
        check_outputs(got, want, n)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_long_values(ctx, device):
    # one 1 MiB value against a pattern that is quadratic for a backtracking matcher
    a = b"a" * (1 << 20)
    values = [a, a + b"b", b"ab", None, a[:1000] + b"b" + a[:7]]
    col = strings_to_column(values, device)
    pat = b"%" + b"a" * 100 + b"b%"
    for op, p in ((LIKE, pat), (CONTAINS, b"a" * 100 + b"b"), (LIKE, b"a%" + b"a" * 100 + b"b"), (LIKE, b"%_b")):
        node = (op, 0, 0, -1 if op == LIKE else 0, 0, len(p))
        got = ctx.evaluate_filter([], [col], [node], (), p)
        check_outputs(got, leaf_truth(values, string_leaf_fn(node, p)), len(values))
    # values longer than 64 KB inside warps of short ones
    rng = np.random.default_rng(233)
    n = 100
    values = random_values(rng, n, 8)
    for i in (3, 40, 70):
        values[i] = exact_bytes(rng, 40000)  # about 72 KB
    col = strings_to_column(values, device, pad=5)
    nodes, consts = pattern_nodes(0, random_patterns(rng, 16) + [(LIKE, -1, b"%b_b%a"), (CONTAINS, -1, b"ab")])
    for node in nodes:
        got = ctx.evaluate_filter([], [col], [node], (), consts)
        check_outputs(got, leaf_truth(values, string_leaf_fn(node, consts)), n)


def _fill_patterns(target):
    """LIKE patterns (escape -1) whose compiled sizes sum to exactly `target` bytes, 40 patterns at most."""
    letters = [bytes([b]) for b in range(0x21, 0x7F) if b not in (0x25, 0x5F)]

    def of_size(size):  # sizes 296 + 16k (k letters, each its own segment) and 288 + 16k (the first two adjacent)
        for k in range(1, 65):
            if 296 + 16 * k == size:
                return b"%".join(letters[:k])
            if k >= 2 and 288 + 16 * k == size:
                return letters[0] + b"%".join(letters[1:k])
        raise ValueError(size)
    out, left = [], target
    while left > 2640:
        out.append(of_size(1320))
        left -= 1320
    half = left // 2 // 8 * 8
    out += [of_size(half), of_size(left - half)]
    assert sum(compiled_size(p) for p in out) == target
    return out


@pytest.mark.gpu
def test_gpu_limits_and_errors(ctx):
    from ytsaurus_b200 import Column
    n = 64
    values = [b"abc", None, b"x" * 300] * (n // 3) + [b"a"] * (n % 3)
    s = strings_to_column(values)
    icol = Column(T.Int64, values=np.arange(n, dtype=np.uint64), value_count=n)
    inv = capi.ERR_INVALID_ARGUMENT

    def ev(prog, consts=b"abc", strings=(s,)):
        return lambda: ctx.evaluate_filter([icol], strings, prog, (), consts)
    # on a scalar column
    assert _code(ev([(CONTAINS, 0, 0, 0, 0, 1)])) == inv and _code(ev([(LIKE, 0, 0, -1, 0, 1)])) == inv
    assert _code(ev([(CONTAINS, 0, 1, 0, 0, 1)])) == capi.OK and _code(ev([(LIKE, 0, 1, -1, 0, 1)])) == capi.OK
    # needle / pattern outside string_constants
    assert _code(ev([(CONTAINS, 0, 1, 0, 1, 2)])) == capi.OK and _code(ev([(CONTAINS, 0, 1, 0, 2, 2)])) == inv
    assert _code(ev([(LIKE, 0, 1, -1, 0, 3)])) == capi.OK and _code(ev([(LIKE, 0, 1, -1, 0, 4)])) == inv
    # the escape: -1 .. 255
    for esc in (-1, 0, 255):
        assert _code(ev([(LIKE, 0, 1, esc, 0, 3)])) == capi.OK
    for esc in (-2, 256):
        assert _code(ev([(LIKE, 0, 1, esc, 0, 3)])) == inv
    # a trailing lone escape; an escaped escape at the end is fine
    assert _code(ev([(LIKE, 0, 1, 0x5C, 0, 3)], b"ab\\")) == inv
    assert _code(ev([(LIKE, 0, 1, 0x5C, 0, 4)], b"ab\\\\")) == capi.OK
    assert _code(ev([(LIKE, 0, 1, -1, 0, 3)], b"ab\\")) == capi.OK  # no escape: an ordinary byte
    # unknown ops next to the new ones
    assert _code(ev([(12, 0, 1)])) == inv and _code(ev([(0, 0, 1)])) == inv
    # positions per pattern: 256 / 257 (LIKE with an escape, _ and literals; CONTAINS by bytes)
    p256 = b"%" + b"_" * 100 + b"\\%" * 50 + b"b" * 106 + b"%"
    assert len(pattern_tokens(p256, 0x5C)) - 2 == 256
    assert _code(ev([(LIKE, 0, 1, 0x5C, 0, len(p256))], p256)) == capi.OK
    assert _code(ev([(LIKE, 0, 1, 0x5C, 0, len(p256) + 1)], p256 + b"c")) == inv
    assert _code(ev([(CONTAINS, 0, 1, 0, 0, 256)], b"q" * 257)) == capi.OK
    assert _code(ev([(CONTAINS, 0, 1, 0, 0, 257)], b"q" * 257)) == inv
    # compiled bytes per call: at the limit / one step (8 bytes) past it
    for target, want in ((capi.FILTER_MAX_PATTERN_BYTES, capi.OK), (capi.FILTER_MAX_PATTERN_BYTES + 8, inv)):
        pats = _fill_patterns(target)
        nodes, consts = pattern_nodes(1, [(LIKE, -1, p) for p in pats])
        prog = nodes[:1] + [x for node in nodes[1:] for x in (node, (OR,))]
        assert len(prog) <= capi.FILTER_MAX_NODES
        if want == capi.OK:
            got = ctx.evaluate_filter([icol], [s], prog, (), consts)
            truth = leaf_truth(values, lambda v: any(like_model(v, p) for p in pats))
            check_outputs(got, truth, n)
        else:
            assert _code(ev(prog, consts)) == inv
    # a string leaving its heap
    h, st, ln, nl = strings_to_column([b"abc"] * n)
    st = st.copy()
    st[n // 2] = len(h) - 1
    assert _code(ev([(LIKE, 0, 1, -1, 0, 1)], b"%", strings=((h, st, ln, nl),))) == inv
    assert _code(ev([(CONTAINS, 0, 1, 0, 0, 1)], b"c", strings=((h, st, ln, nl),))) == inv


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_launch_count(ctx, device):
    rng = np.random.default_rng(239)
    n = 10000
    values = random_values(rng, n, 10)
    col = strings_to_column(values, device)
    prog = [(LIKE, 0, 0, -1, 0, 3), (CONTAINS, 0, 0, 0, 3, 1), (OR,)]
    consts = b"%a_" + b"b"
    before = ctx.launch_count()
    got = ctx.evaluate_filter([], [col], prog, (), consts, want_rows=False)
    assert ctx.launch_count() - before == 1
    want = k_or(leaf_truth(values, lambda v: like_model(v, b"%a_")), leaf_truth(values, lambda v: b"b" in v))
    assert got["rows"] is None and got["count"] == int((want == TRUE).sum())
    before = ctx.launch_count()
    ctx.evaluate_filter([], [col], prog, (), consts, want_rows=True)
    assert ctx.launch_count() - before == 5


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_gpu_groupby_through_a_like_bitmap_matches_the_oracle(ctx, device):
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(241 + int(device))
    n = 20011
    hosts = [b"https://www.site%d.example.com/" % i for i in range(8)] + [b"http://x.example/", "https://ü.example/".encode()]
    values = [None if rng.random() < 0.1 else hosts[int(rng.integers(0, len(hosts)))] + random_bytes(rng, [b"q", b"r", b"/"], 6)
              for _ in range(n)]
    keys = rng.integers(0, 101, n).astype(np.uint64)
    vals = rng.integers(-1000, 1000, n).astype(np.int64).view(np.uint64)
    pat = b"https://www.site_.example.com/%q%"
    f = ctx.evaluate_filter([], [strings_to_column(values, device)], [(LIKE, 0, 0, -1, 0, len(pat))], (), pat)
    sel = leaf_truth(values, lambda v: like_model(v, pat)) == TRUE
    check_outputs(f, np.where(sel, TRUE, FALSE), n)
    kc, vc = Column(T.Int64, values=keys.copy()), Column(T.Int64, values=vals.copy())
    if device:
        kc.values, vc.values = _dev(kc.values), _dev(vc.values)
    bm = Column(T.Boolean, values=f["bitmap"], bit_width=1, value_count=n)
    aggs = [(capi.AGG_SUM, 0), (capi.AGG_MIN, 0), (capi.AGG_COUNT, 0)]
    got = ctx.scan_filter_groupby_multi([kc], [vc, bm], aggs, predicate=(capi.CMP_EQ, 1), predicate_column=1)
    zero = np.zeros(n, np.uint8)
    want = oracle.groupby_multi([keys], [zero], [vals], [zero], [T.Int64], aggs, filt=sel.astype(np.uint8),
                                style=oracle.MINMAX_YQL)
    assert np.array_equal(host(got["count"]), want["count"]) and np.array_equal(host(got["first_row"]), want["first_row"])
    assert np.array_equal(host(got["keys"][0]).view(np.uint64), want["keys"][0])
    for a in range(len(aggs)):
        assert np.array_equal(host(got["value_null"][a]), want["value_null"][a])
        live = want["value_null"][a] == 0
        assert np.array_equal(host(got["values"][a]).view(np.uint64)[live], want["values"][a].view(np.uint64)[live]), a


@pytest.mark.gpu
def test_gpu_host_adapter_like_and_contains():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "host"), "like_ut"], stdout=subprocess.DEVNULL)
    r = subprocess.run([os.path.join(ROOT, "host", "like_ut")], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr

