"""Fixed-width rows across row widths, key layouts and sort-path edges.

ytgpu_sort_fixed_rows, ytgpu_partition_fixed_rows and the one-rank in-box shuffle accept any row width that is a positive
multiple of 16, key columns at any byte offset, INT64 / UINT64 / DOUBLE / BOOLEAN keys and STRING keys of any exact width,
up to 256 normalised key bytes.  Each layout below is chosen to reach one of the key normalisers (scalar, word program
with and without the fused histogram, generic) and the row gather's shift or division path; the sizes reach the plain,
hybrid and packed radix schedules, the multi-chunk prefix sort with its tie fix and its full-LSD fallback, and the edges
of the packed onesweep tile.

References never reuse the GPU's normalised-key encoding: the CPU oracle (TComparator over an equivalent rowset) at every
size, and a plain Python comparator over the decoded values at n <= 5000.  The CPU-only test checks that both agree.
"""
import functools
import math

import numpy as np
import pytest

import oracle
from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import VALUE_DTYPE, EValueType as T, Rowset


@pytest.fixture(scope="module")
def ctx():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from ytsaurus_b200 import GpuContext
    c = GpuContext(0)
    yield c
    c.close()


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()


# ---- layouts: id -> (row_bytes, key columns (offset, width, type, descending)) ----
LAYOUTS = {
    # one 8-byte scalar at an 8-aligned offset: extract_scalar_key_kernel; one granule per row
    "scalar8": (16, [(8, 8, T.Int64, 1)]),
    # odd offset: generic normaliser; 3 granules per row: the gather divides
    "odd_double": (48, [(3, 8, T.Double, 0)]),
    # Boolean: generic normaliser, one active digit (every row ties with many others)
    "boolean": (32, [(5, 1, T.Boolean, 1)]),
    # whole words, 4 chunks: word program with the fused histogram; 5 granules
    "words4": (80, [(16, 8, T.Uint64, 1), (24, 24, T.String, 0)]),
    # whole words, 6 chunks: word program, histogram built by the sort; 7 granules
    "words6": (112, [(0, 40, T.String, 0), (40, 8, T.Int64, 1)]),
    # 33 key bytes at odd offsets: generic normaliser, last chunk partial
    "mixed5": (48, [(0, 1, T.Boolean, 0), (1, 13, T.String, 1), (14, 8, T.Int64, 0), (22, 3, T.String, 0),
                    (25, 8, T.Double, 1)]),
    # 256 key bytes = 32 chunks, the largest normalised key: word program (aligned) and generic (odd offset)
    "max256": (272, [(8, 256, T.String, 0)]),
    "max256_odd": (272, [(5, 256, T.String, 0)]),
    # rows of 64 KiB and more: the word program's 16-bit offsets do not reach, generic normaliser
    "wide_row": (65552, [(65536, 8, T.Uint64, 0)]),
}

_ALPHABET = np.array([0x00, 0x01, 0x61, 0x62, 0xFF], dtype=np.uint8)
_BOOL_BYTES = np.array([0, 1, 2, 255], dtype=np.uint8)
_INT_POOL = np.array([0, 1, 2, 255, 256, 1 << 32, (1 << 63) - 1, 1 << 63, (1 << 64) - 1, (1 << 64) - 2,
                      0x0123456789ABCDEF, 0xFEDCBA9876543210, 0x8000000000000001, 0x7FFFFFFFFFFFFF00], dtype=np.uint64)
_DOUBLE_POOL = np.array([
    0x7FF8000000000000, 0x7FF0000000000001, 0xFFF8000000000000, 0x7FFFFFFFFFFFFFFF, 0xFFF0000000000123,  # NaNs
    0x0000000000000000, 0x8000000000000000,  # +0, -0
    0x7FF0000000000000, 0xFFF0000000000000,  # +inf, -inf
    0x0000000000000001, 0x8000000000000001, 0x000FFFFFFFFFFFFF, 0x800FFFFFFFFFFFFF,  # denormals
    0x3FF0000000000000, 0xBFF0000000000000, 0x3FF8000000000000, 0xC004000000000000,  # +-1, 1.5, -2.5
], dtype=np.uint64)


def _scalar_words(rng, n, typ):
    """n key values as raw little-endian words: half of them from a pool of edge values (ties, extremes)."""
    if typ == T.Double:
        x = rng.normal(size=n) * np.power(10.0, rng.integers(-300, 300, n))
        words = x.view(np.uint64).copy()
        pool = _DOUBLE_POOL
    else:
        words = rng.integers(0, 2**64 - 1, n, dtype=np.uint64, endpoint=True)
        pool = _INT_POOL
    pick = rng.random(n) < 0.5
    words[pick] = pool[rng.integers(0, len(pool), int(pick.sum()))]
    return words


def _strings(rng, n, width):
    """Strings over a small alphabet that share prefixes of every length: each row copies one of a few base strings
    up to a random position and draws the rest."""
    base = _ALPHABET[rng.integers(0, len(_ALPHABET), (32, width))]
    rows = base[rng.integers(0, 32, n)]
    cut = rng.integers(0, width + 1, n)
    tail = _ALPHABET[rng.integers(0, len(_ALPHABET), (n, width))]
    return np.where(np.arange(width)[None, :] >= cut[:, None], tail, rows)


def _make_rows(rng, row_bytes, cols, n):
    rows = rng.integers(0, 256, (n, row_bytes), dtype=np.uint8)
    for off, width, typ, _ in cols:
        if typ == T.String:
            rows[:, off:off + width] = _strings(rng, n, width)
        elif typ == T.Boolean:
            rows[:, off] = _BOOL_BYTES[rng.integers(0, len(_BOOL_BYTES), n)]
        else:
            rows[:, off:off + 8] = _scalar_words(rng, n, typ).view(np.uint8).reshape(n, 8)
    return rows


def _key_spec(cols):
    return [(off, width, typ, desc, 1) for off, width, typ, desc in cols]


# ---- references ----
def _decode(rows, cols):
    """Row i -> tuple of Python values of its key columns."""
    per_col = []
    for off, width, typ, _ in cols:
        if typ == T.String:
            per_col.append([bytes(r) for r in rows[:, off:off + width]])
        elif typ == T.Boolean:
            per_col.append((rows[:, off] != 0).tolist())
        else:
            dt = {T.Int64: "<i8", T.Uint64: "<u8", T.Double: "<f8"}[typ]
            per_col.append(np.ascontiguousarray(rows[:, off:off + 8]).view(dt).reshape(-1).tolist())
    return list(zip(*per_col)) if per_col else []


def _compare_values(typ, a, b):
    if typ == T.Double:  # NaN is the largest value and equals every NaN; -0.0 == 0.0 falls out of float comparison
        an, bn = math.isnan(a), math.isnan(b)
        if an or bn:
            return (an > bn) - (an < bn)
    return (a > b) - (a < b)


def _compare_keys(cols, x, y):
    for (_, _, typ, desc), a, b in zip(cols, x, y):
        c = _compare_values(typ, a, b)
        if c:
            return -c if desc else c
    return 0


def _python_perm(rows, cols):
    """Stable sort by the plain comparator (Python's sort is stable)."""
    keys = _decode(rows, cols)
    order = sorted(range(len(keys)), key=functools.cmp_to_key(lambda i, j: _compare_keys(cols, keys[i], keys[j])))
    return np.array(order, dtype=np.uint32)


def _oracle_perm(rows, row_bytes, cols):
    perm, _ = oracle.sort_fixed_rows(rows, row_bytes, cols, oracle.SORT_STABLE)
    return perm


def _rowset(rows, cols):
    """The equivalent rowset: one typed value per key column; a string is the column's exact `width` bytes (its heap is
    the rows themselves), a boolean is `byte != 0`."""
    n, row_bytes = rows.shape
    vals = np.zeros((n, len(cols)), dtype=VALUE_DTYPE)
    for c, (off, width, typ, _) in enumerate(cols):
        vals["id"][:, c] = c
        vals["type"][:, c] = typ
        if typ == T.String:
            vals["length"][:, c] = width
            vals["data"][:, c] = np.arange(n, dtype=np.uint64) * np.uint64(row_bytes) + np.uint64(off)
        elif typ == T.Boolean:
            vals["data"][:, c] = rows[:, off] != 0
        else:
            vals["data"][:, c] = np.ascontiguousarray(rows[:, off:off + 8]).view(np.uint64).reshape(-1)
    return vals, np.ascontiguousarray(rows).reshape(-1)


def _desc(cols):
    return [d for _, _, _, d in cols]


# ---- 1. the references agree with each other (no device needed) ----
@pytest.mark.parametrize("layout", sorted(LAYOUTS))
def test_python_comparator_matches_oracle(layout):
    row_bytes, cols = LAYOUTS[layout]
    n = 300 if row_bytes > 4096 else 3000
    rng = np.random.default_rng(7 + len(layout))
    rows = _make_rows(rng, row_bytes, cols, n)
    want = _python_perm(rows, cols)
    assert (_oracle_perm(rows, row_bytes, cols) == want).all()
    vals, heap = _rowset(rows, cols)
    perm, _ = oracle.sort_rows(vals, heap, len(cols), _desc(cols), oracle.SORT_STABLE)
    assert (perm == want).all()


def test_comparator_rules():
    # NaN payloads tie with each other above +inf, -0 ties with +0, any nonzero boolean byte is true, strings are bytewise,
    # Int64 is signed and Uint64 unsigned
    d = lambda bits: float(np.array([bits], dtype=np.uint64).view(np.float64)[0])  # noqa: E731
    assert _compare_values(T.Double, d(0x7FF8000000000000), d(0xFFF0000000000123)) == 0
    assert _compare_values(T.Double, d(0x7FF0000000000001), d(0x7FF0000000000000)) == 1
    assert _compare_values(T.Double, -0.0, 0.0) == 0
    assert _compare_values(T.Double, d(0x8000000000000001), -0.0) == -1
    rows = np.zeros((4, 32), dtype=np.uint8)
    rows[:, 5] = [255, 0, 2, 1]
    assert _python_perm(rows, [(5, 1, T.Boolean, 0)]).tolist() == [1, 0, 2, 3]
    assert _python_perm(rows, [(5, 1, T.Boolean, 1)]).tolist() == [0, 2, 3, 1]
    rows = np.zeros((2, 16), dtype=np.uint8)
    rows[0, 0:8] = np.array([1 << 63], dtype=np.uint64).view(np.uint8)
    rows[1, 0:8] = np.array([1], dtype=np.uint64).view(np.uint8)
    assert _python_perm(rows, [(0, 8, T.Int64, 0)]).tolist() == [0, 1]
    assert _python_perm(rows, [(0, 8, T.Uint64, 0)]).tolist() == [1, 0]
    rows[0, 8:11] = [0x61, 0xFF, 0x00]
    rows[1, 8:11] = [0x61, 0x01, 0xFF]
    assert _python_perm(rows, [(8, 3, T.String, 0)]).tolist() == [1, 0]
    assert _python_perm(rows, [(8, 3, T.String, 1)]).tolist() == [0, 1]


# ---- 2. sort: every layout, both memory flavours ----
_SIZES = [0, 1, 2, 33, 4097, 100_003]
_LARGE = [2**18 - 1, 2**18, 300_001]  # 2^18 rows and more: hybrid / packed schedules of the single-chunk sort
SORT_CASES = ([(lay, n) for lay in sorted(LAYOUTS) if lay != "wide_row" for n in _SIZES]
              + [("wide_row", n) for n in (0, 1, 2, 33, 1000)]
              + [(lay, n) for lay in ("scalar8", "words4", "mixed5") for n in _LARGE])


@pytest.mark.gpu
@pytest.mark.parametrize("layout,n", SORT_CASES, ids=[f"{lay}-{n}" for lay, n in SORT_CASES])
def test_sort_layout_matches_references(ctx, layout, n):
    row_bytes, cols = LAYOUTS[layout]
    rng = np.random.default_rng(n * 131 + len(layout))
    rows = _make_rows(rng, row_bytes, cols, n)
    want = _oracle_perm(rows, row_bytes, cols)
    if n <= 5000:
        assert (_python_perm(rows, cols) == want).all()
    spec = _key_spec(cols)
    out, perm = ctx.sort_fixed_rows(_dev(rows), row_bytes, spec, want_rows=True, want_perm=True)
    assert (perm.cpu().numpy().view(np.uint32) == want).all()
    assert (out.cpu().numpy().reshape(n, row_bytes) == rows[want]).all()
    out_h, perm_h = ctx.sort_fixed_rows(rows.reshape(-1), row_bytes, spec, want_rows=True, want_perm=True)
    assert (perm_h == want).all()
    assert (out_h.reshape(n, row_bytes) == rows[want]).all()


# ---- 3. multi-chunk keys: the prefix sort over the 8 most significant active bytes, its tie fix and the fallback ----
_PREFIX_ROW_BYTES = 32
_PREFIX_COLS = [(0, 8, T.Uint64, 0), (8, 16, T.String, 0)]  # 24 normalised bytes = 3 chunks


def _prefix_rows(rng, int_bytes, str_bytes, n):
    """Rows whose key varies only in the low `int_bytes` bytes of the integer and the first `str_bytes` string bytes
    (each drawn from all 256 values); every other key byte is constant."""
    rows = rng.integers(0, 256, (n, _PREFIX_ROW_BYTES), dtype=np.uint8)
    rows[:, 0:8] = 0x5A
    rows[:, 0:int_bytes] = rng.integers(0, 256, (n, int_bytes), dtype=np.uint8)  # little-endian: the low bytes
    rows[:, 8:24] = 0x61
    rows[:, 8:8 + str_bytes] = rng.integers(0, 256, (n, str_bytes), dtype=np.uint8)
    return rows


def _with_prefix_group(rng, rows, size):
    """Gives `size` random rows (spread over the input) the first row's key prefix (5 integer bytes and 3 string bytes)
    with distinct 9th bytes, so that they form one run of equal prefixes that mixes different keys."""
    at = rng.choice(len(rows), size, replace=False)
    rows[at, 0:8] = rows[at[0], 0:8]
    rows[at, 8:11] = rows[at[0], 8:11]
    rows[at, 11] = rng.permutation(256)[:size]
    return rows


def _groups_of(rng, rows, group):
    """Every `group` consecutive rows share their prefix (5 integer bytes, 3 string bytes); then the rows are shuffled."""
    lead = (np.arange(len(rows)) // group) * group
    rows[:, 0:8] = rows[lead, 0:8]
    rows[:, 8:11] = rows[lead, 8:11]
    return rows[rng.permutation(len(rows))]


def _sort_and_check(ctx, rows, row_bytes, cols):
    want = _oracle_perm(rows, row_bytes, cols)
    if len(rows) <= 5000:
        assert (_python_perm(rows, cols) == want).all()
    out, perm = ctx.sort_fixed_rows(_dev(rows), row_bytes, _key_spec(cols), want_rows=True, want_perm=True)
    assert (perm.cpu().numpy().view(np.uint32) == want).all()
    assert (out.cpu().numpy().reshape(len(rows), row_bytes) == rows[want]).all()
    return ctx.last_sort_passes()


def _active_bytes(rows, cols):
    """Key bytes that are not constant over the rows (the sort's active digits)."""
    return sum(len(np.unique(rows[:, off + k])) > 1 for off, width, _, _ in cols for k in range(width))


@pytest.mark.gpu
def test_prefix_sort_nine_active_bytes_tie_fix_orders_ninth_byte(ctx):
    # 5 integer + 4 string bytes vary: the prefix holds 8 of them, rows with equal prefixes (groups of 8) differ in the
    # 9th, and only the tie fix orders them
    rng = np.random.default_rng(91)
    rows = _groups_of(rng, _prefix_rows(rng, 5, 4, 4000), 8)
    assert _active_bytes(rows, _PREFIX_COLS) == 9
    assert _sort_and_check(ctx, rows, _PREFIX_ROW_BYTES, _PREFIX_COLS) <= 8


@pytest.mark.gpu
def test_prefix_sort_eight_active_bytes_is_complete(ctx):
    # 4 integer + 4 string bytes: the prefix is the whole key, ties are true duplicates kept in input order
    rng = np.random.default_rng(92)
    rows = _prefix_rows(rng, 4, 4, 4000)
    rows[:, 0:24] = rows[rng.integers(0, 1000, 4000), 0:24]  # 1000 distinct keys
    assert _active_bytes(rows, _PREFIX_COLS) == 8
    assert _sort_and_check(ctx, rows, _PREFIX_ROW_BYTES, _PREFIX_COLS) <= 8


@pytest.mark.gpu
@pytest.mark.parametrize("n", [4000, 300_001])  # 300 001 rows: the prefix sort itself takes the hybrid schedule
@pytest.mark.parametrize("run", [32, 33])
def test_prefix_sort_tie_run_limit(ctx, run, n):
    # a run of 32 equal prefixes is insertion-sorted; 33 sends the whole key to the complete LSD over every chunk
    rng = np.random.default_rng(93 + run + n)
    rows = _with_prefix_group(rng, _prefix_rows(rng, 5, 4, n), run)
    assert _active_bytes(rows, _PREFIX_COLS) == 9
    passes = _sort_and_check(ctx, rows, _PREFIX_ROW_BYTES, _PREFIX_COLS)
    if run == 32:
        assert passes <= 8
    else:
        assert passes == 9


@pytest.mark.gpu
def test_prefix_sort_clustered_prefix_chunk_takes_its_complete_schedule(ctx):
    # The prefix chunk's three most significant bytes (integer bytes 4, 3, 2) take four values: its hybrid sort (3 passes)
    # leaves four long runs that mix keys and sorts the chunk again with every active byte (8 passes).  Rows with equal
    # prefixes (groups of 8) differ in the 9th byte: the tie fix orders them through the keys of that second sort.
    n = 2**18
    rng = np.random.default_rng(94)
    rows = _prefix_rows(rng, 5, 4, n)
    rows[:, 2:5] = rng.integers(0, 256, (4, 3), dtype=np.uint8)[rng.integers(0, 4, n)]
    rows = _groups_of(rng, rows, 8)
    assert _active_bytes(rows, _PREFIX_COLS) == 9
    assert _sort_and_check(ctx, rows, _PREFIX_ROW_BYTES, _PREFIX_COLS) == 3 + 8


# ---- 4. single-chunk sorts of >= 2^18 rows: packed onesweep tile edges (6144 items per tile) ----
_TILE = 6144
_PACKED_SIZES = [2**18, 43 * _TILE, 43 * _TILE + 1, 43 * _TILE + 769, 300_001]


def _packed_keys(rng, shape, n):
    if shape == "t1_top_byte":
        return rng.integers(0, 256, n, dtype=np.uint64) << np.uint64(56)
    if shape == "t2_digits_1_6":
        return ((rng.integers(0, 256, n, dtype=np.uint64) << np.uint64(8)) | (rng.integers(0, 256, n, dtype=np.uint64) << np.uint64(48))
                | np.uint64(0x5500334455660077))
    if shape == "t4_digits_0_2_5_7":
        k = np.zeros(n, dtype=np.uint64)
        for d in (0, 2, 5, 7):
            k |= rng.integers(0, 256, n, dtype=np.uint64) << np.uint64(8 * d)
        return k | np.uint64(0x00CC00DDEE00FF00)
    keys = rng.integers(0, 2**64 - 1, n, dtype=np.uint64, endpoint=True)
    if shape == "random64":
        return keys
    if shape == "long_mixed_runs":
        # four runs of 64 keys that share their top 3 bytes and differ below: the packed side re-sort
        for r in range(4):
            at = rng.choice(n, 64, replace=False)
            keys[at] = (keys[at] & np.uint64(0xFFFFFFFFFF)) | (np.uint64(0xA0B0C0 + r) << np.uint64(40))
        return keys
    assert shape == "clustered"  # four top-3-byte prefixes: long mixed runs everywhere, the complete schedule
    v = rng.integers(0, 4, n, dtype=np.uint64)
    one = np.uint64(1)
    return (keys & np.uint64(0xFFFFFFFFFF)) | (v << np.uint64(40)) | ((v & one) << np.uint64(48)) | ((v >> one) << np.uint64(56))


def _hybrid_need(n):
    need, span = 1, 256
    while span < 16 * n and need < 8:
        span <<= 8
        need += 1
    return need


def _sort_keys16(ctx, keys):
    n = len(keys)
    rows = np.random.default_rng(n).integers(0, 256, (n, 16), dtype=np.uint8)
    rows[:, :8] = keys.view(np.uint8).reshape(n, 8)
    want = np.argsort(keys, kind="stable").astype(np.uint32)
    out, perm = ctx.sort_fixed_rows(_dev(rows), 16, [(0, 8, T.Uint64, 0, 1)], want_rows=True, want_perm=True)
    assert (perm.cpu().numpy().view(np.uint32) == want).all()
    assert (out.cpu().numpy().reshape(n, 16) == rows[want]).all()
    active = sum(len(np.unique((keys >> np.uint64(8 * d)) & np.uint64(0xFF))) > 1 for d in range(8))
    return active, ctx.last_sort_passes()


@pytest.mark.gpu
@pytest.mark.parametrize("n", _PACKED_SIZES)
@pytest.mark.parametrize("shape", ["t1_top_byte", "t2_digits_1_6", "t4_digits_0_2_5_7", "random64", "long_mixed_runs",
                                   "clustered"])
def test_packed_onesweep_tile_edges(ctx, shape, n):
    rng = np.random.default_rng(n + 17 * len(shape))
    active, passes = _sort_keys16(ctx, _packed_keys(rng, shape, n))
    need = _hybrid_need(n)
    if active < need + 2:  # plain schedule: one packed pass per active digit
        assert passes == active
    elif shape == "clustered":  # hybrid passes, then the complete schedule
        assert passes == need + active
    else:  # hybrid: the top `need` digits, short runs fixed up, the few long mixed runs re-sorted on the side
        assert passes == need


@pytest.mark.gpu
def test_pair_format_read_plan_without_hybrid(ctx):
    # hybrid off: 5 active digits do not fit the packed word's 32-bit prefix, so the plan read back launches pair passes
    n = 300_001
    rng = np.random.default_rng(55)
    keys = rng.integers(0, 2**40, n, dtype=np.uint64) << np.uint64(16)
    before = ctx.get_option("sort_hybrid")
    ctx.set_option("sort_hybrid", 0)
    try:
        active, passes = _sort_keys16(ctx, keys)
    finally:
        ctx.set_option("sort_hybrid", 0 if before == 0 else 1)
    assert active == 5 and passes == 5


# ---- 5. partitioning ----
PARTITION_LAYOUTS = ["odd_double", "boolean", "words4", "mixed5"]
_PARTITION_ROWS = 40_003


def _pivot_rows(rows, row_bytes, cols, count):
    """`count` rows at evenly spaced positions of the sorted order (sorted samples)."""
    order = _oracle_perm(rows, row_bytes, cols)
    return rows[order[np.linspace(0, len(rows) - 1, count + 2).astype(np.int64)[1:-1]]]


def _hand_made_bounds(rng, pivots, cols):
    """Bounds from sorted pivot rows with the prefix lengths cycling through 1..ncols, alternating inclusiveness, and
    strings in the prefix cut shorter than their column width (the cut string is a prefix of the pivot's key, and of
    every key that shares it)."""
    k = len(cols)
    P = len(pivots) + 1
    vals = np.zeros((P, k), dtype=VALUE_DTYPE)
    heap = bytearray()
    blen, binc = [0], [1]
    for b in range(1, P):
        piv = pivots[b - 1]
        plen = 1 + (b - 1) % k
        for c, (off, width, typ, _) in enumerate(cols[:plen]):
            v = vals[b, c]
            v["id"] = c
            v["type"] = typ
            if typ == T.String:
                length = width if (b + c) % 2 else int(rng.integers(0, width))
                v["length"] = length
                v["data"] = len(heap)
                heap += piv[off:off + length].tobytes()
            elif typ == T.Boolean:
                v["data"] = int(piv[off] != 0)
            else:
                v["data"] = int(piv[off:off + 8].copy().view(np.uint64)[0])
        blen.append(plen)
        binc.append(b % 2)
    return Rowset(vals, np.frombuffer(bytes(heap) or b"\0", dtype=np.uint8).copy()), blen, binc


def _ordered_bounds(rng, rows, row_bytes, cols, P, kind):
    from ytsaurus_b200.shuffle import pivot_bounds_from_rows
    pivots = _pivot_rows(rows, row_bytes, cols, P - 1)
    if kind == "sorted_samples":
        return pivot_bounds_from_rows(pivots, _key_spec(cols))
    return _hand_made_bounds(rng, pivots, cols)


def _check_partition(ctx, rows, row_bytes, spec, want, P):
    n = len(rows)
    hist_want = np.bincount(want, minlength=P).astype(np.uint64)
    slabs_want = rows[np.argsort(want, kind="stable")]
    idx, hist, slabs = ctx.partition_fixed_rows(_dev(rows), row_bytes, spec)
    assert (idx.cpu().numpy() == want).all()
    assert (hist.cpu().numpy().view(np.uint64) == hist_want).all()
    assert (slabs.cpu().numpy().reshape(n, row_bytes) == slabs_want).all()
    idx, hist, slabs = ctx.partition_fixed_rows(rows.reshape(-1), row_bytes, spec)
    assert (idx == want).all()
    assert (hist == hist_want).all()
    assert (slabs.reshape(n, row_bytes) == slabs_want).all()


@pytest.mark.gpu
@pytest.mark.parametrize("bounds_kind", ["sorted_samples", "hand_made"])
@pytest.mark.parametrize("P", [2, 9, 5000])  # 5000 > 4096: the histogram lives in global memory
@pytest.mark.parametrize("layout", PARTITION_LAYOUTS)
def test_ordered_partition_matches_oracle(ctx, layout, P, bounds_kind):
    row_bytes, cols = LAYOUTS[layout]
    rng = np.random.default_rng(P * 7 + len(layout) + len(bounds_kind))
    rows = _make_rows(rng, row_bytes, cols, _PARTITION_ROWS)
    bounds, blen, binc = _ordered_bounds(rng, rows, row_bytes, cols, P, bounds_kind)
    vals, heap = _rowset(rows, cols)
    want, _ = oracle.partition_ordered(vals, heap, len(cols), _desc(cols), bounds.values, bounds.heap, blen, binc)
    spec = ctx._partition_spec(capi.PARTITION_ORDERED, P, key_columns=_key_spec(cols), bounds=bounds,
                               bound_prefix_length=blen, bound_inclusive=binc)
    _check_partition(ctx, rows, row_bytes, spec, want, P)


@pytest.mark.gpu
def test_ordered_partition_short_string_bound_splits_its_prefix(ctx):
    # keys that start with a bound string shorter than the column are greater than the bound (ascending column) and
    # smaller than it (descending column): an exclusive and an inclusive bound must both let them pass, resp. not pass
    rng = np.random.default_rng(31)
    for desc in (0, 1):
        cols = [(3, 12, T.String, desc)]
        rows = _make_rows(rng, 32, cols, 5000)
        rows[:2500, 3:6] = [0x61, 0x62, 0x61]
        rows[:10, 6:15] = 0  # the bound string padded with zeros: still longer than the bound
        bound = Rowset(np.zeros((2, 1), dtype=VALUE_DTYPE), np.frombuffer(b"aba", dtype=np.uint8).copy())
        bound.values[1, 0]["type"] = T.String
        bound.values[1, 0]["length"] = 3
        for incl in (0, 1):
            vals, heap = _rowset(rows, cols)
            want, _ = oracle.partition_ordered(vals, heap, 1, [desc], bound.values, bound.heap, [0, 1], [1, incl])
            assert (want[:2500] == (0 if desc else 1)).all()
            spec = ctx._partition_spec(capi.PARTITION_ORDERED, 2, key_columns=_key_spec(cols), bounds=bound,
                                       bound_prefix_length=[0, 1], bound_inclusive=[1, incl])
            _check_partition(ctx, rows, 32, spec, want, 2)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [9, 5000])
@pytest.mark.parametrize("layout", PARTITION_LAYOUTS)
def test_hash_partition_matches_oracle(ctx, layout, P):
    row_bytes, cols = LAYOUTS[layout]
    rng = np.random.default_rng(P + 3 * len(layout))
    rows = _make_rows(rng, row_bytes, cols, _PARTITION_ROWS)
    vals, heap = _rowset(rows, cols)
    for kcc in range(1, len(cols) + 1):
        salt = 0x5EED + kcc
        want, _ = oracle.partition_hash(vals, heap, P, kcc, salt)
        spec = ctx._partition_spec(capi.PARTITION_HASH, P, key_columns=_key_spec(cols), key_column_count=kcc, salt=salt)
        _check_partition(ctx, rows, row_bytes, spec, want, P)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["odd_double", "words4", "mixed5"])
def test_one_rank_shuffle_matches_oracle(ctx, layout):
    from ytsaurus_b200.shuffle import NativeShuffleSorter
    row_bytes, cols = LAYOUTS[layout]
    n = 150_000
    rng = np.random.default_rng(77 + len(layout))
    rows = _make_rows(rng, row_bytes, cols, n)
    want = _oracle_perm(rows, row_bytes, cols)
    s = NativeShuffleSorter(ctx, capacity_rows=n + 16, row_bytes=row_bytes)
    try:
        out, stats = s.sort(_dev(rows), row_bytes, _key_spec(cols))
        assert stats.rows_in == n and stats.rows_out == n
        assert (out.cpu().numpy().reshape(n, row_bytes) == rows[want]).all()
    finally:
        s.close()


# ---- 6. argument errors leave the caller's outputs untouched ----
_FILL = 0xA5
_ERROR_CASES = [  # (id, row_bytes, key columns (offset, width, type, descending), expected code)
    ("row_bytes_24", 24, [(0, 8, T.Uint64, 0)], capi.ERR_INVALID_ARGUMENT),
    ("scalar_past_row_end", 32, [(28, 8, T.Uint64, 0)], capi.ERR_INVALID_ARGUMENT),
    ("string_crosses_row_end", 32, [(0, 8, T.Int64, 0), (20, 13, T.String, 0)], capi.ERR_INVALID_ARGUMENT),
    ("string_width_0", 32, [(0, 0, T.String, 0)], capi.ERR_INVALID_ARGUMENT),
    ("null_type", 32, [(0, 8, T.Null, 0)], capi.ERR_INVALID_ARGUMENT),
    ("any_type", 32, [(0, 8, T.Any, 0)], capi.ERR_UNSUPPORTED),
    ("composite_type", 32, [(0, 8, T.Composite, 0)], capi.ERR_UNSUPPORTED),
    ("key_257_bytes", 272, [(0, 1, T.Boolean, 0), (1, 256, T.String, 0)], capi.ERR_UNSUPPORTED),
]
_ERROR_ROWS = 100


def _filled(nbytes, mem):
    """An output buffer of `nbytes` bytes, every byte _FILL."""
    import torch
    a = np.full(nbytes, _FILL, dtype=np.uint8)
    return a if mem == capi.MEM_HOST else torch.from_numpy(a).cuda()


def _host(x):
    return x if isinstance(x, np.ndarray) else x.cpu().numpy()


def _untouched(*bufs):
    return all((_host(b) == _FILL).all() for b in bufs)


def _ptr(x):
    return x.ctypes.data if isinstance(x, np.ndarray) else x.data_ptr()


@pytest.mark.gpu
@pytest.mark.parametrize("mem", [capi.MEM_DEVICE, capi.MEM_HOST], ids=["device", "host"])
@pytest.mark.parametrize("case", _ERROR_CASES, ids=[c[0] for c in _ERROR_CASES])
def test_sort_argument_errors(ctx, case, mem):
    import ctypes as C
    _, row_bytes, cols, code = case
    rows = np.random.default_rng(1).integers(0, 256, _ERROR_ROWS * row_bytes, dtype=np.uint8)
    src = rows if mem == capi.MEM_HOST else _dev(rows)
    out_rows = _filled(_ERROR_ROWS * row_bytes, mem)
    out_perm = _filled(_ERROR_ROWS * 4, mem)
    view = capi.FixedRowsView(_ptr(src), _ERROR_ROWS, row_bytes, mem)
    spec = capi.make_sort_spec(_key_spec(cols))
    err = capi.Error()
    got = ctx.lib.ytgpu_sort_fixed_rows(ctx.handle, C.byref(view), C.byref(spec), _ptr(out_rows), _ptr(out_perm), mem,
                                        C.byref(err))
    assert got == code, err.message
    assert _untouched(out_rows, out_perm)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [capi.PARTITION_ORDERED, capi.PARTITION_HASH], ids=["ordered", "hash"])
@pytest.mark.parametrize("mem", [capi.MEM_DEVICE, capi.MEM_HOST], ids=["device", "host"])
@pytest.mark.parametrize("case", _ERROR_CASES, ids=[c[0] for c in _ERROR_CASES])
def test_partition_argument_errors(ctx, case, mem, kind):
    import ctypes as C
    _, row_bytes, cols, code = case
    rows = np.random.default_rng(2).integers(0, 256, _ERROR_ROWS * row_bytes, dtype=np.uint8)
    src = rows if mem == capi.MEM_HOST else _dev(rows)
    P = 2
    if kind == capi.PARTITION_ORDERED:
        bounds = Rowset(np.zeros((P, len(cols)), dtype=VALUE_DTYPE), np.zeros(1, dtype=np.uint8))  # universal bounds
        spec = ctx._partition_spec(kind, P, key_columns=_key_spec(cols), bounds=bounds, bound_prefix_length=[0, 0],
                                   bound_inclusive=[1, 1])
    else:
        spec = ctx._partition_spec(kind, P, key_columns=_key_spec(cols), key_column_count=len(cols))
    out_index = _filled(_ERROR_ROWS * 4, mem)
    out_hist = _filled(P * 8, mem)
    out_slabs = _filled(_ERROR_ROWS * row_bytes, mem)
    view = capi.FixedRowsView(_ptr(src), _ERROR_ROWS, row_bytes, mem)
    err = capi.Error()
    got = ctx.lib.ytgpu_partition_fixed_rows(ctx.handle, C.byref(view), C.byref(spec), _ptr(out_index), _ptr(out_hist),
                                             _ptr(out_slabs), mem, C.byref(err))
    assert got == code, err.message
    assert _untouched(out_index, out_hist, out_slabs)


@pytest.mark.gpu
@pytest.mark.parametrize("case", _ERROR_CASES, ids=[c[0] for c in _ERROR_CASES])
def test_shuffle_argument_errors(ctx, case):
    _, row_bytes, cols, code = case
    if row_bytes % 16:
        with pytest.raises(capi.YtGpuError) as e:
            ctx.shuffle_create(1, 0, _ERROR_ROWS, row_bytes)
        assert e.value.code == code
        return
    rows = _dev(np.random.default_rng(3).integers(0, 256, _ERROR_ROWS * row_bytes, dtype=np.uint8))
    out = _filled(_ERROR_ROWS * row_bytes, capi.MEM_DEVICE)
    handle, _ = ctx.shuffle_create(1, 0, _ERROR_ROWS, row_bytes)
    try:
        with pytest.raises(capi.YtGpuError) as e:
            ctx.shuffle_sort(handle, rows, row_bytes, _key_spec(cols), out)
        assert e.value.code == code
        assert _untouched(out)
    finally:
        ctx.shuffle_destroy(handle)
