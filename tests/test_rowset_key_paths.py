"""Rowset sort, merge, sorted join and ordered partitioning on normalised keys, across key layouts, string widths and
the sort paths, against a plain Python restatement of CompareRowValues + TComparator.

The byte rules of keys.cuh are property-tested on the CPU elsewhere; this file tests the device machinery around them:
string width measurement, normalize_rowset_kernel, the multi-chunk radix path (prefix chunk, deep_tie_fix_kernel, the
complete-schedule fallback), the gather of value_count * 16-byte rows, the merge path over up to 32 chunks, the join-key
prefix mask and the ordered partition kernel, on both sides of the 256-byte limit of the normalised form.

The Python model (`compare_values`, `model_*`) is pinned against the oracle on every layout by the CPU tests.  The GPU
tests compare with the model up to MODEL_ROWS rows and with the oracle above that, bit for bit."""
import functools
import heapq
import struct

import numpy as np
import pytest

import oracle
from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import EValueType as T, Rowset, VALUE_DTYPE

MODEL_ROWS = 20_000
HYBRID_MIN_ROWS = 1 << 18  # radix_sort.cu kHybridMinRows
I64_MIN, I64_MAX, U64_MAX = -2**63, 2**63 - 1, 2**64 - 1


# ------------------------------------------------------------------------------------------------------------- model
def _as_double(bits):
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


def compare_values(a, b):
    """CompareRowValues on decoded (type, payload) pairs: type code first; Int64 signed, Uint64 unsigned; Double with
    -0.0 == +0.0 and every NaN equal to every other NaN and above +inf; Boolean; bytes lexicographically with a proper
    prefix first; Null and the Min / Max sentinels equal to themselves."""
    ta, va = a
    tb, vb = b
    if ta != tb:
        return -1 if ta < tb else 1
    if ta == T.Double:
        na, nb = va != va, vb != vb
        if na or nb:
            return (na > nb) - (na < nb)
    elif ta not in (T.Int64, T.Uint64, T.Boolean, T.String):
        return 0
    return (va > vb) - (va < vb)


def compare_rows(a, b, desc):
    """TComparator::CompareKeys over the columns of a (a and b have as many): a descending column inverts its result."""
    for i in range(len(a)):
        c = compare_values(a[i], b[i])
        if c:
            return -c if desc[i] else c
    return 0


def decode(values, heap, key_idx):
    """Key values of every row as tuples of (type, payload)."""
    hb = bytes(heap)
    out = []
    for row in values[:, key_idx].tolist():
        key = []
        for _, t, _, length, data in row:
            if t == T.Int64:
                key.append((t, data - (1 << 64) if data >> 63 else data))
            elif t == T.Uint64:
                key.append((t, data))
            elif t == T.Double:
                key.append((t, _as_double(data)))
            elif t == T.Boolean:
                key.append((t, (data & 0xFF) != 0))
            elif t == T.String:
                key.append((t, hb[data:data + length]))
            else:
                key.append((t, None))
        out.append(tuple(key))
    return out


def model_sort(keys, desc):
    """Stable sort: ties keep input order."""
    return np.array(sorted(range(len(keys)), key=functools.cmp_to_key(lambda i, j: compare_rows(keys[i], keys[j], desc))),
                    dtype=np.uint32)


def model_merge(keys, desc, offsets):
    """TSortedMergingReader: a heap of streams ordered by (key of the head row, stream index)."""
    K = functools.cmp_to_key(lambda i, j: compare_rows(keys[i], keys[j], desc))
    h = [(K(int(offsets[r])), r, int(offsets[r])) for r in range(len(offsets) - 1) if offsets[r] < offsets[r + 1]]
    heapq.heapify(h)
    out = []
    while h:
        _, r, pos = heapq.heappop(h)
        out.append(pos)
        if pos + 1 < offsets[r + 1]:
            heapq.heappush(h, (K(pos + 1), r, pos + 1))
    return np.array(out, dtype=np.uint32)


def _canon(key):
    """A hashable form in which values that compare equal coincide (NaN == NaN, -0.0 == +0.0)."""
    return tuple((t, ("nan" if v != v else v + 0.0) if t == T.Double else v) for t, v in key)


def model_join(keys, desc, jc, offsets):
    """TSortedJoiningReader with stream r carrying table index r: every primary row (stream 0), and the foreign rows
    whose join key (the first jc key columns) occurs in the primary stream, in (join key, stream, position) order."""
    primary = {_canon(keys[i][:jc]) for i in range(offsets[0], offsets[1])}
    rows = [i for i in range(len(keys)) if i < offsets[1] or _canon(keys[i][:jc]) in primary]
    return np.array(sorted(rows, key=functools.cmp_to_key(lambda i, j: compare_rows(keys[i][:jc], keys[j][:jc], desc[:jc]))),
                    dtype=np.uint32)


def model_partition(keys, desc, bounds, plen, incl):
    """TOrderedPartitioner: std::upper_bound over the lower bounds with !TestKey, minus one."""
    out = np.empty(len(keys), dtype=np.int32)
    for r, key in enumerate(keys):
        lo, cnt = 0, len(bounds)
        while cnt > 0:
            step = cnt // 2
            mid = lo + step
            c = compare_rows(key[:plen[mid]], bounds[mid][:plen[mid]], desc)
            if c > 0 or (c == 0 and incl[mid]):
                lo, cnt = mid + 1, cnt - step - 1
            else:
                cnt = step
        out[r] = lo - 1
    return out


def bound_order(a, b, desc):
    """Order of two lower bounds (prefix, inclusive): a prefix stands before every key it starts when inclusive and
    after them when exclusive."""
    (ka, ia), (kb, ib) = a, b
    m = min(len(ka), len(kb))
    c = compare_rows(ka[:m], kb[:m], desc)
    if c:
        return c
    if len(ka) == len(kb):
        return (not ia) - (not ib)
    if len(ka) < len(kb):
        return -1 if ia else 1
    return 1 if ib else -1


# ------------------------------------------------------------------------------------------------- value generators
# A generator returns (type u8[n], length u32[n], data u64[n], heap bytes); a string's data is an offset into the heap.
SPECIAL_I64 = np.array([I64_MIN, I64_MIN + 1, -256, -1, 0, 1, 255, 256, I64_MAX - 1, I64_MAX], dtype=np.int64)
SPECIAL_U64 = np.array([0, 1, 255, 256, 2**63 - 1, 2**63, U64_MAX - 1, U64_MAX], dtype=np.uint64)
SPECIAL_DOUBLE_BITS = np.array([
    0x0000000000000000, 0x8000000000000000,  # +0.0, -0.0
    0x7FF0000000000000, 0xFFF0000000000000,  # +inf, -inf
    0x7FF8000000000000, 0x7FF0000000000001,  # canonical quiet NaN, signalling NaN
    0xFFF8000000000000, 0x7FFFFFFFFFFFFFFF, 0xFFF0000000000123,  # negative NaN, all-ones payload, negative payload
    0x0000000000000001, 0x8000000000000001,  # +-denormal min
    0x3FF0000000000000, 0xBFF0000000000000, 0x4004000000000000,  # 1.0, -1.0, 2.5
], dtype=np.uint64)


def _typed(t, data, n):
    return np.full(n, t, np.uint8), np.zeros(n, np.uint32), np.asarray(data, dtype=np.uint64), b""


def _with_nulls(rng, col, rate):
    types, lengths, data, heap = col
    m = rng.random(len(types)) < rate
    types, lengths, data = types.copy(), lengths.copy(), data.copy()
    types[m], lengths[m], data[m] = T.Null, 0, 0
    return types, lengths, data, heap


def _skew(rng, col, rate, value):
    """Most rows take one value, so that rows tie on this column and later key columns decide."""
    types, lengths, data, heap = col
    m = rng.random(len(types)) < rate
    data = data.copy()
    data[m] = value
    return types, lengths, data, heap


def gen_int64(rng, n, nulls=0.0, skew=0.0):
    v = rng.integers(I64_MIN, I64_MAX, n, dtype=np.int64, endpoint=True)
    cat = rng.random(n)
    small = cat < 0.45
    v[small] = rng.integers(-3, 4, int(small.sum()))
    special = (cat >= 0.45) & (cat < 0.6)
    v[special] = SPECIAL_I64[rng.integers(0, len(SPECIAL_I64), int(special.sum()))]
    col = _skew(rng, _typed(T.Int64, v.view(np.uint64), n), skew, 0)
    return _with_nulls(rng, col, nulls)


def gen_uint64(rng, n, nulls=0.0):
    v = rng.integers(0, U64_MAX, n, dtype=np.uint64, endpoint=True)
    cat = rng.random(n)
    small = cat < 0.45
    v[small] = rng.integers(0, 4, int(small.sum())).astype(np.uint64)
    special = (cat >= 0.45) & (cat < 0.6)
    v[special] = SPECIAL_U64[rng.integers(0, len(SPECIAL_U64), int(special.sum()))]
    return _with_nulls(rng, _typed(T.Uint64, v, n), nulls)


def gen_double(rng, n, nulls=0.0):
    v = rng.normal(size=n).view(np.uint64)
    special = rng.random(n) < 0.5
    v[special] = SPECIAL_DOUBLE_BITS[rng.integers(0, len(SPECIAL_DOUBLE_BITS), int(special.sum()))]
    return _with_nulls(rng, _typed(T.Double, v, n), nulls)


def gen_bool(rng, n, nulls=0.0, skew=0.0):
    v = np.array([0, 1, 0x101], dtype=np.uint64)[rng.integers(0, 3, n)]  # any non-zero low byte is true
    return _with_nulls(rng, _skew(rng, _typed(T.Boolean, v, n), skew, 1), nulls)


def _pool_strings(rng, n, pool, nulls=0.0, force=None):
    heap = b"".join(pool)
    lens = np.array([len(s) for s in pool], dtype=np.uint32)
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).astype(np.uint64)
    idx = rng.integers(0, len(pool), n)
    types = np.where(rng.random(n) < nulls, T.Null, T.String).astype(np.uint8)
    if force is not None and n:
        r = rng.integers(0, n)  # the widest string is present whatever was drawn
        idx[r], types[r] = force, T.String
    is_str = types == T.String
    return types, np.where(is_str, lens[idx], 0).astype(np.uint32), np.where(is_str, offs[idx], 0).astype(np.uint64), heap


def _short_pool():
    rng = np.random.default_rng(1234)
    pool = [b"", b"\x00", b"\x00\x00", b"\xff", b"\xff\xff", b"a", b"ab", b"ab\x00", b"ab\x00\x00", b"ab\xff", b"abc",
            b"b", b"\x00a", b"a\x00b", b"\xff\x00", b"ab\x00\xff"]
    alphabet = np.frombuffer(b"\x00ab\xff", dtype=np.uint8)
    pool += [bytes(rng.choice(alphabet, int(rng.integers(0, 13)))) for _ in range(150)]
    pool.append(b"ab\x00\x00\x00\x00\x00\x00\x00\x00\x00\xff")  # 12 bytes: the widest
    return pool


SHORT_POOL = _short_pool()


def gen_string(rng, n, nulls=0.0):
    return _pool_strings(rng, n, SHORT_POOL, nulls, force=len(SHORT_POOL) - 1)


def edge_pool(width, seed=77):
    """Strings of at most `width` bytes around one `width`-byte string: its prefixes, the prefixes followed by 0x00 or
    0xff, and strings that differ from it only in the last bytes."""
    rng = np.random.default_rng(seed + width)
    alphabet = np.frombuffer(b"\x00ab\xff", dtype=np.uint8)
    base = bytes(rng.choice(alphabet, width))
    pool = [base]
    for k in sorted(set(rng.integers(0, width + 1, 40).tolist()) | {0, width - 1}):
        pool += [base[:k], (base[:k] + b"\x00")[:width], (base[:k] + b"\xff")[:width]]
    for k in (1, 2, 3):
        pool.append(base[:-k] + bytes(rng.choice(alphabet, k)))
    pool += [bytes(rng.choice(alphabet, int(rng.integers(0, width + 1)))) for _ in range(20)]
    assert max(len(s) for s in pool) == width
    return pool


def gen_edge_string(width):
    pool = edge_pool(width)
    return lambda rng, n, nulls=0.0: _pool_strings(rng, n, pool, nulls, force=0)


def gen_any(rng, n):
    """One any-scalar column mixing every kind: Null, Int64, Uint64, Double, Boolean, String, Min and Max."""
    parts = [gen_int64(rng, n), gen_uint64(rng, n), gen_double(rng, n), gen_bool(rng, n), gen_string(rng, n),
             _typed(T.Null, np.zeros(n), n), _typed(T.Min, np.zeros(n), n), _typed(T.Max, np.zeros(n), n)]
    kind = rng.choice(len(parts), n, p=[0.2, 0.15, 0.15, 0.1, 0.25, 0.05, 0.05, 0.05])
    types = np.zeros(n, np.uint8)
    lengths = np.zeros(n, np.uint32)
    data = np.zeros(n, np.uint64)
    for k, (t, ln, d, _) in enumerate(parts):
        m = kind == k
        types[m], lengths[m], data[m] = t[m], ln[m], d[m]
    return types, lengths, data, parts[4][3]


def gen_all_null(rng, n):
    return _typed(T.Null, np.zeros(n), n)


def gen_all_empty(rng, n):
    return np.full(n, T.String, np.uint8), np.zeros(n, np.uint32), np.zeros(n, np.uint64), b""


def build_rowset(value_count, columns, n):
    """columns: {value index: column}; the other values hold the row number (Int64), so a gathered row shows where it
    came from."""
    vals = np.zeros((n, value_count), dtype=VALUE_DTYPE)
    vals["id"] = np.arange(value_count, dtype=np.uint16)
    vals["type"] = T.Int64
    vals["data"] = np.arange(n, dtype=np.uint64)[:, None]
    heap = bytearray()
    for j, (types, lengths, data, h) in columns.items():
        data = data.copy()
        data[types == T.String] += np.uint64(len(heap))
        heap += h
        vals["type"][:, j], vals["length"][:, j], vals["data"][:, j] = types, lengths, data
    return Rowset(vals, np.frombuffer(bytes(heap) or b"\0", dtype=np.uint8).copy())


# ------------------------------------------------------------------------------------------------------------ layouts
def K(index, gen, type=0, required=0, desc=0, width=0):
    return dict(index=index, gen=gen, type=type, required=required, descending=desc, width=width)


def _n(gen, **kw):
    return lambda rng, n: gen(rng, n, **kw)


_SPREAD = [39, 0, 20, 7, 33, 12, 26, 3, 17, 30, 9, 36, 22, 5, 14, 28, 1, 38, 11, 24, 31, 6, 18, 35, 2, 27, 15, 34, 8,
           21, 37, 13]

# Each entry: the code path it reaches, the number of values per row, the key columns, and whether the key is past the
# 256-byte limit of the normalised form (the refinement sort of long_keys.cu and the key-word partitioner).
LAYOUTS = {
    "int64_nullable": dict(
        path="type byte + 8 bytes: 2 chunks", value_count=2, long=False,
        keys=[K(0, _n(gen_int64, nulls=0.1), T.Int64)]),
    "int64_uint64_required": dict(
        path="16 bytes without type bytes: 2 chunks", value_count=3, long=False,
        keys=[K(2, gen_int64, T.Int64, required=1), K(0, gen_uint64, T.Uint64, required=1)]),
    "any_scalar": dict(
        path="type=0: type byte + measured string width + length, every kind in one column", value_count=2, long=False,
        keys=[K(0, gen_any)]),
    "string_required_measured": dict(
        path="required string, width measured on the device (12 + 1 bytes)", value_count=2, long=False,
        keys=[K(1, gen_string, T.String, required=1)]),
    "string_declared_wide": dict(
        path="declared width 40 wider than every value (1 + 40 + 1 bytes)", value_count=2, long=False,
        keys=[K(0, _n(gen_string, nulls=0.1), T.String, width=40)]),
    "empty_strings": dict(
        path="all-NULL and all-empty string columns: measured width 0", value_count=3, long=False,
        keys=[K(2, gen_all_null, T.String), K(0, gen_all_empty, T.String, required=1), K(1, _n(gen_int64, nulls=0.2), T.Int64)]),
    "eight_alternating": dict(
        path="8 columns of every type, alternating ascending / descending", value_count=10, long=False,
        keys=[K(9, _n(gen_bool, nulls=0.2), T.Boolean), K(0, _n(gen_string, nulls=0.1), T.String, desc=1),
              K(3, _n(gen_int64, nulls=0.1, skew=0.5), T.Int64), K(5, _n(gen_double, nulls=0.1), T.Double, desc=1),
              K(1, gen_uint64, T.Uint64, required=1), K(7, gen_any, desc=1),
              K(2, gen_int64, T.Int64, required=1), K(8, gen_string, T.String, required=1, desc=1)]),
    "thirty_two_columns": dict(
        path="32 key columns (the maximum) spread over a 40-value row: 160 bytes, 20 chunks", value_count=40, long=False,
        keys=[K(ix, _n(gen_bool, nulls=0.02, skew=0.9), T.Boolean, desc=(j // 2) % 2) if j % 2 == 0 else
              K(ix, _n(gen_int64, skew=0.9), T.Int64, required=1, desc=(j // 2) % 2) for j, ix in enumerate(_SPREAD)]),
    "int64x28": dict(
        path="28 nullable int64: 252 bytes, 32 chunks, still normalised", value_count=28, long=False,
        keys=[K(j, _n(gen_int64, nulls=0.03, skew=0.9), T.Int64, desc=j % 3 == 2) for j in range(28)]),
    "int64x29": dict(
        path="29 nullable int64: 261 bytes, the long-key path", value_count=29, long=True,
        keys=[K(j, _n(gen_int64, nulls=0.03, skew=0.9), T.Int64, desc=j % 3 == 2) for j in range(29)]),
    "string_254": dict(
        path="nullable string of at most 254 bytes: 1 + 254 + 1 = 256 bytes, the last normalised width", value_count=2,
        long=False, keys=[K(0, _n(gen_edge_string(254), nulls=0.05), T.String)]),
    "string_255": dict(
        path="nullable string of at most 255 bytes: 1 + 255 + 2 bytes, the long-key path", value_count=2, long=True,
        keys=[K(0, _n(gen_edge_string(255), nulls=0.05), T.String)]),
}


def make_layout(name, n, seed=0, flip=0):
    """-> (rowset, key columns for the C ABI, key value indices, per-column descending flags)."""
    lay = LAYOUTS[name]
    rng = np.random.default_rng(seed * 1000 + sorted(LAYOUTS).index(name))
    rs = build_rowset(lay["value_count"], {k["index"]: k["gen"](rng, n) for k in lay["keys"]}, n)
    cols = [dict(index=k["index"], type=k["type"], required=k["required"], width=k["width"],
                 descending=int(bool(k["descending"])) ^ flip) for k in lay["keys"]]
    return rs, cols, [c["index"] for c in cols], [c["descending"] for c in cols]


def key_first(rs, key_idx):
    """The oracle compares the first nkey values of a row: the key columns moved to the front."""
    return np.ascontiguousarray(rs.values[:, key_idx])


def ref_sort(rs, key_idx, desc):
    if rs.row_count <= MODEL_ROWS:
        return model_sort(decode(rs.values, rs.heap, key_idx), desc)
    return oracle.sort_rows(key_first(rs, key_idx), rs.heap, len(key_idx), desc, oracle.SORT_STABLE)[0]


def key_bytes(cols, rs):
    """Byte offsets of the key columns in the normalised key and its total width (keys.cuh build_key_layout), string
    widths measured as resolve_widths does."""
    offs, off = [], 0
    for c in cols:
        t, w = c.get("type", 0), c.get("width", 0)
        col = rs.values[:, c["index"]]
        if t in (0, T.String) and w == 0:
            w = int(col["length"][col["type"] == T.String].max(initial=0))
        p = 0
        if t in (0, T.String):
            p = w + (1 if w < 255 else 2 if w < 65535 else 4)
        if t in (0, T.Int64, T.Uint64, T.Double):
            p = max(p, 8)
        if t == T.Boolean:
            p = 1
        offs.append(off)
        off += (0 if c.get("required") and t != 0 else 1) + p
    return offs, off


def sorted_runs(rs, key_idx, desc, k, rng, empty=()):
    """Splits the rows into k runs (the runs in `empty` get no rows), each sorted: -> (rowset of the concatenated runs,
    run offsets).  Keys repeat across runs."""
    n = rs.row_count
    live = [r for r in range(k) if r not in empty]
    run_of = np.array(live)[rng.integers(0, len(live), n)] if live else np.zeros(n, np.int64)
    order = ref_sort(rs, key_idx, desc).astype(np.int64)
    parts = [order[run_of[order] == r] for r in range(k)]
    offsets = np.cumsum([0] + [len(p) for p in parts]).astype(np.uint64)
    return rs.take(np.concatenate(parts)), offsets


# ---------------------------------------------------------------------------------------------------------- bounds
def _raw_value(t, payload):
    """A model (type, payload) pair back to (type, length, data, string bytes)."""
    if t == T.String:
        return t, len(payload), 0, payload
    if t == T.Double:
        return t, 0, struct.unpack("<Q", struct.pack("<d", payload))[0], b""
    if t in (T.Int64, T.Uint64, T.Boolean):
        return t, 0, int(payload) & U64_MAX, b""
    return t, 0, 0, b""


def bounds_rowset(bounds, ncols):
    """bounds: list of key prefixes (tuples of raw values) -> Rowset of ncols values per bound (Null past the prefix)."""
    vals = np.zeros((max(len(bounds), 1), ncols), dtype=VALUE_DTYPE)
    vals["type"] = T.Null
    heap = bytearray()
    for b, prefix in enumerate(bounds):
        for c, (t, length, data, s) in enumerate(prefix):
            if t == T.String:
                data = len(heap)
                heap += s
            vals[b, c] = (c, t, 0, length, data)
    return Rowset(vals, np.frombuffer(bytes(heap) or b"\0", dtype=np.uint8).copy())


def raw_keys(rs, key_idx):
    """Key values of every row as tuples of raw (type, length, data, string bytes)."""
    hb = rs.heap.tobytes()
    return [tuple((t, ln, d, hb[d:d + ln] if t == T.String else b"") for _, t, _, ln, d in row)
            for row in rs.values[:, key_idx].tolist()]


def handmade_bounds(rs, cols, rng, count=12):
    """Lower bounds at the rules of the bound encoder: prefix lengths 0..ncols, inclusive and exclusive, bounds equal to
    keys, Min / Max, a required column's bound of another type, and bound strings longer than the measured width W whose
    tail holds 0x00 or 0xff.  -> list of (raw prefix, inclusive)."""
    rows = raw_keys(rs, [c["index"] for c in cols])
    ncols = len(cols)
    sentinel = lambda t: (t, 0, 0, b"")  # noqa: E731
    out = []
    for r in rng.integers(0, len(rows), count):
        key = rows[r]
        for plen in range(ncols + 1):
            out.append((key[:plen], bool(rng.integers(0, 2))))
        j = int(rng.integers(0, ncols))
        for t in (T.Min, T.Max):
            out.append((key[:j] + (sentinel(t),), bool(rng.integers(0, 2))))
        for j, c in enumerate(cols):
            if c["required"] and c["type"] != 0:
                for other in (T.Null, T.Int64, T.Uint64, T.Double, T.String):
                    if other != c["type"]:
                        v = (other, 1, 0, b"a") if other == T.String else (other, 0, 1, b"")
                        out.append((key[:j] + (v,), bool(rng.integers(0, 2))))
            if c["type"] in (0, T.String):
                col = rs.values[:, c["index"]]
                w = c["width"] or int(col["length"][col["type"] == T.String].max(initial=0))
                s = key[j][3] if key[j][0] == T.String else b"a"
                pad = w - len(s) if len(s) < w else 0
                for tail in (b"\x00" * (pad + 1), b"\x00" * pad + b"\xff", b"\xff" * (pad + 2), b"\x00" * (pad + 3)):
                    out.append((key[:j] + ((T.String, len(s + tail), 0, s + tail),), bool(rng.integers(0, 2))))
    return out


def sample_bounds(rs, cols, rng, count):
    rows = raw_keys(rs, [c["index"] for c in cols])
    return [(rows[r][:int(rng.integers(1, len(cols) + 1))], bool(rng.integers(0, 2)))
            for r in rng.integers(0, len(rows), count)]


def order_bounds(bounds, desc):
    """Sorts lower bounds into partition order and puts the universal bound first."""
    model = [(tuple((t, _decode_raw(t, ln, d, s)) for t, ln, d, s in p), i) for p, i in bounds]
    order = sorted(range(len(bounds)), key=functools.cmp_to_key(lambda a, b: bound_order(model[a], model[b], desc)))
    return [((), True)] + [bounds[i] for i in order]


def _decode_raw(t, length, data, s):
    if t == T.Int64:
        return data - (1 << 64) if data >> 63 else data
    if t == T.Uint64:
        return data
    if t == T.Double:
        return _as_double(data)
    if t == T.Boolean:
        return (data & 0xFF) != 0
    if t == T.String:
        return s
    return None


def partition_case(rs, cols, bounds):
    """-> (bounds rowset, prefix lengths, inclusive flags, model bounds)."""
    brs = bounds_rowset([p for p, _ in bounds], len(cols))
    plen = [len(p) for p, _ in bounds]
    incl = [int(i) for _, i in bounds]
    model = [tuple((t, _decode_raw(t, ln, d, s)) for t, ln, d, s in p) for p, _ in bounds]
    return brs, plen, incl, model


# ------------------------------------------------------------------------------------------- CPU: model vs oracle
@pytest.mark.parametrize("flip", [0, 1])
@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_model_matches_oracle(name, flip):
    """The Python model agrees with the oracle on every layout: sort, merge, join and ordered partitioning."""
    rng = np.random.default_rng(5 + flip)
    rs, cols, key_idx, desc = make_layout(name, 2500, seed=1, flip=flip)
    kf = key_first(rs, key_idx)
    keys = decode(rs.values, rs.heap, key_idx)
    want = oracle.sort_rows(kf, rs.heap, len(cols), desc, oracle.SORT_STABLE)[0]
    assert (model_sort(keys, desc) == want).all()

    runs, off = sorted_runs(rs, key_idx, desc, 6, rng, empty=(2,))
    rkeys = decode(runs.values, runs.heap, key_idx)
    assert (model_merge(rkeys, desc, off) == oracle.merge_sorted(key_first(runs, key_idx), runs.heap, len(cols), desc, off)).all()
    for jc in sorted({1, len(cols)}):
        want = oracle.join_sorted(key_first(runs, key_idx), runs.heap, jc, desc[:jc], off, list(range(len(off) - 1)))
        assert model_join(rkeys, desc, jc, [int(x) for x in off]).tolist() == want.tolist(), jc

    bounds = order_bounds(handmade_bounds(rs, cols, rng, count=4) + sample_bounds(rs, cols, rng, 40), desc)
    brs, plen, incl, model = partition_case(rs, cols, bounds)
    want, _ = oracle.partition_ordered(kf, rs.heap, len(cols), desc, brs.values, brs.heap, plen, incl)
    assert (model_partition(keys, desc, model, plen, incl) == want).all()


def test_model_value_rules():
    """The rules the model restates, on hand-picked pairs."""
    nan2 = _as_double(0x7FF0000000000001)
    pairs = [((T.Int64, -1), (T.Int64, 0), -1), ((T.Uint64, 2**63), (T.Uint64, 1), 1), ((T.Int64, 5), (T.Uint64, 0), -1),
             ((T.Double, -0.0), (T.Double, 0.0), 0), ((T.Double, float("nan")), (T.Double, nan2), 0),
             ((T.Double, float("inf")), (T.Double, nan2), -1), ((T.Boolean, False), (T.Boolean, True), -1),
             ((T.String, b"ab"), (T.String, b"ab\x00"), -1), ((T.String, b"ab\xff"), (T.String, b"b"), -1),
             ((T.Min, None), (T.Null, None), -1), ((T.Max, None), (T.String, b"\xff"), 1), ((T.Null, None), (T.Null, None), 0)]
    for a, b, want in pairs:
        assert compare_values(a, b) == want and compare_values(b, a) == -want, (a, b)
    assert compare_rows([(T.Int64, 1), (T.Int64, 2)], [(T.Int64, 1), (T.Int64, 3)], [0, 1]) == 1
    assert model_sort([((T.Int64, 1),), ((T.Int64, 0),), ((T.Int64, 1),)], [0]).tolist() == [1, 0, 2]


def test_layouts_reach_the_paths_they_name():
    """The normalised widths the layout table promises, computed as build_key_layout does."""
    widths = {}
    for name in LAYOUTS:
        rs, cols, _, _ = make_layout(name, 3000)
        widths[name] = key_bytes(cols, rs)[1]
        assert (widths[name] > 256) == LAYOUTS[name]["long"], name
    assert widths["int64_nullable"] == 9 and widths["int64_uint64_required"] == 16
    assert widths["thirty_two_columns"] == 160 and len(LAYOUTS["thirty_two_columns"]["keys"]) == 32
    assert widths["int64x28"] == 252 and widths["int64x29"] == 261
    assert widths["string_254"] == 256 and widths["string_255"] == 258
    assert widths["empty_strings"] == 1 + 1 + 1 + 9 and widths["string_declared_wide"] == 42
    idx = LAYOUTS["thirty_two_columns"]["keys"]
    assert len({k["index"] for k in idx}) == 32 and max(k["index"] for k in idx) == 39


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def ctx():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from ytsaurus_b200 import GpuContext
    c = GpuContext(0)
    yield c
    c.close()


def _dev(rs):
    import torch
    return (torch.from_numpy(rs.values.view(np.uint8).reshape(rs.row_count, -1).copy()).cuda(),
            torch.from_numpy(rs.heap.copy()).cuda())


def _host(t, dtype=np.uint32):
    return t.cpu().numpy().view(dtype)


def _values(t, shape):
    return t.cpu().numpy().reshape(-1).view(VALUE_DTYPE).reshape(shape)


def gpu_sort(ctx, rs, cols, device):
    """-> (permutation, gathered values) from one flavour."""
    v, h = _dev(rs) if device else (rs.values, rs.heap)
    perm, vals = ctx.sort_rowset(v, h, cols, want_values=True)
    if device:
        perm, vals = _host(perm), _values(vals, rs.values.shape)
    return perm, vals


def check_path(ctx, long):
    rounds = ctx.get_option("last_sort_refine_rounds")
    assert (rounds >= 1) if long else (rounds == 0), rounds


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 3001])
@pytest.mark.parametrize("flip", [0, 1])
@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_sort_layout(ctx, name, flip, n):
    rs, cols, key_idx, desc = make_layout(name, n, seed=2, flip=flip)
    want = ref_sort(rs, key_idx, desc)
    for device in (False, True):
        perm, vals = gpu_sort(ctx, rs, cols, device)
        assert (perm == want).all(), device
        assert vals.tobytes() == rs.values[want.astype(np.int64)].tobytes(), device
        check_path(ctx, LAYOUTS[name]["long"])


def _prefix_shape(shape, n, rng):
    """Two required uint64 key columns (a, b) shaped so that the multi-chunk sort takes one outcome:
    complete: 8 active bytes in all (4 of a, 4 of b): the prefix chunk is the whole key;
    tie32 / tie33: a unique per row except groups of exactly 32 (33) rows that share a and differ in b: deep_tie_fix_kernel
      insertion-sorts the 32-row runs; a 33-row run that mixes keys sends the sort to the complete schedule;
    equal_runs: few distinct (a, b) pairs: long runs of fully equal keys, which need no fallback and keep input order."""
    a = rng.integers(0, U64_MAX, n, dtype=np.uint64, endpoint=True)
    b = rng.integers(0, U64_MAX, n, dtype=np.uint64, endpoint=True)
    if shape == "complete":
        a &= np.uint64(0xFFFFFFFF)
        b &= np.uint64(0xFFFFFFFF)
    elif shape in ("tie32", "tie33"):
        size = 32 if shape == "tie32" else 33
        groups = min(50, n // (2 * size))
        pos = rng.permutation(n)[:groups * size].reshape(groups, size)
        for g in range(groups):
            a[pos[g]] = a[pos[g][0]]
    elif shape == "equal_runs":
        pool = rng.integers(0, 100, n)
        a = rng.integers(0, U64_MAX, 100, dtype=np.uint64, endpoint=True)[pool]
        b = rng.integers(0, U64_MAX, 100, dtype=np.uint64, endpoint=True)[pool]
    cols = {0: _typed(T.Uint64, a, n), 2: _typed(T.Uint64, b, n)}
    return build_rowset(3, cols, n), [dict(index=0, type=T.Uint64, required=1), dict(index=2, type=T.Uint64, required=1)]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["complete", "tie32", "tie33", "equal_runs"])
@pytest.mark.parametrize("n", [1, 2, 2047, 2048, 2049, HYBRID_MIN_ROWS - 1, HYBRID_MIN_ROWS, 300_001])
def test_multi_chunk_sort_outcomes(ctx, shape, n):
    """The prefix path of radix_sort_keys runs one single-chunk sort of the prefix chunk: at most 8 digit passes.  The
    complete-schedule fallback sorts every active byte of the key, more than 8 (it only runs when the key has more
    than 8 active bytes).  So last_sort_passes() tells the two apart."""
    rng = np.random.default_rng(n * 7 + len(shape))
    rs, cols = _prefix_shape(shape, n, rng)
    want = ref_sort(rs, [0, 2], [0, 0])
    fallback = shape == "tie33" and n >= 66
    for hybrid in (1, 0):
        ctx.set_option("sort_hybrid", hybrid)
        try:
            for device in (False, True):
                perm, vals = gpu_sort(ctx, rs, cols, device)
                passes = ctx.last_sort_passes()
                assert (perm == want).all(), (hybrid, device)
                assert vals.tobytes() == rs.values[want.astype(np.int64)].tobytes()
                assert (passes > 8) if fallback else (passes <= 8), (passes, hybrid, device)
        finally:
            ctx.set_option("sort_hybrid", 1)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ["tie32", "tie33"])
def test_multi_chunk_sort_near_a_million_rows(ctx, shape):
    rng = np.random.default_rng(99 + len(shape))
    n = 1_000_003
    rs, cols = _prefix_shape(shape, n, rng)
    want = ref_sort(rs, [0, 2], [0, 0])
    perm, vals = gpu_sort(ctx, rs, cols, device=True)
    assert (perm == want).all()
    assert vals.tobytes() == rs.values[want.astype(np.int64)].tobytes()
    assert (ctx.last_sort_passes() > 8) if shape == "tie33" else (ctx.last_sort_passes() <= 8)


@pytest.mark.gpu
@pytest.mark.parametrize("name,n", [("thirty_two_columns", 300_001), ("int64x28", HYBRID_MIN_ROWS), ("string_254", HYBRID_MIN_ROWS),
                                    ("eight_alternating", HYBRID_MIN_ROWS + 1), ("any_scalar", 300_001)])
def test_sort_layout_at_scale(ctx, name, n):
    """Multi-chunk layouts past kHybridMinRows: the prefix chunk takes the hybrid schedule."""
    rs, cols, key_idx, desc = make_layout(name, n, seed=3)
    want = ref_sort(rs, key_idx, desc)
    perm, vals = gpu_sort(ctx, rs, cols, device=True)
    assert (perm == want).all()
    assert vals.tobytes() == rs.values[want.astype(np.int64)].tobytes()
    check_path(ctx, LAYOUTS[name]["long"])
    ctx.set_option("sort_hybrid", 0)
    try:
        assert (ctx.sort_rowset(rs.values, rs.heap, cols) == want).all()
    finally:
        ctx.set_option("sort_hybrid", 1)


def _merge(ctx, runs, cols, off, device):
    v, h = _dev(runs) if device else (runs.values, runs.heap)
    got = ctx.merge_sorted_runs(v, h, cols, off)
    return _host(got) if device else got


@pytest.mark.gpu
@pytest.mark.parametrize("k,empty", [(1, ()), (2, ()), (15, (3,)), (16, ()), (17, ()), (20, (0, 5, 6, 19))])
@pytest.mark.parametrize("name", ["int64_nullable", "eight_alternating", "thirty_two_columns", "int64x28", "string_254",
                                  "string_255", "any_scalar"])
def test_merge_sorted_runs(ctx, name, k, empty):
    """Equal keys across runs: the lower run wins.  Up to 16 non-empty runs of multi-chunk keys take the merge path."""
    rng = np.random.default_rng(k * 31 + len(name))
    rs, cols, key_idx, desc = make_layout(name, 6000, seed=4)
    runs, off = sorted_runs(rs, key_idx, desc, k, rng, empty=empty)
    want = model_merge(decode(runs.values, runs.heap, key_idx), desc, off)
    live = int((np.diff(off) > 0).sum())
    for device in (False, True):
        assert (_merge(ctx, runs, cols, off, device) == want).all(), device
        assert ctx.get_option("last_merge_used_merge_path") == int(live <= 16 and not LAYOUTS[name]["long"])
        check_path(ctx, LAYOUTS[name]["long"])
    ctx.set_option("merge_path", 0)
    try:
        assert (_merge(ctx, runs, cols, off, False) == want).all()
        assert ctx.get_option("last_merge_used_merge_path") == 0
    finally:
        ctx.set_option("merge_path", 1)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [2, 16, 17])
def test_merge_sorted_runs_near_a_million_rows(ctx, k):
    """32-chunk keys (the 256-byte string layout) at about 10^6 rows."""
    rng = np.random.default_rng(k)
    rs, cols, key_idx, desc = make_layout("string_254", 1_000_003, seed=5)
    runs, off = sorted_runs(rs, key_idx, desc, k, rng)
    want = oracle.merge_sorted(key_first(runs, key_idx), runs.heap, len(cols), desc, off)
    assert (_merge(ctx, runs, cols, off, True) == want).all()
    assert ctx.get_option("last_merge_used_merge_path") == int(k <= 16)


def _few_doubles(rng, n, nulls):
    """Doubles from a small set, so that join keys repeat: +-0.0, +-inf and NaN payloads."""
    pool = SPECIAL_DOUBLE_BITS[:9]
    return _with_nulls(rng, _typed(T.Double, pool[rng.integers(0, len(pool), n)], n), nulls)


def join_case(n, ncols, tag, string_width=0, seed=0):
    """Streams 0 (primary) .. 3, each sorted, over ncols join columns of 9 bytes each (nullable double / int64 from
    small sets: NULL, NaN payloads and +-0.0 join), or one nullable string column when string_width is given.  The key
    is the join columns, then, with `tag`, the stream index as a required int64: rows of one join key stay in stream
    order, as the joining reader emits them.
    -> (rowset of the concatenated streams, key columns, join value indices, run offsets)."""
    rng = np.random.default_rng(seed)
    if string_width:
        gens = {0: gen_edge_string(string_width)(rng, n, 0.05)}
        cols = [dict(index=0, type=T.String)]
    else:
        gens = {}
        cols = []
        for j in range(ncols):
            if j % 2 == 0:
                gens[j] = _few_doubles(rng, n, 0.1)
                cols.append(dict(index=j, type=T.Double))
            else:
                gens[j] = _with_nulls(rng, _typed(T.Int64, rng.integers(-2, 3, n).astype(np.int64).view(np.uint64), n), 0.1)
                cols.append(dict(index=j, type=T.Int64))
    vc = max(gens) + 2
    rs = build_rowset(vc, gens, n)
    key_idx = [c["index"] for c in cols]
    runs, off = sorted_runs(rs, key_idx, [0] * len(cols), 4, rng)
    runs.values["type"][:, vc - 1] = T.Int64
    runs.values["data"][:, vc - 1] = np.repeat(np.arange(4, dtype=np.uint64), np.diff(off).astype(np.int64))
    spec = cols + ([dict(index=vc - 1, type=T.Int64, required=1)] if tag else [])
    return runs, spec, key_idx, off


JOIN_CASES = {
    # name: (join columns, tag column): where the join prefix ends
    "mid_chunk": (1, True),            # 9 bytes: inside chunk 1
    "mid_chunk_7": (7, True),          # 63 bytes: inside chunk 7
    "chunk_boundary": (8, True),       # 72 bytes: the end of chunk 8, no partial chunk
    "whole_key": (3, False),           # the whole 27-byte key
    "whole_key_boundary": (8, False),  # the whole 72-byte key
}


def _join_check(ctx, runs, spec, key_idx, off, jc, device=False, long=False):
    tables = list(range(len(off) - 1))
    if runs.row_count <= MODEL_ROWS:
        want = model_join(decode(runs.values, runs.heap, key_idx), [0] * len(key_idx), jc, [int(x) for x in off])
    else:
        want = oracle.join_sorted(key_first(runs, key_idx), runs.heap, jc, None, off, tables)
    v, h = _dev(runs) if device else (runs.values, runs.heap)
    got = ctx.join_sorted_runs(v, h, spec, jc, off)
    if device:
        got = _host(got)
    assert got.tolist() == want.tolist()
    check_path(ctx, long)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [3000, HYBRID_MIN_ROWS + 7])
@pytest.mark.parametrize("case", sorted(JOIN_CASES))
def test_join_prefix_ends(ctx, case, n):
    jc, tag = JOIN_CASES[case]
    runs, spec, key_idx, off = join_case(n, jc, tag, seed=jc * 2 + tag)
    offs, total = key_bytes(spec, runs)
    prefix = offs[jc] if jc < len(spec) else total
    assert (prefix % 8 == 0) == ("boundary" in case) and (jc == len(spec)) == ("whole" in case)
    for device in (False, True):
        _join_check(ctx, runs, spec, key_idx, off, jc, device)


@pytest.mark.gpu
@pytest.mark.parametrize("width,tag,long", [(254, False, False), (255, False, True), (246, True, False), (247, True, True)])
def test_join_at_the_256_byte_edge(ctx, width, tag, long):
    runs, spec, key_idx, off = join_case(4000, 1, tag, string_width=width, seed=width)
    assert (key_bytes(spec, runs)[1] > 256) == long
    _join_check(ctx, runs, spec, key_idx, off, 1, long=long)


def _ordered_spec(ctx, cols, brs, plen, incl):
    return ctx._partition_spec(capi.PARTITION_ORDERED, len(plen), key_columns=cols, bounds=brs, bound_prefix_length=plen,
                               bound_inclusive=incl)


def _partition_check(ctx, rs, cols, bounds, name, use_model, slabs=False):
    key_idx = [c["index"] for c in cols]
    desc = [c["descending"] for c in cols]
    brs, plen, incl, model = partition_case(rs, cols, bounds)
    if use_model:
        want = model_partition(decode(rs.values, rs.heap, key_idx), desc, model, plen, incl)
    else:
        want, _ = oracle.partition_ordered(key_first(rs, key_idx), rs.heap, len(cols), desc, brs.values, brs.heap, plen, incl)
    spec = _ordered_spec(ctx, cols, brs, plen, incl)
    idx, hist = ctx.partition_rowset(rs.values, rs.heap, spec)
    assert (idx == want).all()
    assert hist.tolist() == np.bincount(want, minlength=len(plen)).tolist()
    assert ctx.get_option("last_partition_key_words") == int(LAYOUTS[name]["long"])
    if slabs:
        order = np.argsort(want, kind="stable")
        for device in (False, True):
            v, h = _dev(rs) if device else (rs.values, rs.heap)
            idx, hist, slab, perm = ctx.partition_rowset_slabs(v, h, spec)
            if device:
                idx, hist, perm = _host(idx, np.int32), _host(hist, np.uint64), _host(perm)
                slab = _values(slab, rs.values.shape)
            assert (idx == want).all() and hist.tolist() == np.bincount(want, minlength=len(plen)).tolist()
            assert perm.tolist() == order.tolist()
            assert slab.tobytes() == rs.values[order].tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("flip", [0, 1])
@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_partition_handmade_bounds(ctx, name, flip):
    """Every hand-made bound of the layout at once, against the model."""
    rng = np.random.default_rng(17 + flip)
    rs, cols, _, desc = make_layout(name, 2500, seed=6, flip=flip)
    bounds = order_bounds(handmade_bounds(rs, cols, rng, count=6), desc)
    _partition_check(ctx, rs, cols, bounds, name, use_model=True, slabs=True)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [2, 9, 4096, 4097, 5000])
@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_partition_partition_counts(ctx, name, P):
    """Bounds from sorted samples mixed with hand-made ones; past 4096 partitions the histogram leaves shared memory."""
    rng = np.random.default_rng(P)
    rs, cols, _, desc = make_layout(name, 12000, seed=7, flip=P % 2)
    hand = handmade_bounds(rs, cols, rng, count=2)
    pool = hand + sample_bounds(rs, cols, rng, max(0, P - 1 - len(hand)))
    chosen = [pool[i] for i in sorted(rng.choice(len(pool), P - 1, replace=False))]
    _partition_check(ctx, rs, cols, order_bounds(chosen, desc), name, use_model=False, slabs=P in (9, 4097))


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(LAYOUTS))
def test_hash_partition_over_the_key_columns(ctx, name):
    rs, cols, _, _ = make_layout(name, 5000, seed=8)
    sentinel = (rs.values["type"] == T.Min) | (rs.values["type"] == T.Max)
    rs.values["type"][sentinel] = T.Null  # the hash partitioner rejects sentinels
    ncols = len(cols)
    for P in (7, 5000):
        want, _ = oracle.partition_hash(rs.values, rs.heap, P, ncols, salt=3)
        idx, hist = ctx.partition_rowset(rs.values, rs.heap, ctx._partition_spec(capi.PARTITION_HASH, P, key_column_count=ncols, salt=3))
        assert (idx == want).all()
        assert hist.tolist() == np.bincount(want, minlength=P).tolist()


# ------------------------------------------------------------------------------------------------------------ errors
def _error_case(kind, long):
    """A rowset and key columns that every entry point must reject with one code.  `long` puts the key past 256 bytes
    (a 300-byte string in another key column)."""
    n = 64
    rng = np.random.default_rng(1)
    strings = _pool_strings(rng, n, [b"x" * 300] if long else [b"xy", b"x"])
    rs = build_rowset(3, {0: strings, 1: gen_int64(rng, n)}, n)
    cols = [dict(index=0, type=T.String), dict(index=1, type=T.Int64, required=1)]
    if kind == "width":
        cols[0]["width"] = 299 if long else 1
        return rs, cols, capi.ERR_SCHEMA_VIOLATION
    if kind == "null_required":
        rs.values["type"][n // 2, 1] = T.Null
        return rs, cols, capi.ERR_SCHEMA_VIOLATION
    if kind in ("any", "composite"):
        rs.values["type"][n - 1, 0] = T.Any if kind == "any" else T.Composite
        return rs, cols, capi.ERR_UNSUPPORTED
    cols[1]["index"] = 3  # == value_count
    return rs, cols, capi.ERR_INVALID_ARGUMENT


@pytest.mark.gpu
@pytest.mark.parametrize("long", [False, True])
@pytest.mark.parametrize("kind", ["width", "null_required", "any", "composite", "index"])
def test_errors_on_every_entry_point(ctx, kind, long):
    rs, cols, code = _error_case(kind, long)
    off = np.array([0, 20, 64], dtype=np.uint64)
    bounds = bounds_rowset([(), ()], len(cols))
    calls = {
        "sort": lambda: ctx.sort_rowset(rs.values, rs.heap, cols, want_values=True),
        "merge": lambda: ctx.merge_sorted_runs(rs.values, rs.heap, cols, off),
        "join": lambda: ctx.join_sorted_runs(rs.values, rs.heap, cols, 1, off),
        "partition": lambda: ctx.partition_rowset(rs.values, rs.heap, _ordered_spec(ctx, cols, bounds, [0, 0], [1, 1])),
        "partition_slabs": lambda: ctx.partition_rowset_slabs(rs.values, rs.heap, _ordered_spec(ctx, cols, bounds, [0, 0], [1, 1])),
    }
    good, good_cols = make_layout("eight_alternating", 500, seed=9)[:2]
    want = ref_sort(good, [c["index"] for c in good_cols], [c["descending"] for c in good_cols])
    for name, call in calls.items():
        with pytest.raises(capi.YtGpuError) as e:
            call()
        assert e.value.code == code, (name, e.value.code, e.value.message)
        # the context stays usable
        assert (ctx.sort_rowset(good.values, good.heap, good_cols) == want).all(), name
