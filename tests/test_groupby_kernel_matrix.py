"""Both hash GROUP BY kernels, specialisation by specialisation, against exact references.

ytgpu_scan_filter_groupby (csrc/columnar.cu) compiles groupby_kernel<LOCAL, KDIRECT, VDIRECT, DBL, PLAIN> twenty ways and
groupby_impl picks one from the shape of its input:
  KDIRECT / VDIRECT  the column is a plain 64-bit vector: no null bitmap, dictionary or RLE (base / zig-zag allowed);
  LOCAL              0 < hint <= 2048 and no MIN / MAX requested (a shared-memory front table per CTA);
  PLAIN              both columns direct without base / zig-zag, no predicate, no first rows, no MIN / MAX.
ytgpu_scan_filter_groupby_multi (csrc/groupby_multi.cu) compiles mg_assign_kernel<DIRECT, NK> six ways:
  DIRECT             every key column is direct without base / zig-zag;  NK = 1, 2, else 0 (3..8 key columns).
FUSED_CASES and ASSIGN_CASES below name, for every instantiation, the input that reaches it.

References: the C++ oracle (oracle/yt_oracle.cpp) for grouping, first-seen order, counts, integer aggregates, MIN / MAX and
row selection; a plain Python model for SUM / AVG of doubles — math.fsum per group, and a result is right when
|got - exact| <= gamma(c - 1) * sum|x| (gamma(k) = k u / (1 - k u), u = 2^-53), the bound of every summation order over c
values.  Float edges follow one rule for all aggregators: MIN / MAX use the order-free total order (NaN the largest,
returned as the canonical quiet NaN) and are compared with the oracle's YQL style on data with NaN, with its QL style
otherwise; -0.0 and +0.0 compare equal by value, every other result bit for bit."""
import math
import struct

import numpy as np
import pytest

import oracle
from oracle import AGG_ARGMAX, AGG_ARGMIN, AGG_AVG, AGG_COUNT, AGG_FIRST, AGG_MAX, AGG_MIN, AGG_SUM
from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import EValueType as T

U = 2.0 ** -53
VKIND = {T.Int64: oracle.VAL_INT64, T.Uint64: oracle.VAL_UINT64, T.Double: oracle.VAL_DOUBLE}
OPS = [capi.CMP_LT, capi.CMP_LE, capi.CMP_GT, capi.CMP_GE, capi.CMP_EQ, capi.CMP_NE]

# (LOCAL, KDIRECT, VDIRECT, DBL, PLAIN, key encoding, value encoding, what keeps a direct/direct pair off PLAIN)
# encodings: plain = 64-bit vector; base = 64-bit vector with base and zig-zag (direct, not PLAIN); bitmap = null bitmap;
# dict = dictionary, index 0 = NULL; rle = run-length with a null bitmap over the runs; packed = bit-packed with a base
FUSED_CASES = [
    (True, True, True, False, True, "plain", "plain", None),
    (True, True, True, True, True, "plain", "plain", None),
    (False, True, True, False, True, "plain", "plain", None),
    (False, True, True, True, True, "plain", "plain", None),
    (True, True, True, False, False, "base", "plain", "base"),
    (True, True, True, True, False, "plain", "plain", "first"),
    (True, True, False, False, False, "plain", "bitmap", None),
    (True, True, False, True, False, "base", "dict", None),
    (True, False, True, False, False, "rle", "base", None),
    (True, False, True, True, False, "bitmap", "plain", None),
    (True, False, False, False, False, "dict", "packed", None),
    (True, False, False, True, False, "packed", "rle", None),
    (False, True, True, False, False, "plain", "base", "base"),
    (False, True, True, True, False, "base", "plain", "base"),
    (False, True, False, False, False, "base", "rle", None),
    (False, True, False, True, False, "plain", "bitmap", None),
    (False, False, True, False, False, "packed", "plain", None),
    (False, False, True, True, False, "dict", "plain", None),
    (False, False, False, False, False, "bitmap", "dict", None),
    (False, False, False, True, False, "rle", "bitmap", None),
]

# (DIRECT, NK, key column counts, key encodings cycled over the columns)
ASSIGN_CASES = [
    (True, 1, (1,), ("plain",)),
    (True, 2, (2,), ("plain",)),
    (True, 0, (3, 5, 8), ("plain",)),
    (False, 1, (1,), ("bitmap", "base", "dict", "rle", "packed")),
    (False, 2, (2,), ("plain", "dict", "rle", "bitmap", "base", "packed")),
    (False, 0, (3, 5, 8), ("plain", "base", "bitmap", "dict", "rle", "packed")),
]


def _case_id(c):
    return "{}{}{}{}{}-{}-{}".format("L" if c[0] else "G", "K" if c[1] else "k", "V" if c[2] else "v", "D" if c[3] else "I",
                                     "P" if c[4] else "", c[5], c[6])


# ------------------------------------------------------------------------------------------------- references
def _f(bits):
    return struct.unpack("<d", struct.pack("<Q", int(bits) & 0xFFFFFFFFFFFFFFFF))[0]


def _bits(x):
    return struct.unpack("<Q", struct.pack("<d", float(x)))[0]


def _gamma(k):
    return k * U / (1 - k * U)


def exact_sum(xs, dbl):
    """-> (exact sum, sum of |x|): a Python int mod 2^64 for integers; for doubles math.fsum, NaN when any value is NaN or
    both infinities occur, the infinity otherwise."""
    if not dbl:
        return sum(int(x) for x in xs) % 2**64, 0.0
    xs = [float(x) for x in xs]
    if any(math.isnan(x) for x in xs) or (math.inf in xs and -math.inf in xs):
        return math.nan, math.inf
    if math.inf in xs or -math.inf in xs:
        return (math.inf if math.inf in xs else -math.inf), math.inf
    return math.fsum(xs), math.fsum(abs(x) for x in xs)


def sum_ok(got, xs, avg=False):
    """A double SUM (or AVG) of the values xs, in any summation order."""
    exact, mag = exact_sum(xs, True)
    c = len(xs)
    if avg:
        exact /= c
    if math.isnan(exact) or math.isinf(exact):
        return (math.isnan(got) and math.isnan(exact)) or got == exact
    bound = _gamma(c - 1) * mag
    if avg:
        bound = bound / c + 2 * U * abs(got)  # the sum's error shrinks by c; the division rounds once
    return abs(got - exact) <= bound


def same_extremum(got_bits, want_bits, dbl):
    if not dbl:
        return int(got_bits) == int(want_bits)
    g, w = _f(got_bits), _f(want_bits)
    return (math.isnan(g) and math.isnan(w)) or g == w  # -0.0 == +0.0 by value, everything else bit for bit


def passes(op, vtype, vals, vnull, const):
    """passes() of columnar.cuh over a whole column: a NULL never passes; with a NaN only NE holds."""
    if vtype == T.Double:
        a, c = vals.view(np.float64), np.float64(_f(const))
    elif vtype == T.Int64:
        a, c = vals.view(np.int64), np.int64(np.uint64(const & 0xFFFFFFFFFFFFFFFF).view(np.int64))
    else:
        a, c = vals, np.uint64(const & 0xFFFFFFFFFFFFFFFF)
    with np.errstate(invalid="ignore"):
        r = {capi.CMP_LT: a < c, capi.CMP_LE: a <= c, capi.CMP_GT: a > c, capi.CMP_GE: a >= c, capi.CMP_EQ: a == c,
             capi.CMP_NE: a != c}[op]
    return r & ~vnull


def _groups_sorted(keys, knull, valid):
    """Rows that pass, grouped by (key_null, key) in the fused kernel's output order -> (rows in group order, starts)."""
    rows = np.flatnonzero(valid)
    kn = knull[rows]
    k = np.where(kn, np.uint64(0), keys[rows])
    order = np.lexsort((rows, k, kn))
    rows, k, kn = rows[order], k[order], kn[order]
    starts = np.flatnonzero(np.r_[True, (k[1:] != k[:-1]) | (kn[1:] != kn[:-1])]) if len(rows) else np.zeros(0, np.int64)
    return rows, starts, k[starts], kn[starts]


# ------------------------------------------------------------------------------------------------- inputs
def _bm(mask):
    return np.packbits(np.asarray(mask, dtype=np.uint8), bitorder="little")


def encode(kind, vtype, logical, nulls, start, rng):
    """A Column of `kind` whose rows [start, start + n) decode to `logical` (NULL where `nulls`); the rows before the window
    hold other values, so a kernel that ignores start_index reads wrong data."""
    from ytsaurus_b200 import Column
    n = len(logical)
    full = np.concatenate([rng.integers(0, 2**64 - 1, start, dtype=np.uint64, endpoint=True), logical]).astype(np.uint64)
    fnull = np.zeros(start + n, bool)
    if nulls is not None:
        fnull[start:] = nulls
    if kind in ("plain", "base", "packed"):
        assert nulls is None or not nulls.any(), kind
    if kind == "plain":
        return Column(vtype, values=full, start_index=start, value_count=n)
    if kind == "base":
        base = int(rng.integers(0, 2**64 - 1, dtype=np.uint64, endpoint=True))
        x = full.view(np.int64)
        zz = ((x << 1) ^ (x >> 63)).view(np.uint64)
        return Column(vtype, values=zz - np.uint64(base), start_index=start, value_count=n, base_value=base, zigzag=True)
    if kind == "bitmap":
        return Column(vtype, values=full, start_index=start, value_count=n, null_bitmap=_bm(fnull))
    if kind == "dict":
        uniq, inv = np.unique(full, return_inverse=True)
        idx = (inv.reshape(-1) + 1).astype(np.uint32)
        idx[fnull] = 0
        return Column(vtype, values=uniq, dictionary_indexes=idx, start_index=start, value_count=n)
    if kind == "rle":
        change = np.r_[True, (full[1:] != full[:-1]) | (fnull[1:] != fnull[:-1])]
        runs = np.flatnonzero(change)
        return Column(vtype, values=full[runs].copy(), rle_indexes=runs.astype(np.uint64), null_bitmap=_bm(fnull[runs]),
                      start_index=start, value_count=n)
    if kind == "packed":
        base = full.min()
        raw = full - base
        col = Column(vtype, values=oracle.bit_pack(raw, int(raw.max())), bit_width=0, base_value=int(base), start_index=start,
                     value_count=n)
        col.unpacked = raw  # for the encoders' own test
        return col
    raise ValueError(kind)


def nullable(kind):
    return kind in ("bitmap", "dict", "rle")


def to_device(col):
    import torch
    for attr in ("values", "null_bitmap", "dictionary_indexes", "rle_indexes"):
        a = getattr(col, attr)
        if a is not None:
            signed = {1: np.uint8, 4: np.int32, 8: np.int64}[a.dtype.itemsize]
            setattr(col, attr, torch.from_numpy(np.ascontiguousarray(a).view(signed)).cuda())
    return col


def host(x):
    import torch
    if torch.is_tensor(x):
        x = x.cpu().numpy()
    return x.view(np.uint64) if x.dtype.itemsize == 8 else x


def make_keys(rng, n, groups, pattern, with_nulls):
    """Keys from `groups` distinct 64-bit values including 0 and 2^64 - 1 (the tables' empty-slot marker), every value
    present when n allows; sorted: runs of at least 64 rows (whole warps on one key)."""
    assert groups >= 2
    domain = rng.permutation(np.unique(rng.integers(1, 2**64 - 2, groups * 2, dtype=np.uint64)))[: groups - 2]
    domain = np.r_[np.asarray([0, 2**64 - 1], dtype=np.uint64), domain]
    keys = domain[rng.permutation(n) % groups] if n >= groups else domain[rng.integers(0, groups, n)]
    if pattern == "sorted":
        keys = np.sort(keys)
        # stretch short runs so that every run covers 64 rows
        keys = np.repeat(keys[::64], 64)[:n] if n >= 64 else keys
    knull = np.zeros(n, bool)
    if with_nulls:
        if pattern == "sorted":
            knull[: min(n, 128)] = True
        else:
            knull = rng.random(n) < 0.02
    return keys.astype(np.uint64), knull, domain


def make_values(rng, vtype, n, keys, domain, with_nulls, nan=False):
    """Values at the edges of each type; with NULLs: one group whose values are all NULL."""
    if vtype == T.Int64:
        v = rng.integers(-2**62, 2**62, n, dtype=np.int64)
        pick = rng.random(n)
        v[pick < 0.2] = -1
        v[(pick >= 0.2) & (pick < 0.45)] = 0xFFFFFFFF          # the low word carries in every 2 x 32-bit add
        v[(pick >= 0.45) & (pick < 0.5)] = np.iinfo(np.int64).min
        v[(pick >= 0.5) & (pick < 0.55)] = np.iinfo(np.int64).max
        if len(domain) > 2:
            v[keys == domain[2]] = 0xFFFFFFFF                  # one heavy group of carries
        bits = v.view(np.uint64)
    elif vtype == T.Uint64:
        bits = rng.integers(0, 2**64 - 1, n, dtype=np.uint64, endpoint=True)
        pick = rng.random(n)
        bits[pick < 0.3] |= np.uint64(2**63)
        bits[(pick >= 0.3) & (pick < 0.4)] = 0xFFFFFFFF
        bits[(pick >= 0.4) & (pick < 0.45)] = 2**64 - 1
    else:
        d = rng.standard_normal(n) * 1e3
        pick = rng.random(n)
        big = (pick < 0.005)
        d[big] = np.where(rng.random(int(big.sum())) < 0.5, 1e300, -1e300)   # huge values that cancel
        d[(pick >= 0.05) & (pick < 0.1)] = rng.integers(-50, 50, int(((pick >= 0.05) & (pick < 0.1)).sum())) * 5e-324
        d[(pick >= 0.1) & (pick < 0.15)] = -0.0
        d[(pick >= 0.15) & (pick < 0.2)] = 0.0
        d[(pick >= 0.2) & (pick < 0.202)] = np.inf
        d[(pick >= 0.202) & (pick < 0.204)] = -np.inf
        if nan:
            d[(pick >= 0.204) & (pick < 0.21)] = np.nan
        if len(domain) > 3:
            sel = keys == domain[3]
            d[sel] = np.where(np.arange(int(sel.sum())) % 2, -0.0, 0.0)       # a group of signed zeros only
        bits = d.view(np.uint64)
    vnull = np.zeros(n, bool)
    if with_nulls:
        vnull = rng.random(n) < 0.1
        if len(domain) > 4:
            vnull[keys == domain[4]] = True                    # a group whose values are all NULL
    return bits.copy(), vnull


# ------------------------------------------------------------------------------------------------- CPU: references
def test_exact_sum_model():
    assert exact_sum([2**64 - 1, 1, 5], False)[0] == 5
    assert exact_sum([1e300, 1.0, -1e300], True)[0] == 1.0
    assert math.isnan(exact_sum([math.inf, -math.inf], True)[0]) and math.isnan(exact_sum([1.0, math.nan], True)[0])
    assert exact_sum([math.inf, 1.0], True)[0] == math.inf and exact_sum([-math.inf, -1e308, -1e308], True)[0] == -math.inf
    assert not sum_ok(1.0 + 2**-40, [1.0]) and not sum_ok(3.0 + 2**-40, [1.0, 1.0, 1.0])
    assert sum_ok(1.0, [1e16, 1.0, -1e16]) and sum_ok(0.0, [1e16, 1.0, -1e16])  # both orders of a cancelling sum
    xs = [0.1] * 10
    assert sum_ok(sum(xs), xs) and sum_ok(math.fsum(xs), xs) and sum_ok(sum(xs) / 10, xs, avg=True)
    assert sum_ok(-0.0, [-0.0]) and sum_ok(0.0, [-0.0])     # the sign of a zero sum is not part of the rule


def test_case_tables_cover_every_instantiation():
    fused = {c[:5] for c in FUSED_CASES}
    want = {(loc, True, True, d, True) for loc in (True, False) for d in (True, False)}
    want |= {(loc, k, v, d, False) for loc in (True, False) for k in (True, False) for v in (True, False) for d in (True, False)}
    assert fused == want and len(FUSED_CASES) == 20
    for loc, kd, vd, dbl, plain, kk, vk, breaker in FUSED_CASES:
        assert kd == (kk in ("plain", "base")) and vd == (vk in ("plain", "base"))
        if kd and vd:
            assert plain == (kk == vk == "plain" and breaker is None)
    assert {(d, nk) for d, nk, _, _ in ASSIGN_CASES} == {(d, nk) for d in (True, False) for nk in (1, 2, 0)}
    for direct, nk, counts, kinds in ASSIGN_CASES:
        assert all((c == nk) if nk else c >= 3 for c in counts)
        assert direct == (set(kinds) == {"plain"})


def test_encodings_decode_to_the_logical_values():
    rng = np.random.default_rng(5)
    n = 300
    logical = rng.integers(0, 2**64 - 1, n, dtype=np.uint64, endpoint=True)
    logical[:40] = logical[0]
    nulls = rng.random(n) < 0.1
    for kind in ("plain", "base", "bitmap", "dict", "rle", "packed"):
        for start in (0, 1, 3):
            col = encode(kind, T.Uint64, logical, nulls if nullable(kind) else None, start, rng)
            kw = dict(dict_idx=col.dictionary_indexes, rle_idx=col.rle_indexes, bitmap=col.null_bitmap)
            raw = col.values if kind != "packed" else col.unpacked
            got = oracle.decode_integer_vector(start, start + n, col.base_value & 0xFFFFFFFFFFFFFFFF, col.zigzag, raw, **kw)
            mode = {"bitmap": 0, "dict": 1, "rle": 2}.get(kind, 4)
            gn = oracle.build_null_bytemap(mode, start, start + n, **kw).astype(bool)
            want_null = nulls if nullable(kind) else np.zeros(n, bool)
            assert (gn == want_null).all(), kind
            assert (got[~want_null] == logical[~want_null]).all(), (kind, start)


def test_oracle_multi_min_max_styles():
    """QL: min replaces when state >= new, max when state < new — next to a NaN both are false, so the row order decides;
    YQL (the kernels' order): NaN the largest value, of equal values the first stays."""
    def run(vals, style, op):
        bits = np.asarray([_bits(x) for x in vals], dtype=np.uint64)
        r = oracle.groupby_multi([np.zeros(len(vals), np.uint64)], None, [bits], None, [T.Double], [(op, 0)], style=style)
        return _f(r["values"][0][0])
    QL, YQL = oracle.MINMAX_QL, oracle.MINMAX_YQL
    assert run([1.0, math.nan], QL, AGG_MIN) == 1.0 and math.isnan(run([math.nan, 1.0], QL, AGG_MIN))
    assert run([1.0, math.nan], QL, AGG_MAX) == 1.0 and math.isnan(run([math.nan, 1.0], QL, AGG_MAX))
    for order in ([1.0, math.nan], [math.nan, 1.0]):
        assert run(order, YQL, AGG_MIN) == 1.0 and math.isnan(run(order, YQL, AGG_MAX))
    # signed zeros: QL's `state >= new` takes the later of two equal values, YQL keeps the first
    assert math.copysign(1, run([0.0, -0.0], QL, AGG_MIN)) == -1 and math.copysign(1, run([0.0, -0.0], YQL, AGG_MIN)) == 1
    assert math.copysign(1, run([0.0, -0.0], QL, AGG_MAX)) == 1 and math.copysign(1, run([-0.0, 0.0], YQL, AGG_MAX)) == -1
    # argmin / argmax: the first row wins ties in both styles; YQL orders NaN last
    arg = np.arange(3, dtype=np.uint64)
    by = np.asarray([_bits(x) for x in (math.nan, 2.0, 2.0)], dtype=np.uint64)
    r = oracle.groupby_multi([np.zeros(3, np.uint64)], None, [arg, by], None, [T.Int64, T.Double],
                             [(AGG_ARGMIN, 0, 1), (AGG_ARGMAX, 0, 1)], style=YQL)
    assert r["values"][0].tolist() == [1] and r["values"][1].tolist() == [0]


def test_oracle_multi_styles_agree_with_the_single_key_oracle():
    rng = np.random.default_rng(8)
    n = 20000
    keys = rng.integers(0, 50, n, dtype=np.uint64)
    d = rng.standard_normal(n)
    d[rng.random(n) < 0.05] = np.nan
    d[rng.random(n) < 0.05] = 0.0
    d[rng.random(n) < 0.05] = -0.0
    vn = rng.random(n) < 0.1
    for style in (oracle.MINMAX_QL, oracle.MINMAX_YQL):
        one = oracle.groupby_min_max(keys, d, oracle.VAL_DOUBLE, val_null=vn.astype(np.uint8), style=style)
        many = oracle.groupby_multi([keys], None, [d.view(np.uint64)], [vn], [T.Double], [(AGG_MIN, 0), (AGG_MAX, 0)], style=style)
        o = np.argsort(many["keys"][0])
        assert many["keys"][0][o].tolist() == one["keys"].tolist()
        if style == oracle.MINMAX_YQL:  # both keep the first of equal values: bit for bit
            assert many["values"][0][o].tolist() == one["min"].tolist() and many["values"][1][o].tolist() == one["max"].tolist()
        else:  # the single-key oracle's QL min is !(state < new); the same as state >= new on NaN-free groups
            nan_free = np.asarray([not np.isnan(d[(keys == k) & ~vn]).any() for k in one["keys"]])
            assert (many["values"][0][o][nan_free] == one["min"][nan_free]).all()
            assert many["values"][1][o].tolist() == one["max"].tolist()


# ------------------------------------------------------------------------------------------------- GPU: fused kernel
@pytest.fixture(scope="module")
def ctx():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from ytsaurus_b200 import GpuContext
    c = GpuContext(0)
    yield c
    c.close()


def check_fused(got, keys, knull, bits, vnull, valid, vtype, first=False, minmax=False, nan=False):
    dbl = vtype == T.Double
    want = oracle.groupby_sum_count(keys, bits, VKIND[vtype], knull.astype(np.uint8), vnull.astype(np.uint8),
                                    filt=valid.astype(np.uint8), style=oracle.STYLE_CH)
    got = {k: host(v) for k, v in got.items()}
    g = len(want["count"])
    assert len(got["count"]) == g
    assert got["keys"].tolist() == want["keys"].tolist()
    assert got["key_null"].tolist() == want["key_null"].tolist()
    assert got["count"].tolist() == want["count"].tolist()
    assert got["sum_null"].tolist() == want["sum_null"].tolist()
    rows, starts, mk, mkn = _groups_sorted(keys, knull, valid)
    assert mk.tolist() == want["keys"].tolist() and mkn.astype(np.uint8).tolist() == want["key_null"].tolist()
    ends = np.r_[starts[1:], len(rows)]
    for j in range(g):
        r = rows[starts[j]:ends[j]]
        r = r[~vnull[r]]
        if not len(r):
            continue
        if dbl:
            xs = bits[r].view(np.float64)
            assert sum_ok(_f(got["sum"][j]), xs), (j, _f(got["sum"][j]), exact_sum(xs, True))
        else:
            assert int(got["sum"][j]) == exact_sum(bits[r], False)[0] == int(want["sum"][j]), j
    if first:
        assert got["first_row"].tolist() == rows[starts].tolist()
    if minmax:
        mm = oracle.groupby_min_max(keys, bits, VKIND[vtype], knull.astype(np.uint8), vnull.astype(np.uint8),
                                    filt=valid.astype(np.uint8), style=oracle.MINMAX_YQL if nan else oracle.MINMAX_QL)
        assert mm["keys"].tolist() == want["keys"].tolist()
        for j in np.flatnonzero(mm["null"] == 0):
            assert same_extremum(got["min"][j], mm["min"][j], dbl), ("min", j, got["min"][j], mm["min"][j])
            assert same_extremum(got["max"][j], mm["max"][j], dbl), ("max", j, got["max"][j], mm["max"][j])


def run_fused(ctx, case, rng, n, start, pattern, groups, hint, device, predicate=None, nan=False, minmax=False):
    loc, kd, vd, dbl, plain, kk, vk, breaker = case
    vtype = T.Double if dbl else (T.Int64 if rng.random() < 0.5 else T.Uint64)
    keys, knull, domain = make_keys(rng, n, groups, pattern, nullable(kk))
    bits, vnull = make_values(rng, vtype, n, keys, domain, nullable(vk), nan=nan)
    kcol = encode(kk, T.Uint64, keys, knull if nullable(kk) else None, start, rng)
    vcol = encode(vk, vtype, bits, vnull if nullable(vk) else None, start, rng)
    if device:
        kcol, vcol = to_device(kcol), to_device(vcol)
    first = breaker == "first" or (not plain and (start + n) % 2 == 1)
    minmax = minmax and not loc and not plain
    valid = np.ones(n, bool)
    pred = None
    if predicate is not None:
        op, const = predicate
        valid = passes(op, vtype, bits, vnull, const)
        pred = predicate
    got = ctx.scan_filter_groupby(kcol, vcol, pred, group_count_hint=hint, want_first_rows=first, want_min_max=minmax,
                                  capacity=n + 2)
    check_fused(got, keys, knull, bits, vnull, valid, vtype, first=first, minmax=minmax, nan=nan)


def _fused_hint(case, groups):
    loc = case[0]
    if loc:
        return min(groups, 2048)
    return 0 if groups < 3000 else 3000  # hints above 2048 keep the global table


@pytest.mark.gpu
@pytest.mark.parametrize("case", FUSED_CASES, ids=_case_id)
def test_fused_instance(ctx, case):
    loc, kd, vd, dbl, plain, kk, vk, breaker = case
    rng = np.random.default_rng(FUSED_CASES.index(case))
    it = 0
    for start in (0, 1, 3):
        for n in (20001, 20000):
            for pattern in ("random", "sorted"):
                it += 1
                run_fused(ctx, case, rng, n, start, pattern, 300, _fused_hint(case, 300), device=it % 2 == 0,
                          nan=dbl and it % 3 == 0, minmax=it % 2 == 1)
    # group counts around the small-result sort (<= 4096 groups) and a small hint that overflows the tables
    for groups, hint in ((4096, None), (4097, None), (6000, 16 if loc else (3000 if plain else 16))):
        run_fused(ctx, case, rng, 30001, 1, "random", groups, _fused_hint(case, groups) if hint is None else hint,
                  device=groups % 2 == 1, minmax=not plain and not loc and hint is not None)
    if plain:
        return
    # the predicate on the value column, every op; uint64 constants >= 2^63, NaN values and a NaN constant for doubles
    for i, op in enumerate(OPS):
        run_fused_pred(ctx, case, rng, op, (_bits(math.nan) if i % 2 else _bits(0.0)) if dbl else None, i)


def run_fused_pred(ctx, case, rng, op, const, i):
    loc, kd, vd, dbl, plain, kk, vk, breaker = case
    n, start = 20001, i % 4
    vtype = T.Double if dbl else (T.Int64, T.Uint64)[i % 2]
    keys, knull, domain = make_keys(rng, n, 500, "random" if i % 3 else "sorted", nullable(kk))
    bits, vnull = make_values(rng, vtype, n, keys, domain, nullable(vk), nan=dbl)
    if const is None:
        const = int(bits[rng.integers(0, n)]) if i % 2 else ({T.Int64: 0, T.Uint64: 2**63}[vtype])
        if vtype == T.Uint64:
            const |= 2**63
    kcol = encode(kk, T.Uint64, keys, knull if nullable(kk) else None, start, rng)
    vcol = encode(vk, vtype, bits, vnull if nullable(vk) else None, start, rng)
    valid = passes(op, vtype, bits, vnull, const)
    got = ctx.scan_filter_groupby(kcol, vcol, (op, const), group_count_hint=_fused_hint(case, 500), want_first_rows=i % 2 == 0,
                                  capacity=n + 2)
    check_fused(got, keys, knull, bits, vnull, valid, vtype, first=i % 2 == 0)


@pytest.mark.gpu
def test_fused_signed_zeros_nan_and_double_keys(ctx):
    """MIN / MAX: -0.0 orders below +0.0 and NaN above +inf, whatever the row order; double keys group by bit pattern."""
    from ytsaurus_b200 import Column
    z, nz, nan = _bits(0.0), _bits(-0.0), _bits(math.nan)
    keys = np.asarray([1, 1, 2, 2, 3, 3, 4, 4], dtype=np.uint64)
    vals = np.asarray([z, nz, nz, z, _bits(1.0), nan, nan, _bits(1.0)], dtype=np.uint64)
    got = ctx.scan_filter_groupby(Column(T.Uint64, values=keys), Column(T.Double, values=vals), want_min_max=True)
    assert got["min"].tolist() == [nz, nz, _bits(1.0), _bits(1.0)]
    assert got["max"].tolist() == [z, z, 0x7ff8000000000000, 0x7ff8000000000000]
    # double keys: -0.0 / +0.0 and two NaN payloads are four groups (the sort's key order treats each pair as equal)
    dk = np.asarray([z, nz, nan, nan | 1, z, nz, nan, nan | 1], dtype=np.uint64)
    v = np.arange(8, dtype=np.uint64)
    got = ctx.scan_filter_groupby(Column(T.Double, values=dk), Column(T.Int64, values=v))
    assert sorted(got["keys"].tolist()) == sorted({z, nz, nan, nan | 1}) and got["count"].tolist() == [2] * 4
    multi = ctx.scan_filter_groupby_multi([Column(T.Double, values=dk)], [Column(T.Int64, values=v)], [(AGG_SUM, 0)])
    want = oracle.groupby_multi([dk], None, [v], None, [T.Int64], [(AGG_SUM, 0)])
    assert multi["keys"][0].tolist() == want["keys"][0].tolist() == [z, nz, nan, nan | 1]
    assert multi["values"][0].tolist() == want["values"][0].tolist() == [4, 6, 8, 10]


@pytest.mark.gpu
def test_fused_million_groups_per_group(ctx):
    """1.2 * 10^6 groups: the output order comes from the radix sort's packed three-pass schedule; every group's key,
    count and sum is compared, the sentinel key and NULL keys included."""
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(12)
    n, groups = 3_000_001, 1_200_000
    keys, knull, domain = make_keys(rng, n, groups, "random", True)
    bits, vnull = make_values(rng, T.Int64, n, keys, domain, True)
    for hint in (0, groups):
        got = ctx.scan_filter_groupby(Column(T.Uint64, values=keys, null_bitmap=_bm(knull)),
                                      Column(T.Int64, values=bits, null_bitmap=_bm(vnull)), group_count_hint=hint)
        want = oracle.groupby_sum_count(keys, bits, oracle.VAL_INT64, knull.astype(np.uint8), vnull.astype(np.uint8),
                                        style=oracle.STYLE_CH)
        assert len(want["count"]) > 1_100_000
        for f in ("keys", "key_null", "count", "sum", "sum_null"):
            assert np.array_equal(got[f], want[f]), f


# ------------------------------------------------------------------------------------------------- GPU: general GROUP BY
def aggregates_32():
    """32 aggregates over value columns 0 = int64, 1 = uint64, 2 = double, 3 = boolean (4 = int64 with ties)."""
    aggs = [(AGG_SUM, c) for c in (0, 1, 2)] + [(AGG_AVG, c) for c in (0, 1, 2)]
    for op in (AGG_MIN, AGG_MAX, AGG_COUNT, AGG_FIRST):
        aggs += [(op, c) for c in (0, 1, 2, 3)]
    aggs += [(AGG_ARGMIN, 4, b) for b in (0, 1, 2, 3)] + [(AGG_ARGMAX, 2, b) for b in (0, 1, 2, 3)]
    aggs += [(AGG_SUM, 4), (AGG_MIN, 4)]
    assert len(aggs) == 32
    return aggs


def bool_column(bits, nulls, start, rng):
    from ytsaurus_b200 import Column
    n = len(bits)
    full = np.concatenate([rng.integers(0, 2, start).astype(bool), bits.astype(bool)])
    fnull = np.zeros(start + n, bool)
    fnull[start:] = nulls
    return Column(T.Boolean, values=_bm(full), bit_width=1, start_index=start, value_count=n, null_bitmap=_bm(fnull))


def multi_values(rng, n, keys0, domain, nan):
    i64, in_ = make_values(rng, T.Int64, n, keys0, domain, True)
    u64, _ = make_values(rng, T.Uint64, n, keys0, domain, False)
    d, dn = make_values(rng, T.Double, n, keys0, domain, True, nan=nan)
    b = (rng.random(n) < 0.5).astype(np.uint64)
    bn = rng.random(n) < 0.1
    ties = rng.integers(-3, 3, n).astype(np.int64).view(np.uint64)
    return [i64, u64, d, b, ties], [in_, np.zeros(n, bool), dn, bn, np.zeros(n, bool)]


def check_multi(got, want, aggs, vals, vnulls, vtypes, gids_rows):
    got = {k: ([host(x) for x in v] if isinstance(v, list) else host(v)) for k, v in got.items()}
    g = len(want["count"])
    assert len(got["count"]) == g
    for a, b in zip(got["keys"], want["keys"]):
        assert a.tolist() == b.tolist()
    for a, b in zip(got["key_null"], want["key_null"]):
        assert a.tolist() == b.tolist()
    assert got["count"].tolist() == want["count"].tolist()
    assert got["first_row"].tolist() == want["first_row"].tolist()
    for a, agg in enumerate(aggs):
        op, col = agg[0], agg[1]
        gv, gn = got["values"][a], got["value_null"][a]
        assert gn.tolist() == want["value_null"][a].tolist(), f"aggregate {a} {agg} nulls"
        dbl = vtypes[col] == T.Double
        if dbl and op in (AGG_SUM, AGG_AVG):
            for j in np.flatnonzero(gn == 0):
                r = gids_rows[j]
                r = r[~vnulls[col][r]]
                assert sum_ok(_f(gv[j]), vals[col][r].view(np.float64), avg=op == AGG_AVG), (a, agg, j)
        elif op in (AGG_MIN, AGG_MAX) and dbl:
            for j in np.flatnonzero(gn == 0):
                assert same_extremum(gv[j], want["values"][a][j], True), (a, agg, j)
        else:
            assert gv.tolist() == want["values"][a].tolist(), f"aggregate {a} {agg}"


def first_seen_groups(keys, knulls, valid):
    """Rows of each group, groups in first-seen order (the general kernel's output order)."""
    rows = np.flatnonzero(valid)
    if not len(rows):
        return []
    cols = []
    for k, kn in zip(keys, knulls):
        cols += [kn[rows].astype(np.uint64), np.where(kn[rows], np.uint64(0), k[rows])]
    tup = np.stack(cols, axis=1)
    _, first, inv = np.unique(tup, axis=0, return_index=True, return_inverse=True)
    inv = inv.reshape(-1)
    order = np.argsort(first, kind="stable")
    rank = np.empty_like(order)
    rank[order] = np.arange(len(order))
    gid = rank[inv]
    srt = np.argsort(gid, kind="stable")
    bounds = np.flatnonzero(np.r_[True, gid[srt][1:] != gid[srt][:-1], True])
    return [rows[srt[bounds[i]:bounds[i + 1]]] for i in range(len(bounds) - 1)]


def run_multi(ctx, rng, kinds, nk, n, pattern, groups, hint, device, nan=False, predicate=None, aggs=None):
    aggs = aggs or aggregates_32()
    keys, knulls, kcols = [], [], []
    per_col = max(2, int(round(groups ** (1.0 / nk))))
    k0, kn0, domain = make_keys(rng, n, per_col if nk > 1 else groups, pattern, False)
    for c in range(nk):
        kind = kinds[c % len(kinds)]
        k, kn, _ = (k0, kn0, domain) if c == 0 else make_keys(rng, n, per_col, pattern, False)
        if pattern == "sorted" and c:
            k = np.sort(k)   # a sorted tuple: every column sorted keeps whole warps on one tuple
        if nullable(kind):
            kn = rng.random(n) < 0.03 if pattern == "random" else np.r_[np.ones(min(n, 64), bool), np.zeros(max(n - 64, 0), bool)]
        start = int(rng.integers(0, 4))
        col = encode(kind, T.Uint64 if c % 2 else T.Int64, k, kn if nullable(kind) else None, start, rng)
        keys.append(k)
        knulls.append(kn)
        kcols.append(col)
    vals, vnulls = multi_values(rng, n, k0, domain, nan)
    vtypes = [T.Int64, T.Uint64, T.Double, T.Boolean, T.Int64]
    vcols = []
    for c, (v, vn, t) in enumerate(zip(vals, vnulls, vtypes)):
        start = int(rng.integers(0, 4))
        if t == T.Boolean:
            vcols.append(bool_column(v, vn, start, rng))
        else:
            vcols.append(encode("bitmap" if vn.any() else "plain", t, v, vn if vn.any() else None, start, rng))
    if device:
        kcols, vcols = [to_device(c) for c in kcols], [to_device(c) for c in vcols]
    valid = np.ones(n, bool)
    kw = {}
    if predicate is not None:
        pcol, op, const = predicate
        valid = passes(op, vtypes[pcol] if vtypes[pcol] != T.Boolean else T.Uint64, vals[pcol], vnulls[pcol], const)
        kw = dict(predicate=(op, const), predicate_column=pcol)
    got = ctx.scan_filter_groupby_multi(kcols, vcols, aggs, group_count_hint=hint, **kw)
    want = oracle.groupby_multi(keys, [kn.astype(np.uint8) for kn in knulls], vals, [vn.astype(np.uint8) for vn in vnulls], vtypes,
                                aggs, filt=valid.astype(np.uint8), style=oracle.MINMAX_YQL if nan else oracle.MINMAX_QL)
    check_multi(got, want, aggs, vals, vnulls, vtypes, first_seen_groups(keys, knulls, valid))
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("case", ASSIGN_CASES, ids=lambda c: f"{'D' if c[0] else 'd'}{c[1]}")
def test_multi_assign_instance(ctx, case):
    direct, nk_t, counts, kinds = case
    rng = np.random.default_rng(100 + 10 * int(direct) + nk_t)
    for nk in counts:
        for n in (1, 31, 32, 33):
            run_multi(ctx, rng, kinds, nk, n, "random", 8, 0, device=n == 32)
        it = 0
        for pattern in ("random", "sorted"):
            # shared-memory caches (table <= 4096 slots), the global table, and a hint that forces table-full retries
            for groups, hint in ((200, 200), (3000, 0), (1500, 1)):
                it += 1
                run_multi(ctx, rng, kinds, nk, 20001, pattern, groups, hint, device=it % 2 == 0, nan=it % 3 == 0)


@pytest.mark.gpu
@pytest.mark.parametrize("pcol,consts", [(0, [0, -1, 2**32 - 1]), (1, [2**63, 2**63 + 7, 2**64 - 1]),
                                         (2, [_bits(0.0), _bits(math.nan), _bits(-1e300)]), (3, [0, 1, 1])],
                         ids=["int64", "uint64", "double", "boolean"])
def test_multi_predicate_on_each_type(ctx, pcol, consts):
    rng = np.random.default_rng(300 + pcol)
    for i, op in enumerate(OPS):
        run_multi(ctx, rng, ("dict", "plain"), 2, 20001, "random", 500, 500 if i % 2 else 0, device=i == 3,
                  nan=pcol == 2, predicate=(pcol, op, consts[i % len(consts)]))


@pytest.mark.gpu
def test_multi_all_null_group_and_nothing_passes(ctx):
    from ytsaurus_b200 import Column
    k = np.asarray([5, 5, 6, 6, 5], dtype=np.uint64)
    v = np.asarray([1, 2, 3, 4, 5], dtype=np.uint64)
    vn = np.asarray([0, 0, 1, 1, 0], dtype=bool)
    aggs = [(AGG_SUM, 0), (AGG_MIN, 0), (AGG_MAX, 0), (AGG_AVG, 0), (AGG_FIRST, 0), (AGG_COUNT, 0), (AGG_ARGMIN, 0, 0)]
    for hint in (0, 2):
        got = ctx.scan_filter_groupby_multi([Column(T.Uint64, values=k)], [Column(T.Int64, values=v, null_bitmap=_bm(vn))], aggs,
                                            group_count_hint=hint)
        assert got["keys"][0].tolist() == [5, 6] and got["count"].tolist() == [3, 2]
        assert [x[1] for x in got["value_null"]] == [1, 1, 1, 1, 1, 0, 1] and got["values"][5].tolist() == [3, 0]
        assert [int(x[0]) for x in got["values"][:3]] == [8, 1, 5]
    got = ctx.scan_filter_groupby_multi([Column(T.Uint64, values=k)], [Column(T.Int64, values=v, null_bitmap=_bm(vn))], aggs,
                                        predicate=(capi.CMP_GT, 100), predicate_column=0)
    assert len(got["count"]) == 0 and all(len(x) == 0 for x in got["values"])


@pytest.mark.gpu
def test_multi_limits(ctx):
    """8 key columns and 32 aggregates are accepted; 9 keys, 33 aggregates and SUM / AVG over a Boolean are refused."""
    from ytsaurus_b200 import Column
    rng = np.random.default_rng(41)
    run_multi(ctx, rng, ("plain", "dict"), 8, 5001, "random", 100, 0, device=False)
    k = Column(T.Int64, values=np.arange(4, dtype=np.uint64) % 2)
    v = Column(T.Int64, values=np.arange(4, dtype=np.uint64))
    b = bool_column(np.asarray([1, 0, 1, 1]), np.zeros(4, bool), 0, rng)
    for args, code in (((([k] * 9), [v], [(AGG_SUM, 0)]), capi.ERR_INVALID_ARGUMENT),
                       (([k], [v], [(AGG_COUNT, 0)] * 33), capi.ERR_INVALID_ARGUMENT),
                       (([k], [v, b], [(AGG_SUM, 1)]), capi.ERR_UNSUPPORTED),
                       (([k], [v, b], [(AGG_AVG, 1)]), capi.ERR_UNSUPPORTED)):
        with pytest.raises(capi.YtGpuError) as e:
            ctx.scan_filter_groupby_multi(*args)
        assert e.value.code == code
    got = ctx.scan_filter_groupby_multi([k] * 8, [v], [(AGG_COUNT, 0)] * 32)
    assert got["count"].tolist() == [2, 2] and all(x.tolist() == [2, 2] for x in got["values"])


@pytest.mark.gpu
def test_multi_signed_zeros_and_nan(ctx):
    """MIN / MAX over {+0.0, -0.0} and {1.0, NaN} in both row orders: the kernel's total order, whatever the order of rows;
    ARGMIN / ARGMAX by a double: -0.0 and +0.0 are equal there, the first row wins."""
    from ytsaurus_b200 import Column
    z, nz, nan, one = _bits(0.0), _bits(-0.0), _bits(math.nan), _bits(1.0)
    keys = np.asarray([1, 1, 2, 2, 3, 3, 4, 4], dtype=np.uint64)
    vals = np.asarray([z, nz, nz, z, one, nan, nan, one], dtype=np.uint64)
    arg = np.arange(8, dtype=np.uint64)
    aggs = [(AGG_MIN, 0), (AGG_MAX, 0), (AGG_ARGMIN, 1, 0), (AGG_ARGMAX, 1, 0)]
    for hint in (0, 4):
        got = ctx.scan_filter_groupby_multi([Column(T.Uint64, values=keys)], [Column(T.Double, values=vals), Column(T.Int64, values=arg)],
                                            aggs, group_count_hint=hint)
        assert got["values"][0].tolist() == [nz, nz, one, one]
        assert got["values"][1].tolist() == [z, z, 0x7ff8000000000000, 0x7ff8000000000000]
        assert got["values"][2].tolist() == [0, 2, 4, 7] and got["values"][3].tolist() == [0, 2, 5, 6]
        want = oracle.groupby_multi([keys], None, [vals, arg], None, [T.Double, T.Int64], aggs, style=oracle.MINMAX_YQL)
        assert want["values"][2].tolist() == [0, 2, 4, 7] and want["values"][3].tolist() == [0, 2, 5, 6]
        for a in (0, 1):
            assert all(same_extremum(g, w, True) for g, w in zip(got["values"][a], want["values"][a]))
