"""The columnar chunk writers and readers at the edges random data does not reach.

The integer writer (ytgpu_encode_integer_column), the string writer (ytgpu_encode_string_column), the string value ids of
string GROUP BY / JOIN keys (ytgpu_string_value_ids) and the readers (ytgpu_decode_column / _typed over bit-packed vectors,
ytgpu_decode_string_segment) are checked byte for byte against the oracle at every bit width, at segment cuts on and next
to every limit, at ties between the four layout size estimates, and on values built to share the writers' hash-table
fingerprint and start bucket, so that only the value compare behind a slot tells them apart.

Every constructed case asserts its own premise (the layout the oracle chose, the width reached, the shared fingerprint and
bucket under the table size of that call), so that a change to the format or the hashing cannot leave a case testing
nothing.  The hash restatements are pinned to the CUDA sources by name at the end of the file."""
import functools
import importlib.util
import os
import re

import numpy as np
import pytest

import oracle
from oracle import SEGMENT_DICTIONARY_DENSE, SEGMENT_DICTIONARY_RLE, SEGMENT_DIRECT_DENSE, SEGMENT_DIRECT_RLE

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "ytsaurus_b200", "csrc")
U64 = 2**64
LAYOUTS = (SEGMENT_DICTIONARY_RLE, SEGMENT_DICTIONARY_DENSE, SEGMENT_DIRECT_RLE, SEGMENT_DIRECT_DENSE)  # enum order


def _load(name):
    """A sibling test module's helpers, loaded by path so no import mode matters."""
    spec = importlib.util.spec_from_file_location("_codec_edges_" + name[:-3], os.path.join(HERE, name))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


IW = _load("test_column_writer.py")         # _split_parts, _check_roundtrip, _assert_same_encoding, _zigzag, _unzigzag
SW = _load("test_string_column_writer.py")  # _gpu_read_back


# ---------------------------------------------------------------------------------------------------------------- model
def width_of(v: int) -> int:
    return int(v).bit_length()


def packed_bytes(max_value: int, count: int) -> int:
    return 8 * (1 + ((width_of(max_value) * count + 63) >> 6))


def i32(x: int) -> int:
    return ((int(x) + 2**31) % 2**32) - 2**31


def first_minimum(sizes) -> int:
    sizes = [i32(s) for s in sizes]
    return sizes.index(min(sizes))


def div_round(num: int, den: int) -> int:
    """DivRound<int> of the offsets' expected length."""
    return num // den + (1 if num % den >= (den + 1) // 2 else 0)


def integer_sizes(enc, nulls, chunk_rows):
    """The integer writer's four size estimates for one segment of encoded (zig-zag for signed) values, enum order."""
    enc = np.asarray(enc, dtype=np.uint64)
    nulls = np.asarray(nulls, dtype=bool)
    live = enc[~nulls]
    count = len(enc)
    vmin, vmax = (int(live.min()), int(live.max())) if len(live) else (U64 - 1, 0)
    rng_ = (vmax - vmin) % U64  # 1 for a segment without values, as the reference has it
    nd = len(np.unique(live))
    vals = np.where(nulls, np.uint64(0), enc)
    runs = 1 + int(((nulls[1:] != nulls[:-1]) | (vals[1:] != vals[:-1])).sum()) if count else 0
    return [packed_bytes(rng_, nd) + packed_bytes(nd + 1, runs) + packed_bytes(chunk_rows, runs),
            packed_bytes(rng_, nd) + packed_bytes(nd + 1, count),
            packed_bytes(rng_, runs) + packed_bytes(chunk_rows, runs) + runs // 8,
            packed_bytes(rng_, count) + count // 8]


def string_sizes(values):
    """The string writer's four size estimates for one segment (list of bytes / None), enum order."""
    count = len(values)
    live = [v for v in values if v is not None]
    dictionary = list(dict.fromkeys(live))
    dsize = len(dictionary)
    dict_bytes = sum(len(v) for v in dictionary)
    direct_bytes = sum(len(v) for v in live)
    max_len = max((len(v) for v in dictionary), default=0)
    starts = [i for i in range(count) if i == 0 or values[i] != values[i - 1]]
    runs = len(starts)
    rle_bytes = sum(len(values[i]) for i in starts if values[i] is not None)
    return [dict_bytes + packed_bytes(max_len, dsize) + packed_bytes(dsize + 1, runs) + packed_bytes(count, runs),
            dict_bytes + packed_bytes(max_len, dsize) + packed_bytes(dsize + 1, count),
            rle_bytes + packed_bytes(max_len, runs) + packed_bytes(count, runs) + count // 8,
            direct_bytes + packed_bytes(max_len, count) + count // 8]


# mix64 (the finaliser of both writers' tables): x ^= x >> 33 is its own inverse, and the odd multiplier has an inverse mod 2^64
MIX_MUL = 0xff51afd7ed558ccd
MIX_INV = pow(MIX_MUL, -1, U64)
FNV_BASIS, FNV_PRIME = 0xcbf29ce484222325, 0x100000001b3


def mix64(x: int) -> int:
    x ^= x >> 33
    x = (x * MIX_MUL) % U64
    return x ^ (x >> 33)


def unmix64(y: int) -> int:
    y ^= y >> 33
    y = (y * MIX_INV) % U64
    return y ^ (y >> 33)


def table_cap(rows: int) -> int:
    """Slots of a writer's table for `rows` rows: a power of two >= 2 x rows, at least 8."""
    cap = 8
    while cap < 2 * rows:
        cap <<= 1
    return cap


def int_slot(e: int, cap: int):
    """-> (fingerprint, start bucket) of an encoded integer value."""
    mx = mix64(e)
    return mx >> 32, mx & (cap - 1)


def colliding_integers(count: int, fp: int, bucket: int, cap_bits: int):
    """`count` distinct encoded values whose mix64 has fingerprint fp and start bucket `bucket` under any table of at most
    2^cap_bits slots."""
    return [unmix64((fp << 32) | (j << cap_bits) | bucket) for j in range(1, count + 1)]


def fnv_mix(s: bytes) -> int:
    h = FNV_BASIS ^ len(s)
    for b in s:
        h = ((h ^ b) * FNV_PRIME) % U64
    return mix64(h)


def string_slot(s: bytes, cap: int):
    mx = fnv_mix(s)
    return mx >> 32, mx & (cap - 1)


@functools.lru_cache(maxsize=None)
def colliding_string_pairs(bucket_bits: int = 4, count: int = 2**21, seed: int = 7):
    """Birthday search over `count` random 8-byte strings: pairs of distinct strings whose FNV-1a + mix64 hash shares the
    32-bit fingerprint and the low `bucket_bits` bits (the start bucket of any table of at most 2^bucket_bits slots)."""
    rng = np.random.default_rng(seed)
    raw = rng.integers(0, 256, (count, 8), dtype=np.uint8)
    with np.errstate(over="ignore"):
        h = np.full(count, FNV_BASIS ^ 8, dtype=np.uint64)
        for k in range(8):
            h = (h ^ raw[:, k].astype(np.uint64)) * np.uint64(FNV_PRIME)
        h ^= h >> np.uint64(33)
        h *= np.uint64(MIX_MUL)
        h ^= h >> np.uint64(33)
    order = np.argsort(h >> np.uint64(32), kind="stable")
    fp = (h >> np.uint64(32))[order]
    same = np.nonzero(fp[1:] == fp[:-1])[0]
    mask = np.uint64((1 << bucket_bits) - 1)
    pairs = []
    for i in same:
        a, b = order[i], order[i + 1]
        if (h[a] & mask) == (h[b] & mask) and raw[a].tobytes() != raw[b].tobytes():
            pairs.append((raw[a].tobytes(), raw[b].tobytes()))
    return tuple(pairs)


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_mix64_inverse_builds_colliding_integers():
    rng = np.random.default_rng(1)
    for y in [0, 1, U64 - 1, 2**63, *[int(x) for x in rng.integers(0, 2**63, 50, dtype=np.uint64)]]:
        assert mix64(unmix64(y)) == y and unmix64(mix64(y)) == y
    for cap_bits, bucket in ((3, 7), (13, 0), (18, 12345)):
        vals = colliding_integers(6, 0x9e3779b9, bucket, cap_bits)
        assert len(set(vals)) == 6
        for cap in (8, 1 << cap_bits):
            assert {int_slot(v, cap) for v in vals} == {(0x9e3779b9, bucket & (cap - 1))}


def test_birthday_search_finds_string_collisions():
    pairs = colliding_string_pairs()
    assert len(pairs) >= 8
    for a, b in pairs:
        assert a != b and len(a) == len(b) == 8
        for cap in (8, 16):
            assert string_slot(a, cap) == string_slot(b, cap)


def _random_int_segment(rng):
    n = int(rng.integers(1, 40))
    pool = rng.integers(0, 2**int(rng.integers(1, 64)), int(rng.integers(1, 6)), dtype=np.uint64)
    vals, nulls = [], []
    while len(vals) < n:
        k = int(rng.integers(1, 8))
        nl = rng.random() < 0.2
        vals += [int(pool[int(rng.integers(0, len(pool)))])] * k
        nulls += [nl] * k
    return np.asarray(vals[:n], dtype=np.uint64), np.asarray(nulls[:n], dtype=np.uint8), int(rng.integers(0, 3)) * int(rng.integers(0, 2**20))


def _random_string_segment(rng):
    n = int(rng.integers(1, 30))
    pool = [bytes(rng.integers(97, 100, int(rng.integers(0, 12)), dtype=np.uint8)) for _ in range(int(rng.integers(1, 6)))]
    vals = []
    while len(vals) < n:
        v = None if rng.random() < 0.15 else pool[int(rng.integers(0, len(pool)))]
        vals += [v] * int(rng.integers(1, 6))
    return vals[:n]


def test_size_estimates_restate_the_oracle():
    rng = np.random.default_rng(3)
    for _ in range(400):
        vals, nulls, off = _random_int_segment(rng)
        _, segs = oracle.encode_integer_column(vals, nulls, chunk_row_offset=off)
        assert int(segs[0]["type"]) == first_minimum(integer_sizes(vals, nulls, off + len(vals)))
        values = _random_string_segment(rng)
        data, segs = SW._encode(values)
        assert int(segs[0]["type"]) == first_minimum(string_sizes(values))


@functools.lru_cache(maxsize=None)
def integer_ties(count: int = 24, seed: int = 4):
    """Random small segments whose smallest size estimate is shared by two or more layouts."""
    rng = np.random.default_rng(seed)
    found = []
    for _ in range(200000):
        vals, nulls, off = _random_int_segment(rng)
        sizes = [i32(s) for s in integer_sizes(vals, nulls, off + len(vals))]
        if sizes.count(min(sizes)) > 1:
            found.append((vals, nulls, off, sizes))
            if len(found) == count:
                break
    return found


@functools.lru_cache(maxsize=None)
def string_ties(count: int = 24, seed: int = 5):
    rng = np.random.default_rng(seed)
    found = []
    for _ in range(200000):
        values = _random_string_segment(rng)
        sizes = [i32(s) for s in string_sizes(values)]
        if sizes.count(min(sizes)) > 1:
            found.append((values, sizes))
            if len(found) == count:
                break
    return found


def test_layout_ties_take_the_first_minimum_in_the_oracle():
    ties = integer_ties()
    assert len(ties) == 24
    for vals, nulls, off, sizes in ties:
        _, segs = oracle.encode_integer_column(vals, nulls, chunk_row_offset=off)
        assert int(segs[0]["type"]) == sizes.index(min(sizes))
    sties = string_ties()
    assert len(sties) == 24
    for values, sizes in sties:
        _, segs = SW._encode(values)
        assert int(segs[0]["type"]) == sizes.index(min(sizes))


# integer columns whose every segment spans exactly 2^w values in one layout --------------------------------------------
WIDTH_ROWS = 2048
SHAPES = [(nd, run, alt) for nd in (2048, 64, 16, 4, 2, 1) for run in (1, 15, 32, 128) for alt in (False, True)]


def _shaped_segment(w, nd, run, alt, m, rng):
    """m encoded values (and nulls) spanning exactly [lo, lo + 2^w - 1]: runs of `run` rows cycling through nd values,
    every other run NULL when `alt`."""
    span = 1 << w
    # odd widths end at 2^64 - 2 (zig-zag INT64_MAX), width 64 ends at 2^64 - 1 (INT64_MIN), even widths lie anywhere
    lo = U64 - 1 - span if w % 2 else int(rng.integers(0, U64 - span, dtype=np.uint64, endpoint=True))
    nd = min(nd, span)
    pool = [lo, lo + span - 1][:nd]
    seen = set(pool)
    while len(pool) < nd:
        v = lo + int(rng.integers(0, span - 1, dtype=np.uint64, endpoint=True))
        if v not in seen:
            seen.add(v)
            pool.append(v)
    enc, nulls = [], []
    r = 0
    while len(enc) < m:
        nl = alt and r % 2 == 1
        v = pool[(r // 2 if alt else r) % nd]
        enc += [0 if nl else v] * run
        nulls += [nl] * run
        r += 1
    enc, nulls = enc[:m], nulls[:m]
    live = [e for e, nl in zip(enc, nulls) if not nl]
    assert min(live) == lo and max(live) == lo + span - 1  # the width is reached
    return enc, nulls


@functools.lru_cache(maxsize=None)
def width_columns(layout, seed, chunk_row_offset):
    """-> (encoded values, nulls, widths): one WIDTH_ROWS-row segment per width 0..64 that the estimates let `layout` win."""
    rng = np.random.default_rng(seed)
    enc, nulls, widths = [], [], []
    for w in range(65):
        chunk_rows = chunk_row_offset + (len(widths) + 1) * WIDTH_ROWS
        for nd, run, alt in SHAPES:
            if nd < min(2, 1 << w):
                continue  # both ends of the range take two values
            e, nl = _shaped_segment(w, nd, run, alt, WIDTH_ROWS, rng)
            if first_minimum(integer_sizes(e, nl, chunk_rows)) == layout:
                enc += e
                nulls += nl
                widths.append(w)
                break
    return np.asarray(enc, dtype=np.uint64), np.asarray(nulls, dtype=np.uint8), widths


# widths the size estimates leave to each layout: DictionaryDense never beats DirectDense below width 2 (its ids take two
# bits a row where DirectDense takes one value bit and one NULL bit), nor DictionaryRle DirectRle for the same reason
REACHABLE_WIDTHS = {
    SEGMENT_DIRECT_DENSE: set(range(65)),
    SEGMENT_DIRECT_RLE: set(range(65)),
    SEGMENT_DICTIONARY_DENSE: set(range(2, 65)),
    SEGMENT_DICTIONARY_RLE: set(range(2, 65)),
}


@pytest.mark.parametrize("layout", LAYOUTS)
def test_width_columns_reach_every_width_in_the_oracle(layout):
    enc, nulls, widths = width_columns(layout, 10 + layout, 1000)
    assert set(widths) >= REACHABLE_WIDTHS[layout]
    for signed in (False, True):
        vals = IW._unzigzag(enc) if signed else enc
        data, segs = oracle.encode_integer_column(vals, nulls, signed=signed, max_segment_values=WIDTH_ROWS, chunk_row_offset=1000)
        assert segs["type"].tolist() == [layout] * len(widths)
        assert segs["values_width"].tolist() == widths
        IW._check_roundtrip(data, segs, vals, nulls, signed)


# ---------------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def ctx():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from ytsaurus_b200 import GpuContext
    c = GpuContext(0)
    yield c
    c.close()


def _to_device(a):
    import torch
    if a is None:
        return None
    a = np.ascontiguousarray(a)
    view = {np.dtype(np.uint64): np.int64, np.dtype(np.uint32): np.int32}.get(a.dtype)
    return torch.from_numpy(a.view(view) if view else a).cuda()


def _host(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def _int_same(ctx, vals, nulls, name, signed=False, max_segment_values=128 * 1024, chunk_row_offset=0):
    """Both memory flavours of the integer writer against the oracle, byte for byte -> (oracle data, segments)."""
    want = oracle.encode_integer_column(vals, nulls, signed=signed, max_segment_values=max_segment_values,
                                        chunk_row_offset=chunk_row_offset)
    for device in (False, True):
        v = _to_device(np.ascontiguousarray(vals).view(np.uint64)) if device else vals
        nl = _to_device(nulls) if device else nulls
        data, segs = ctx.encode_integer_column(v, nl, signed=signed, max_segment_values=max_segment_values,
                                               chunk_row_offset=chunk_row_offset)
        IW._assert_same_encoding(_host(data), segs, *want, name=(name, "device" if device else "host"))
    return want


def _gpu_decode_segment(ctx, data, seg, signed):
    """One integer segment through the product's reader, its parts as TColumn views -> (values u64, null bytemap)."""
    from ytsaurus_b200 import Column
    from ytsaurus_b200.rowset import EValueType as T
    n = int(seg["row_count"])
    p = IW._split_parts(data, seg)
    t = int(seg["type"])
    kw = dict(value_type=T.Int64 if signed else T.Uint64, base_value=int(seg["min_value"]), zigzag=signed, bit_width=0,
              value_count=n, values=p[0].copy())
    if t in (SEGMENT_DIRECT_DENSE, SEGMENT_DIRECT_RLE):
        kw["null_bitmap"] = p[1].view(np.uint8).copy()
    else:
        kw["dictionary_indexes"] = oracle.bit_unpack(p[1]).astype(np.uint32)
    if t in (SEGMENT_DIRECT_RLE, SEGMENT_DICTIONARY_RLE):
        kw["rle_indexes"] = oracle.bit_unpack(p[2])
    return ctx.decode_column(Column(**kw))


def _gpu_read_back_integers(ctx, data, segs, vals, nulls, signed):
    at = 0
    for s in segs:
        n = int(s["row_count"])
        got, gn = _gpu_decode_segment(ctx, data, s, signed)
        wn = np.zeros(n, np.uint8) if nulls is None else nulls[at:at + n]
        want = np.where(wn.astype(bool), 0, np.ascontiguousarray(vals[at:at + n]).view(np.uint64))
        assert (gn == wn).all(), (at, int(s["type"]))
        assert (np.where(wn.astype(bool), 0, got) == want).all(), (at, int(s["type"]), int(s["values_width"]))
        at += n
    assert at == len(vals)


# 1. integer writer ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("signed", [False, True])
@pytest.mark.parametrize("layout", LAYOUTS)
def test_gpu_integer_every_width_in_every_layout(ctx, layout, signed):
    enc, nulls, widths = width_columns(layout, 10 + layout, 1000)
    assert set(widths) >= REACHABLE_WIDTHS[layout]
    vals = IW._unzigzag(enc) if signed else enc
    data, segs = _int_same(ctx, vals, nulls, (layout, signed), signed=signed, max_segment_values=WIDTH_ROWS, chunk_row_offset=1000)
    assert segs["type"].tolist() == [layout] * len(widths) and segs["values_width"].tolist() == widths
    if signed:
        assert {-2**63, 2**63 - 1} <= set(vals[~nulls.astype(bool)].tolist())
    _gpu_read_back_integers(ctx, data, segs, vals, nulls, signed)


def _ids_and_rows_cases():
    """(name, values, nulls, max_segment_values, chunk_row_offset): dictionary sizes and last run starts around powers of
    two, and a chunk row count whose width grows inside the column."""
    rng = np.random.default_rng(17)
    cases = []
    for k in range(1, 11):
        for nd in (2**k - 2, 2**k - 1, 2**k):
            if nd < 1:
                continue
            pool = rng.integers(0, 2**62, nd, dtype=np.uint64)
            dense = np.concatenate([pool, pool[rng.integers(0, nd, 3 * nd + 5)]])             # every value, then repeats
            cases.append((f"dense-nd{nd}", dense, None, len(dense), 0))
            runs = np.repeat(np.concatenate([pool, pool[rng.integers(0, nd, nd)]]), 40)     # long runs, revisited values
            cases.append((f"rle-nd{nd}", runs, None, len(runs), 0))
        for last in (2**k - 1, 2**k, 2**k + 1):                                           # the last run starts at row `last`
            v = np.zeros(last + 3, np.uint64)
            v[last:] = 5
            cases.append((f"last-run-{last}", v, None, len(v), 0))
            nl = np.zeros(last + 3, np.uint8)
            nl[last:] = 1                                                                 # ... as a run of NULLs
            cases.append((f"last-null-run-{last}", np.full(last + 3, 9, np.uint64), nl, len(v), 0))
    # segments of 1000 rows from chunk row 2^16 - 2500: width_of(chunk_rows) goes from 16 to 17 at the third segment
    v = np.repeat(rng.integers(0, 50, 80, dtype=np.uint64), 50)
    cases.append(("chunk-rows-cross-2^16", v, None, 1000, 2**16 - 2500))
    v = np.repeat(rng.integers(0, 3, 400, dtype=np.uint64), 10)
    cases.append(("chunk-rows-cross-2^32", v, None, 512, 2**32 - 1500))
    return cases


@pytest.mark.gpu
def test_gpu_integer_dictionary_ids_and_row_indexes_at_powers_of_two(ctx):
    seen = set()
    for name, vals, nulls, m, off in _ids_and_rows_cases():
        data, segs = _int_same(ctx, vals, nulls, name, max_segment_values=m, chunk_row_offset=off)
        for s in segs:
            t = int(s["type"])
            seen.add((t, int(s["ids_width"]), int(s["row_indexes_width"])))
            if t in (SEGMENT_DICTIONARY_DENSE, SEGMENT_DICTIONARY_RLE):
                assert int(s["ids_width"]) == width_of(int(s["values_size"]) + 1)
        if name.startswith("chunk-rows"):
            w = [width_of(int(c)) for c in segs["chunk_row_count"]]
            assert w[0] < w[-1], name  # the premise: the width of chunk_rows grows inside the column
        _gpu_read_back_integers(ctx, data, segs, vals, nulls, False)
    widths = {(t, iw) for t, iw, _ in seen}
    # the id vectors crossed every width 3..11 in both dictionary layouts
    for t in (SEGMENT_DICTIONARY_DENSE, SEGMENT_DICTIONARY_RLE):
        assert {iw for tt, iw in widths if tt == t} >= set(range(3, 12)), t
    assert {rw for t, _, rw in seen if t in (SEGMENT_DIRECT_RLE, SEGMENT_DICTIONARY_RLE)} >= set(range(6, 12))


GRID = [(m, n) for m in (1, 2, 3, 63, 64, 65, 2047, 2048, 2049, 131072) for n in (m - 1, m, m + 1, 3 * m + 1) if n > 0]


@pytest.mark.gpu
@pytest.mark.parametrize("m,n", GRID)
def test_gpu_integer_segment_grid(ctx, m, n):
    rng = np.random.default_rng(m * 7 + n)
    # runs of a few hundred distinct values, with NULL runs: every segment gets runs, repeats and a dictionary
    pool = rng.integers(-2**40, 2**40, 300)
    lens = rng.integers(1, 9, n)
    vals = np.repeat(pool[rng.integers(0, len(pool), n)], lens)[:n].astype(np.int64)
    nulls = np.repeat((rng.random(n) < 0.1).astype(np.uint8), lens)[:n]
    data, segs = _int_same(ctx, vals, nulls, (m, n), signed=True, max_segment_values=m, chunk_row_offset=3)
    assert len(segs) == (n + m - 1) // m
    _gpu_read_back_integers(ctx, data, segs, vals, nulls, True)


@pytest.mark.gpu
def test_gpu_integer_layout_ties_take_the_first_minimum(ctx):
    for vals, nulls, off, sizes in integer_ties():
        data, segs = _int_same(ctx, vals, nulls, sizes, chunk_row_offset=off)
        assert int(segs[0]["type"]) == sizes.index(min(sizes))
    assert len({tuple(i for i, s in enumerate(sz) if s == min(sz)) for *_, sz in integer_ties()}) >= 2  # several kinds of tie


@pytest.mark.gpu
def test_gpu_string_layout_ties_take_the_first_minimum(ctx):
    for values, sizes in string_ties():
        _, segs = _string_same(ctx, values, sizes)
        assert int(segs[0]["type"]) == sizes.index(min(sizes))
    assert len({tuple(i for i, s in enumerate(sz) if s == min(sz)) for _, sz in string_ties()}) >= 2


def _first_seen_after_later_blocks(first, filler, rows, rng):
    """A column of `rows` rows (a multiple of 2048) whose values `first` are first seen, in that order, at the end of the
    first 2048-row block, and which open every later block in the reverse order: a later block's thread claims each value's
    slot before the thread of its first row gets there, so only the lowering of the row decides the first-seen order."""
    col = list(filler[rng.integers(0, len(filler), rows)])
    col[2048 - len(first):2048] = first
    for b in range(2048, rows, 2048):
        col[b:b + len(first)] = first[::-1]
    return col


@pytest.mark.gpu
@pytest.mark.parametrize("signed", [False, True])
def test_gpu_integer_colliding_fingerprints_stay_distinct(ctx, signed):
    rng = np.random.default_rng(23)
    # one segment of 4096 rows (two stats blocks, 8192 slots); the last slot so that the probe wraps around
    rows = 4096
    cap = table_cap(rows)
    group = colliding_integers(6, 0x1234abcd, cap - 1, 14)
    assert len({int_slot(e, cap) for e in group}) == 1 and len(set(group)) == 6
    filler = np.asarray(rng.integers(0, 2**63, 10, dtype=np.uint64), dtype=np.uint64)
    cases = []
    enc = np.asarray(_first_seen_after_later_blocks(group, filler, rows, rng), dtype=np.uint64)
    cases.append(("late-first-rows", enc, rows, SEGMENT_DICTIONARY_DENSE))
    # two segments of 4096 rows that see the group in opposite orders
    enc2 = np.concatenate([enc, np.asarray(_first_seen_after_later_blocks(group[::-1], filler, rows, rng), dtype=np.uint64)])
    cases.append(("two-segments", enc2, rows, SEGMENT_DICTIONARY_DENSE))
    # runs of the group: DictionaryRle
    enc3 = np.repeat(np.asarray([group[i % 6] for i in (0, 1, 2, 3, 4, 5, 3, 0, 5, 1)] * 8, dtype=np.uint64), 50)
    cases.append(("runs", enc3, len(enc3), SEGMENT_DICTIONARY_RLE))
    # a 4-row segment whose table has 8 slots: the whole group in one bucket, the probe wraps at slot 7
    tiny_group = colliding_integers(4, 0x0badf00d, 7, 3)
    assert len({int_slot(e, table_cap(4)) for e in tiny_group}) == 1
    enc4 = np.asarray([tiny_group[i] for i in (2, 0, 2, 1, 3, 0, 1, 2)] * 4, dtype=np.uint64)
    cases.append(("tiny", enc4, 4, None))
    for name, enc, m, layout in cases:
        vals = IW._unzigzag(enc) if signed else enc
        data, segs = _int_same(ctx, vals, None, name, signed=signed, max_segment_values=m)
        if layout is not None:
            assert segs["type"].tolist() == [layout] * len(segs), name
        for s in segs:
            part = enc[int(s["chunk_row_count"]) - int(s["row_count"]):int(s["chunk_row_count"])]
            if int(s["type"]) in (SEGMENT_DICTIONARY_DENSE, SEGMENT_DICTIONARY_RLE):
                assert int(s["values_size"]) == len(set(part.tolist())), name  # no two colliding values merged
        _gpu_read_back_integers(ctx, data, segs, vals, None, signed)


@pytest.mark.gpu
def test_gpu_integer_null_patterns(ctx):
    rng = np.random.default_rng(29)
    n, m = 4 * 2048 + 130, 2048
    vals = rng.integers(0, 40, n).astype(np.uint64)
    nulls = np.zeros(n, np.uint8)
    nulls[0] = nulls[-1] = 1                       # first and last row
    nulls[m:2 * m] = 1                             # an all-NULL segment between non-NULL ones
    nulls[3 * m - 100:3 * m + 77] = 1              # a NULL run across a segment edge
    nulls[4 * m - 3:4 * m + 2] = 1                 # ... and across the next one, a few rows on each side
    nulls[63] = nulls[64] = nulls[127] = nulls[128] = 1   # bits 63 and 64 of the bitmap words
    nulls[2 * m + 63] = nulls[2 * m + 64] = 1
    for signed in (False, True):
        data, segs = _int_same(ctx, vals, nulls, "nulls", signed=signed, max_segment_values=m, chunk_row_offset=9)
        assert int(segs[1]["values_size"]) in (0, 1) and int(segs[1]["row_count"]) == m
        _gpu_read_back_integers(ctx, data, segs, vals.view(np.int64) if signed else vals, nulls, signed)
    # a dense layout with the bitmap words in play: every value distinct
    vals = rng.integers(0, 2**60, n, dtype=np.uint64)
    data, segs = _int_same(ctx, vals, nulls, "dense-nulls", max_segment_values=m)
    assert int(segs[0]["type"]) == SEGMENT_DIRECT_DENSE
    _gpu_read_back_integers(ctx, data, segs, vals, nulls, False)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
def test_gpu_reader_windows_on_every_packed_width(ctx, device):
    """decode_column / decode_column_typed over bit-packed vectors of every width, in windows that start at 0, 1, 63, 64
    and 65 and end on the last value; device vectors are exactly the packed size."""
    from ytsaurus_b200 import Column
    from ytsaurus_b200.rowset import EValueType as T
    rng = np.random.default_rng(31)
    count = 200
    for w in range(65):
        top = (1 << w) - 1
        raw = rng.integers(0, top, count, dtype=np.uint64, endpoint=True) if w else np.zeros(count, np.uint64)
        raw[::7] = top                             # every value that spills into the next word has its top bit set
        packed = oracle.bit_pack(raw, top)
        assert int(packed[0]) >> 56 == w and len(packed) == 1 + (w * count + 63) // 64
        bitmap = np.packbits((rng.random(count) < 0.2).astype(np.uint8), bitorder="little")
        for start in (0, 1, 63, 64, 65):
            for zigzag, base, vt in ((False, 0, T.Uint64), (True, 3, T.Int64), (False, 2**63 + 5, T.Uint64)):
                vec = _to_device(packed) if device else packed
                bm = _to_device(bitmap) if device else bitmap
                col = Column(vt, values=vec, bit_width=0, start_index=start, value_count=count - start, base_value=base,
                             zigzag=zigzag, null_bitmap=bm)
                want = oracle.decode_integer_vector(start, count, base, zigzag, raw, bitmap=bitmap)
                want_null = oracle.build_null_bytemap(0, start, count, bitmap=bitmap)
                got, gn = ctx.decode_column(col)
                assert (_host(got).view(np.uint64) == want).all(), (w, start, zigzag)
                assert (_host(gn) == want_null).all(), (w, start)
                if zigzag or base:
                    continue
                for eb, dt in ((1, np.uint8), (2, np.uint16), (4, np.uint32), (8, np.uint64)):
                    got, gn = ctx.decode_column_typed(col, eb)
                    got = _host(got).view(dt)
                    assert (got == want.astype(dt)).all(), (w, start, eb)  # narrowed by assignment; NULL rows read 0


# 2. string writer, reader and value ids -------------------------------------------------------------------------------
def _string_same(ctx, values, name, device=(False, True), **kw):
    """The string writer against the oracle in both memory flavours, byte for byte, and read back through
    ytgpu_decode_string_segment -> (data, segments)."""
    heap, starts, lengths, nulls = oracle.flatten_strings(values)
    return _string_same_flat(ctx, heap, starts, lengths, nulls, values, name, device=device, **kw)


def _string_same_flat(ctx, heap, starts, lengths, nulls, values, name, device=(False, True), **kw):
    want_data, want_segs = oracle.encode_string_column(heap, starts, lengths, nulls, **kw)
    for dev in device:
        args = [_to_device(x) for x in (heap, starts, lengths, nulls)] if dev else (heap, starts, lengths, nulls)
        data, segs = ctx.encode_string_column(*args, **kw)
        assert segs.tobytes() == want_segs.tobytes(), (name, dev, segs, want_segs)
        got = _host(data)
        for w in want_segs:  # the bytes between the 8-byte aligned segments are the container's own
            a, b = int(w["data_offset"]), int(w["data_offset"] + w["data_bytes"])
            assert got[a:b].tobytes() == want_data[a:b].tobytes(), (name, dev)
    if values is not None:
        assert SW._gpu_read_back(ctx, got, want_segs) == values, name
    return got, want_segs


def _distinct(count, length, rng, prefix=b""):
    out = set()
    while len(out) < count:
        out.add(prefix + bytes(rng.integers(0, 256, length, dtype=np.uint8)))
    return sorted(out)


@pytest.mark.gpu
def test_gpu_string_buffer_rule_edges(ctx):
    ten = [bytes([65 + i]) * 10 for i in range(26)]
    # exactly max_buffer bytes: no cut; one byte more: the value that crosses the limit ends the segment
    _, segs = _string_same(ctx, ten[:7], "exact", max_buffer_bytes=30)
    assert segs["row_count"].tolist() == [4, 3]
    _, segs = _string_same(ctx, ten[:7], "plus-one", max_buffer_bytes=29)
    assert segs["row_count"].tolist() == [3, 3, 1]
    vals = [b"x" * 9] * 3 + [b"x" * 3] + [b"y" * 30]
    _, segs = _string_same(ctx, vals, "exact-then-over", max_buffer_bytes=30)
    assert segs["row_count"].tolist() == [5]
    # a buffer cut on the same row as a max_values cut
    _, segs = _string_same(ctx, ten[:9], "both-cuts", max_buffer_bytes=25, max_segment_values=3)
    assert segs["row_count"].tolist() == [3, 3, 3]
    # one value longer than the buffer: a segment of its own, and the buffer starts over after it
    vals = [b"a", b"b" * 100, b"c", b"d" * 40, b"e", b"f"]
    _, segs = _string_same(ctx, vals, "longer-than-buffer", max_buffer_bytes=30)
    assert segs["row_count"].tolist() == [2, 2, 2]
    # empty strings and NULLs add no bytes: they never cut, however many
    vals = [b"q" * 10, b"r" * 10] + [b"", None] * 500 + [b"s" * 10, b"", b"t" * 2, None]
    _, segs = _string_same(ctx, vals, "empty-and-null-runs", max_buffer_bytes=30)
    assert segs["row_count"].tolist() == [1005, 1]


@pytest.mark.gpu
def test_gpu_string_expected_length_rounding(ctx):
    rng = np.random.default_rng(41)
    for den in (4, 5, 8, 9):
        for rem in ((den + 1) // 2, (den + 1) // 2 - 1):
            q = 20
            lengths = [q] * den
            lengths[-1] += rem
            vals = [bytes(rng.integers(97, 123, ln, dtype=np.uint8)) for ln in lengths]
            assert len(set(vals)) == den
            _, segs = _string_same(ctx, vals, (den, rem))
            s = segs[0]
            assert int(s["type"]) == SEGMENT_DIRECT_DENSE and sum(lengths) % den == rem
            assert int(s["expected_length"]) == div_round(sum(lengths), den) == q + (rem >= (den + 1) // 2)


@pytest.mark.gpu
def test_gpu_string_every_offsets_width(ctx):
    # two distinct values a segment: lengths b + 2^(w-1) and b give the zig-zag difference 2^(w-1), width w (w >= 2);
    # b + 2 after b gives difference -1, width 1; equal lengths give width 0
    rng = np.random.default_rng(43)
    vals, want = [], []
    for w in range(25):
        b = 3
        a = b if w == 0 else (b + (1 << (w - 1)) if w >= 2 else None)
        pair = (b, b + 2) if w == 1 else (a, b)
        vals += [bytes(rng.integers(97, 123, pair[0], dtype=np.uint8)), bytes(rng.integers(97, 123, pair[1], dtype=np.uint8))]
        want.append(w)
    assert all(vals[2 * i] != vals[2 * i + 1] for i in range(25))
    _, segs = _string_same(ctx, vals, "widths", device=(False,), max_segment_values=2)
    assert segs["type"].tolist() == [SEGMENT_DIRECT_DENSE] * 25 and segs["offsets_width"].tolist() == want


@pytest.mark.gpu
def test_gpu_string_value_of_2_28_bytes(ctx):
    big = 1 << 28
    heap = np.zeros(big + 16, np.uint8)
    heap[:big] = np.arange(big, dtype=np.uint64).astype(np.uint8)
    heap[big:] = 7
    starts = np.asarray([0, big, big + 3], np.uint64)
    lengths = np.asarray([big, 0, 5], np.uint32)
    nulls = np.zeros(3, np.uint8)
    data, segs = _string_same_flat(ctx, heap, starts, lengths, nulls, None, "2^28", device=(False,), max_buffer_bytes=1 << 30)
    assert len(segs) == 1 and int(segs[0]["type"]) == SEGMENT_DIRECT_DENSE and int(segs[0]["offsets_width"]) >= 29
    st, ln, nl = ctx.decode_string_segment(data, segs[0])
    st = st.tolist()
    assert ln.tolist() == [big, 0, 5] and nl.tolist() == [0, 0, 0] and st[1] - st[0] == big and st[2] == st[1]


@pytest.mark.gpu
def test_gpu_string_dictionary_id_widths(ctx):
    rng = np.random.default_rng(47)
    for k in range(1, 9):
        for dsize in (2**k - 1, 2**k):
            if dsize < 2:
                continue  # a single value takes no dictionary
            words = _distinct(dsize, 24, rng)
            # DictionaryDense: every value, then repeats without runs; ids are packed with width_of(dsize + 1)
            order = list(range(dsize)) + [int(i) for i in rng.integers(0, dsize, 6 * dsize + 8)]
            dense = [words[i] for i in order]
            dense = [v for j, v in enumerate(dense) if j == 0 or v != dense[j - 1]]
            _, segs = _string_same(ctx, dense, ("dense", dsize))
            assert int(segs[0]["type"]) == SEGMENT_DICTIONARY_DENSE and int(segs[0]["ids_width"]) == width_of(dsize + 1)
            # DictionaryRle: long runs over the dictionary twice; ids are packed with width_of(dsize)
            runs = [words[i] for i in list(range(dsize)) * 2 for _ in range(30)]
            _, segs = _string_same(ctx, runs + [None] * 30, ("rle", dsize))
            assert int(segs[0]["type"]) == SEGMENT_DICTIONARY_RLE and int(segs[0]["ids_width"]) == width_of(dsize)


@pytest.mark.gpu
def test_gpu_string_colliding_fingerprints_stay_distinct(ctx):
    pairs = colliding_string_pairs()[:8]
    for a, b in pairs:
        for rows, order in ((8, [a, b, a, b, b, a, a, b]), (4, [b, a, b, a])):
            cap = table_cap(rows)
            assert string_slot(a, cap) == string_slot(b, cap)  # the premise under this call's table size
            vals = order * 3 + [None, a, b""] + order
            _, segs = _string_same(ctx, vals, (a, b), max_segment_values=rows)
            for s in segs[:3]:
                assert int(s["type"]) in (SEGMENT_DICTIONARY_DENSE, SEGMENT_DICTIONARY_RLE) and int(s["offsets_size"]) == 2
        # string_value_ids over a column of 8 rows (a 16-slot table): two ids, each the first row of its value
        for vals in ([a, b, a, b, None, b"", b, a], [b, b, a, a, b, None, a, b""]):
            assert string_slot(a, table_cap(len(vals))) == string_slot(b, table_cap(len(vals)))
            _check_value_ids(ctx, vals)
    # values that differ only in their last byte, embedded NULs, and b"" against NULL
    rng = np.random.default_rng(53)
    base = bytes(rng.integers(0, 256, 40, dtype=np.uint8))
    tricky = [base[:-1] + bytes([x]) for x in (0, 1, 255)] + [b"\0", b"\0\0", b"a\0b", b"a\0c", b"", None, b"a", b"a\0"]
    vals = [tricky[int(i)] for i in rng.integers(0, len(tricky), 3000)]
    _string_same(ctx, vals, "tricky", max_segment_values=700)
    _check_value_ids(ctx, vals)


def _check_value_ids(ctx, values):
    heap, starts, lengths, nulls = oracle.flatten_strings(values)
    first = {}
    want = [first.setdefault(v, i) if v is not None else 0 for i, v in enumerate(values)]
    for dev in (False, True):
        args = [_to_device(x) for x in (heap, starts, lengths, nulls)] if dev else (heap, starts, lengths, nulls)
        ids, nl = ctx.string_value_ids(*args)
        assert _host(ids).view(np.uint64).tolist() == want and _host(nl).tolist() == nulls.tolist(), (values[:8], dev)


@pytest.mark.gpu
def test_gpu_first_rows_win_when_later_blocks_claim_first(ctx):
    """The value's slot is claimed by a later 2048-row block before the thread of its first row gets there: only the
    lowering of the slot's row keeps the dictionary in first-seen order and the ids on the first rows."""
    rng = np.random.default_rng(59)
    rows = 4 * 2048
    first = _distinct(40, 16, rng, b"first-")
    filler = np.asarray(_distinct(30, 16, rng, b"fill-"), dtype=object)
    vals = _first_seen_after_later_blocks(first, filler, rows, rng)
    _, segs = _string_same(ctx, vals, "strings")
    assert int(segs[0]["type"]) == SEGMENT_DICTIONARY_DENSE
    _check_value_ids(ctx, vals)
    ints = np.asarray(_first_seen_after_later_blocks(list(range(10**12, 10**12 + 40)), np.arange(30, dtype=np.uint64) * 977,
                                                     rows, rng), dtype=np.uint64)
    _, isegs = _int_same(ctx, ints, None, "integers")
    assert int(isegs[0]["type"]) == SEGMENT_DICTIONARY_DENSE


@pytest.mark.gpu
def test_gpu_string_copy_edges(ctx):
    rng = np.random.default_rng(61)
    # lengths around the warp's 32-byte stride, all distinct so every row supplies its string (DirectDense)
    lens = [0, 1, 31, 32, 33, 4097] * 40
    vals = [bytes(rng.integers(0, 256, ln, dtype=np.uint8)) for ln in lens]
    vals = [v + bytes([i % 251]) if len(v) else v for i, v in enumerate(vals)]
    _, segs = _string_same(ctx, vals, "lengths")
    # warps where all 32 rows or none of them supply a string: NULL warps, and warps of one repeated value (DictionaryDense)
    words = _distinct(5, 33, rng)
    col = []
    for warp in range(40):
        kind = warp % 4
        col += [None] * 32 if kind == 0 else ([words[warp % 5]] * 32 if kind == 1 else
                                              [words[int(i)] for i in rng.integers(0, 5, 32)])
    _string_same(ctx, col, "warps")
    _string_same(ctx, [None] * 32 + [b"z" * 40] * 32 + [None] * 64, "warps-rle")
    # starts that are not sorted, and rows that share heap bytes
    heap = np.frombuffer(rng.bytes(1 << 21), dtype=np.uint8).copy()  # more bytes than the rows' lengths add up to
    n = 3000
    starts = rng.integers(0, 9000, n).astype(np.uint64)
    starts[::5] = 17                                  # many rows on the same bytes
    lengths = rng.integers(0, 900, n).astype(np.uint32)
    lengths[::7] = 33
    nulls = (rng.random(n) < 0.05).astype(np.uint8)
    values = [None if nulls[i] else heap[int(starts[i]):int(starts[i]) + int(lengths[i])].tobytes() for i in range(n)]
    _string_same_flat(ctx, heap, starts, lengths, nulls, values, "aliased", max_segment_values=1000)


@pytest.mark.gpu
def test_gpu_string_many_tiny_segments(ctx):
    """2*10^5 ten-byte values cut by a 25-byte buffer: 66667 segments of 3 rows.  Every segment's table is sized by its own
    rows; a table sized by max_segment_values for every segment would take about 140 GB."""
    n = 200_000
    rng = np.random.default_rng(67)
    words = _distinct(1000, 10, rng)
    vals = [words[int(i)] for i in rng.integers(0, 1000, n)]
    heap, starts, lengths, nulls = oracle.flatten_strings(vals)
    data, segs = _string_same_flat(ctx, heap, starts, lengths, nulls, None, "tiny", max_buffer_bytes=25)
    assert segs["row_count"].tolist() == [3] * (n // 3) + [n % 3]


@pytest.mark.gpu
def test_gpu_string_buffer_cut_column_of_gigabytes(ctx):
    """A column of 2 GiB in 2^20 values of 2 KiB under the default 32 MiB buffer: 64 segments of 16384 rows (one buffer
    cut each), written in device memory and compared with the oracle."""
    n, ln = 1 << 20, 2048
    rng = np.random.default_rng(71)
    heap = np.frombuffer(rng.bytes(n * ln), dtype=np.uint8)
    starts = np.arange(n, dtype=np.uint64) * np.uint64(ln)
    lengths = np.full(n, ln, np.uint32)
    data, segs = _string_same_flat(ctx, heap, starts, lengths, None, None, "gigabytes", device=(True,))
    assert segs["row_count"].tolist() == [16385] * 63 + [n - 63 * 16385]  # 16384 values fill the buffer, the next one cuts


# 3. tripwires ---------------------------------------------------------------------------------------------------------
def _source(name):
    with open(os.path.join(CSRC, name)) as f:
        return re.sub(r"\s+", " ", f.read())


@pytest.mark.parametrize("name", ["column_writer.cu", "string_column_writer.cu"])
def test_hash_restatements_match_the_sources(name):
    src = _source(name)
    mix = re.search(r"u64 mix64\(u64 x\) \{(.*?)\}", src).group(1)
    assert mix.split(";")[:3] == [" x ^= x >> 33", " x *= 0xff51afd7ed558ccdull", " x ^= x >> 33"]
    assert f"{MIX_MUL:#x}ull" in mix
    assert "const u32 fp = (u32)(mx >> 32);" in src and "h = (u32)mx & mask;" in src and "h = (h + 1) & mask;" in src
    assert "cap = 8; while (" in src and "cap < 2 * " in src and "cap <<= 1;" in src  # a power of two >= 2 x rows, at least 8
    if name == "string_column_writer.cu":
        assert "u64 hsh = 0xcbf29ce484222325ull ^ len;" in src and f"{FNV_BASIS:#x}ull" in src
        assert "hsh = (hsh ^ p[k]) * 0x100000001b3ull;" in src and f"{FNV_PRIME:#x}ull" in src
        assert "const u64 rows = seg_start[s + 1] - seg_start[s];" in src  # each segment's table is sized by its own rows
    else:
        assert "const u64 seg_rows = std::min<u64>(max_values, n);" in src  # every integer segment holds max_values rows
