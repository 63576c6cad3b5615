"""The format converters on both sides of the hot path at the edges random data does not reach.

The horizontal block codec (ytgpu_encode_horizontal_block / ytgpu_decode_horizontal_block), the string column -> ClickHouse
conversion (ytgpu_convert_string_column_to_ch), the ClickHouse -> values conversion (ytgpu_convert_ch_column_to_values),
the column readers' flag and dictionary-index helpers (columnar_flags.cu) and the string offset decoders (columnar.cu) are
compared byte for byte with the oracle at varint, run, window and alignment edges, in HOST and DEVICE memory.  Every
output buffer is surrounded by guard bytes that must come back untouched, also when a call is refused.

On the CPU the oracle is checked against the plain Python restatements below; the GPU cases compare the product with the
oracle.  Cases built to reach a fast path assert their own premise (alignment, run lengths, the 48-byte boundary), and the
constants restated here are pinned to the CUDA sources at the end of the file."""
import ctypes as C
import os
import re
import struct

import numpy as np
import pytest

import oracle
from oracle import FLAGS_BITMAP as BM, FLAGS_DICTIONARY_ZERO as DZ
from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import VALUE_DTYPE, EValueType as T

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "ytsaurus_b200", "csrc")
U64, U32 = 2**64, 2**32
INT64_MIN, INT64_MAX = -2**63, 2**63 - 1

# restated from the sources (pinned by test_restated_constants_match_the_sources)
SHORT_VALUE = 48  # string_to_ch.cu: longer values are copied by the whole warp
VEC_STEP = 256    # columnar_flags.cu: rows per warp step of the dictionary-index -> bitmap vector path
ALIGN = 16        # the vector paths need 16-byte aligned pointers

GUARD = 32
_PATTERN = ((np.arange(251 * 64) * 89 + 17) % 251).astype(np.uint8)  # period 251: a shifted write cannot match it


# ---------------------------------------------------------------------------------------------------------------- buffers
class Buf:
    """A buffer in HOST (numpy) or DEVICE (torch) memory whose payload starts at `shift` mod 16, with guard bytes around
    it.  `data`: the payload to place (input), or None and `nbytes` (output, pre-filled with the pattern)."""

    def __init__(self, device, data=None, nbytes=None, shift=0):
        raw = None if data is None else np.ascontiguousarray(data).view(np.uint8).reshape(-1)
        self.n = len(raw) if raw is not None else int(nbytes)
        self.device = device
        arr = np.resize(_PATTERN, 2 * GUARD + ALIGN + self.n)
        # device allocations are 256-byte aligned; a host array may start anywhere
        base = 0 if device else arr.ctypes.data
        self.lead = GUARD + (shift - (base + GUARD)) % ALIGN
        if raw is not None:
            arr[self.lead:self.lead + self.n] = raw
        self.before = arr.copy()
        if device:
            import torch
            self.store = torch.from_numpy(arr).cuda()
            base = self.store.data_ptr()
        else:
            self.store = arr
        self.ptr = base + self.lead
        assert self.ptr % ALIGN == shift % ALIGN

    def host(self):
        return self.store.cpu().numpy() if self.device else self.store

    def get(self):
        """The payload; asserts that the guard bytes around it are untouched."""
        h = self.host()
        lo, hi = self.lead, self.lead + self.n
        assert (h[:lo] == self.before[:lo]).all() and (h[hi:] == self.before[hi:]).all(), "guard bytes changed"
        return h[lo:hi].copy()

    def untouched(self):
        return (self.host() == self.before).all()


def mem_of(device):
    return capi.MEM_DEVICE if device else capi.MEM_HOST


def _opt(device, a, shift=0):
    return None if a is None else Buf(device, a, shift=shift)


def _p(b):
    return None if b is None else b.ptr


# ---------------------------------------------------------------------------------------------------------------- block codec
def py_varuint(v: int) -> bytes:
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


def py_zigzag(v: int) -> int:
    return ((v << 1) ^ (v >> 63)) % U64


def py_unzigzag(z: int) -> int:
    return (z >> 1) ^ -(z & 1)


def py_block_encode(values, heap, counts=None) -> bytes:
    """THorizontalBlockWriter restated: offsets, then per row varuint count and (id, type, payload) per value."""
    heap = bytes(heap)
    n, c = values.shape
    rows = []
    for r in range(n):
        cnt = c if counts is None else min(int(counts[r]), c)
        row = bytearray(py_varuint(cnt))
        for v in values[r, :cnt]:
            t = T.Any if v["type"] == T.Composite else int(v["type"])
            row += py_varuint(int(v["id"])) + py_varuint(t)
            d = int(v["data"])
            if t == T.Int64:
                row += py_varuint(py_zigzag(d - U64 if d >= 2**63 else d))
            elif t == T.Uint64:
                row += py_varuint(d)
            elif t == T.Double:
                row += struct.pack("<Q", d)
            elif t == T.Boolean:
                row += b"\x01" if d & 0xFF else b"\x00"
            elif t in (T.String, T.Any):
                row += py_varuint(int(v["length"])) + heap[d:d + int(v["length"])]
        rows.append(bytes(row))
    offs = np.cumsum([0] + [len(x) for x in rows[:-1]]).tolist() if rows else []
    return struct.pack(f"<{n}I", *offs) + b"".join(rows)


def boundaries(bits):
    """0, 1 and 2^b - 1, 2^b, 2^b + 1 for every b of the form 7k - 1, 7k, 7k + 1 below `bits`, and 2^bits - 1."""
    out = {0, 1, 2**bits - 1}
    for k in range(1, bits // 7 + 2):
        for b in (7 * k - 1, 7 * k, 7 * k + 1):
            if b < bits:
                out |= {2**b - 1, 2**b, 2**b + 1}
    return sorted(out)


def make_values(rows, ncols):
    """rows: lists of (id, type, length, data) tuples -> VALUE_DTYPE [len(rows), ncols] (missing values Null)."""
    v = np.zeros((len(rows), ncols), VALUE_DTYPE)
    v["type"] = T.Null
    for r, row in enumerate(rows):
        for c, (i, t, ln, d) in enumerate(row):
            v[r, c] = (i, t, 0, ln, d % U64)
    return v


def edge_rowsets():
    """(name, values, heap, row_value_counts or None)."""
    rng = np.random.default_rng(5)
    heap = np.frombuffer(rng.bytes(2**21 + 8), np.uint8).copy()
    sets = []

    def chunked(vals, per_row=4):
        return [vals[i:i + per_row] for i in range(0, len(vals), per_row)]

    ids = boundaries(16)
    assert ids[-1] == 65535
    sets.append(("ids", make_values(chunked([(i, T.Int64, 0, i) for i in ids]), 4), heap[:0], None))
    zz = sorted({py_unzigzag(z) for z in boundaries(64)} | {s * b for b in boundaries(63) for s in (1, -1)}
                | {INT64_MIN, INT64_MAX, INT64_MIN + 1, INT64_MAX - 1})
    assert min(zz) == INT64_MIN and max(zz) == INT64_MAX
    sets.append(("int64", make_values(chunked([(7, T.Int64, 0, x) for x in zz]), 4), heap[:0], None))
    u = boundaries(64)
    assert u[-1] == U64 - 1
    sets.append(("uint64", make_values(chunked([(1, T.Uint64, 0, x) for x in u]), 4), heap[:0], None))
    lens = [x for x in boundaries(22) if x <= 2**21 + 1]
    assert 2**21 + 1 in lens and 2**14 - 1 in lens
    sets.append(("string-lengths", make_values(chunked([(2, T.String if k % 2 else T.Any, ln, k % 7) for k, ln in enumerate(lens)], 3), 3),
                 heap, None))
    # value counts at the varint boundaries of the count itself: one row of each, 16385 columns
    vc = [0, 1, 127, 128, 129, 16383, 16384, 16385]
    wide = np.zeros((len(vc), 16385), VALUE_DTYPE)
    wide["type"] = T.Uint64
    wide["data"] = np.arange(wide.size, dtype=np.uint64).reshape(wide.shape) % 300
    wide["id"] = np.arange(16385, dtype=np.uint16)
    sets.append(("value-counts", wide, heap[:0], np.array(vc, np.uint32)))
    # counts of 0, exactly value_count and above it (clamped)
    small = make_values([[(0, T.Int64, 0, -5), (1, T.String, 3, 0), (2, T.Uint64, 0, 9)]] * 5, 3)
    sets.append(("counts-clamped", small, heap, np.array([0, 3, 4, 1000, U32 - 1], np.uint32)))
    # Composite is written as Any; Null / Min / Max / Bottom carry no payload even with bits in data; Boolean of any byte
    odd = [[(0, T.Composite, 5, 11), (1, T.Null, 7, 99), (2, T.Min, 0, 1), (3, T.Max, 0, 2), (4, T.TheBottom, 3, 3)],
           [(5, T.Boolean, 0, 2), (6, T.Boolean, 0, 0x100), (7, T.Boolean, 0, 0xFF), (8, T.Boolean, 0, 1), (9, T.Double, 0, U64 - 1)]]
    sets.append(("types", make_values(odd, 5), heap, None))
    # rows whose data crosses 2^16 and 2^24 bytes
    big = make_values([[(0, T.String, 40000, 0), (1, T.String, 40000, 3)],
                       [(0, T.String, 2**21, 1), (1, T.Int64, 0, -1)],
                       [(0, T.String, 2**21, 5), (1, T.String, 2**21, 2)]] +
                      [[(0, T.String, 2**21, k), (1, T.Any, 2**21, 2 * k)] for k in range(3)], 2)
    sets.append(("cross-2^16-2^24", big, heap, None))
    return sets


def hand_block(rows):
    offs = np.cumsum([0] + [len(r) for r in rows[:-1]]).tolist()
    return np.frombuffer(struct.pack(f"<{len(rows)}I", *offs) + b"".join(rows), np.uint8).copy()


def good_hand_blocks():
    """Well-formed blocks the encoder never writes: (name, block, rows, value_count)."""
    vi = py_varuint
    return [
        ("boolean-bytes", hand_block([b"\x04" + b"".join(b"\x00\x06" + bytes([x]) for x in (0, 1, 2, 0xFF))]), 1, 4),
        ("empty-rows", hand_block([b"\x00", b"\x00", b"\x01\x00\x02"]), 3, 2),
        ("count-above-value-count", hand_block([b"\x03\x00\x03\x02\x01\x04\x05\x02\x02"]), 1, 1),
        ("ten-byte-varints", hand_block([b"\x02" + vi(3) + b"\x03" + vi(U64 - 1) + b"\x01\x04" + vi(U64 - 1)]), 1, 2),
        ("string-to-the-end", hand_block([b"\x01\x00\x10\x03abc"]), 1, 1),
    ]


def malformed_blocks():
    """(name, block, rows, value_count): every one must be refused."""
    vi = py_varuint
    ok_row = b"\x01\x00\x03\x02"
    blk = hand_block([ok_row, ok_row])
    past = blk.copy()
    past[4:8] = np.frombuffer(struct.pack("<I", 100), np.uint8)
    at_end = blk.copy()
    at_end[4:8] = np.frombuffer(struct.pack("<I", len(blk) - 8), np.uint8)
    return [
        ("overlong-count", hand_block([b"\x80" * 10 + b"\x01"]), 1, 1),
        ("overlong-id", hand_block([b"\x01" + b"\x80" * 10 + b"\x01\x03\x02"]), 1, 1),
        ("overlong-int64", hand_block([b"\x01\x00\x03" + b"\xff" * 10 + b"\x01"]), 1, 1),
        ("overlong-length", hand_block([b"\x01\x00\x10" + b"\x80" * 10 + b"\x00"]), 1, 1),
        ("offset-past-end", past, 2, 1),
        ("offset-at-end", at_end, 2, 1),
        ("type-0x102", hand_block([b"\x01\x00" + vi(0x102)]), 1, 1),           # (u8) would read it as Null
        ("type-0x110", hand_block([b"\x01\x00" + vi(0x110) + b"\x01x"]), 1, 1),  # (u8) would read it as String
        ("type-unknown", hand_block([b"\x01\x00\x07"]), 1, 1),
        ("string-past-end", hand_block([b"\x01\x00\x10\x05abcd"]), 1, 1),
        ("string-wraps-2^64", hand_block([b"\x01\x00\x10" + vi(U64 - 1) + b"abc"]), 1, 1),
        ("string-wraps-2^64-2", hand_block([b"\x01\x00\x11" + vi(U64 - 2) + b"abc"]), 1, 1),
        ("truncated-double", hand_block([b"\x01\x00\x05" + b"\x00" * 7]), 1, 1),
        ("truncated-boolean", hand_block([b"\x01\x00\x06"]), 1, 1),
        ("truncated-value", hand_block([b"\x02\x00\x03\x02"]), 1, 2),
        ("offset-table-only", np.zeros(8, np.uint8), 2, 1),
    ]


def test_oracle_block_encoder_matches_the_restatement():
    assert [py_varuint(2**b) for b in (7, 14, 63)] == [oracle.varuint_encode(2**b) for b in (7, 14, 63)]
    for name, values, heap, counts in edge_rowsets():
        got = oracle.block_encode(values, heap, counts).tobytes()
        assert got == py_block_encode(values, heap, counts), name
        n, c = values.shape
        want_cnt = [c] * n if counts is None else [min(int(x), c) for x in counts]
        if name == "cross-2^16-2^24":  # rows that start below 2^16 / 2^24 and end above
            offs = np.frombuffer(got[:4 * n], np.uint32).tolist() + [len(got) - 4 * n]
            assert any(a < 2**16 < b for a, b in zip(offs, offs[1:])) and any(a < 2**24 < b for a, b in zip(offs, offs[1:]))
        for vc in (1, c, c + 2):
            vals, cnt = oracle.block_decode(np.frombuffer(got, np.uint8), n, vc)
            assert cnt.tolist() == want_cnt, name
            for r in range(n):
                for k in range(vc):
                    if k >= want_cnt[r]:
                        assert vals[r, k]["type"] == T.Null and vals[r, k]["id"] == 0xFFFF
                    else:
                        w = values[r, k]
                        wt = T.Any if w["type"] == T.Composite else int(w["type"])
                        assert vals[r, k]["type"] == wt and vals[r, k]["id"] == w["id"], (name, r, k)
                        if wt in (T.Int64, T.Uint64, T.Double):
                            assert vals[r, k]["data"] == w["data"]
                        elif wt == T.Boolean:
                            assert vals[r, k]["data"] == (1 if int(w["data"]) & 0xFF else 0)
                        elif wt in (T.String, T.Any):
                            o, ln = int(vals[r, k]["data"]), int(vals[r, k]["length"])
                            assert ln == w["length"] and got[o:o + ln] == bytes(heap[int(w["data"]):int(w["data"]) + ln])
            if name == "value-counts":
                break  # 16385 x 8 values: one pass is enough


def test_oracle_block_decoder_edges():
    for name, block, n, vc in malformed_blocks():
        with pytest.raises(oracle.OracleError):
            oracle.block_decode(block, n, vc)
    vals, cnt = oracle.block_decode(good_hand_blocks()[0][1], 1, 4)
    assert vals["data"][0].tolist() == [0, 1, 0, 0] and (vals["type"][0] == T.Boolean).all()  # only the byte 1 is true
    vals, cnt = oracle.block_decode(good_hand_blocks()[3][1], 1, 2)
    assert vals["data"][0].tolist() == [INT64_MIN % U64, U64 - 1]


# ---------------------------------------------------------------------------------------------------------------- string -> CH
def zz32(x: int) -> int:
    return ((x << 1) ^ (x >> 31)) & 0xFFFFFFFF


def unzz32(z: int) -> int:
    return (z >> 1) ^ -(z & 1)


def yt_strings(strings, avg=None):
    """A string value column: chars + 32-bit zig-zag differences of the END offsets from avg_length * (k + 1)."""
    chars = b"".join(strings)
    avg = len(chars) // max(len(strings), 1) if avg is None else avg
    ends = np.cumsum([len(s) for s in strings]).tolist()
    offsets = np.array([zz32(e - ((avg * (k + 1)) % U32)) for k, e in enumerate(ends)], dtype=np.uint32)
    return offsets, avg, np.frombuffer(chars, np.uint8).copy()


def py_string_to_ch(offsets, avg, chars, d, rle, start, count, filt=None):
    """ConvertStringLikeYTColumnToCHColumn restated per row: the value behind row i (RLE run, then dictionary index, 0 =
    null = empty), its range as DecodeStringRange computes it (32-bit avg * index), then value + '\\0'."""
    def rng_(s):
        if s == 0:
            return 0, avg + unzz32(int(offsets[0]))
        base = (avg * s) % U32
        return base + unzz32(int(offsets[s - 1])), base + avg + unzz32(int(offsets[s]))
    out, ends = bytearray(), []
    for i in range(count):
        k = start + i
        if rle is not None:
            k = int(np.searchsorted(rle, k, side="right")) - 1
        s, empty = k, False
        if d is not None:
            empty = int(d[k]) == 0
            s = int(d[k]) - 1
        if filt is not None and filt[i] == 0:
            empty = True
        if not empty:
            b, e = rng_(s)
            out += bytes(chars[b:e])
        out += b"\0"
        ends.append(len(out))
    return bytes(out), ends


def mixed_trips(rng):
    """32 trips of 32 values, trip p with one long value at lane p among short ones (0 .. 48 bytes), then trips of short
    values only, at most 48 bytes with a 48 in each, then a trip of long values only."""
    long_lens = (SHORT_VALUE + 1, 10**5)
    strings = []
    for p in range(32):
        trip = [bytes(rng.integers(1, 256, int(rng.choice([0, 1, 5, 16, 47, 48])), dtype=np.uint8)) for _ in range(32)]
        trip[p] = bytes(rng.integers(1, 256, long_lens[p % 2], dtype=np.uint8))
        assert [len(s) > SHORT_VALUE for s in trip] == [j == p for j in range(32)]
        strings += trip
    for _ in range(3):
        trip = [bytes(rng.integers(1, 256, int(rng.choice([0, 47, 48])), dtype=np.uint8)) for _ in range(32)]
        trip[int(rng.integers(0, 32))] = bytes(SHORT_VALUE)
        assert max(len(s) for s in trip) == SHORT_VALUE
        strings += trip
    strings += [bytes(rng.integers(1, 256, SHORT_VALUE + 1 + j, dtype=np.uint8)) for j in range(32)]
    return strings


def run_starts(lengths):
    return np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.uint64)


def string_cases():
    """(name, offsets, avg, chars, dict, rle, windows [(start, count)])."""
    rng = np.random.default_rng(21)
    cases = []
    trips = mixed_trips(rng)
    off, avg, ch = yt_strings(trips)
    n = len(trips)
    cases.append(("direct-trips", off, avg, ch, None, None, [(0, n), (1, n - 1), (31, 33), (n - 1, 1)]))
    off2, avg2, ch2 = yt_strings(trips, len(ch))  # every difference negative
    assert all(unzz32(int(z)) < 0 for z in off2[:-1])
    cases.append(("direct-negative-zigzag", off2, avg2, ch2, None, None, [(0, n), (100, 200)]))
    pool = [b"", b"a", bytes(47), bytes(range(48)), bytes(range(49)), bytes(rng.integers(0, 256, 10**5, dtype=np.uint8))] + \
        [bytes(rng.integers(0, 256, int(rng.integers(0, 60)), dtype=np.uint8)) for _ in range(30)]
    poff, pavg, pch = yt_strings(pool)
    d_direct = rng.integers(0, len(pool) + 1, 3000).astype(np.uint32)
    d_direct[::5] = 0                                    # NULL entries
    cases.append(("dictionary", poff, pavg, pch, d_direct, None, [(0, 3000), (17, 1000), (2999, 1)]))
    lens = [1] * 40 + [31, 32, 33] * 10 + [100, 5000, 1, 1, 70, 2, 12000]
    rle = run_starts(lens)
    d_rle = rng.integers(0, len(pool) + 1, len(rle)).astype(np.uint32)
    d_rle[1::4] = 0
    total = int(sum(lens))
    inside = int(rle[45]) + 7                           # inside a run of 32
    wins = [(0, total), (inside, total - inside), (int(rle[60]), 500), (int(rle[-1]), lens[-1]), (int(rle[-1]) + 5, 100),
            (int(rle[-3]) - 1, 3), (int(rle[70]) + 99, 4000)]
    assert rle[45] < inside < rle[46]
    cases.append(("dictionary-rle", poff, pavg, pch, d_rle, rle, wins))
    # RLE straight over the strings: one string per run
    many = [bytes(rng.integers(0, 256, int(rng.choice([0, 3, 48, 49, 300])), dtype=np.uint8)) for _ in range(len(rle))]
    moff, mavg, mch = yt_strings(many)
    cases.append(("rle", moff, mavg, mch, None, rle, wins))
    return cases


def test_oracle_string_to_ch_matches_the_restatement():
    for name, off, avg, ch, d, rle, wins in string_cases():
        for start, count in wins:
            for filt in (None, np.zeros(count, np.uint8), np.arange(count, dtype=np.uint8) % 2):
                want = py_string_to_ch(off, avg, ch, d, rle, start, count, filt)
                got_c, got_o = oracle.string_column_to_ch(off, avg, ch, d, rle, start, count, filt)
                assert got_c.tobytes() == want[0] and got_o.tolist() == want[1], (name, start, count)


# ---------------------------------------------------------------------------------------------------------------- CH -> values
def f32(bits):
    return np.array(bits, np.uint32).view(np.float32)


def ch_cases():
    """(name, ch type, data, adjust)."""
    cases = []
    for t, dt in ((capi.CH_INT8, np.int8), (capi.CH_INT16, np.int16), (capi.CH_INT32, np.int32), (capi.CH_INT64, np.int64),
                  (capi.CH_UINT8, np.uint8), (capi.CH_UINT16, np.uint16), (capi.CH_UINT32, np.uint32), (capi.CH_UINT64, np.uint64)):
        i = np.iinfo(dt)
        cases.append((f"limits-{dt.__name__}", t, np.array([i.min, i.max, 0, 1, i.max - 1, i.min + 1], dt), 0))
    # subnormals, NaN payloads (quiet and signalling), infinities and -0.0
    cases.append(("float32", capi.CH_FLOAT32, f32([1, 0x7FFFFF, 0x80000001, 0x7FC00000, 0x7FC12345, 0xFFC00001, 0x7F800001,
                                                    0x7FA00000, 0x7F800000, 0xFF800000, 0x80000000, 0, 0x3F800000]), 0))
    cases.append(("float64", capi.CH_FLOAT64, np.array([1, 0x7FF8000000000001, 0xFFF0000000000001, 0x8000000000000000,
                                                        0x000FFFFFFFFFFFFF], np.uint64).view(np.float64), 0))
    cases.append(("bool", capi.CH_BOOL, np.array([0, 1, 1, 0], np.uint8), 0))
    for adj in (3, -1, -65536 * 3 - 1, 2**40 + 5):
        cases.append((f"date{adj}", capi.CH_DATE, np.array([0, 1, 65535, 65533, 100], np.uint16), adj))
        cases.append((f"date32{adj}", capi.CH_DATE32, np.array([-2**31, 2**31 - 1, -1, 0, 5], np.int32), adj))
        cases.append((f"datetime{adj}", capi.CH_DATETIME, np.array([0, U32 - 1, 10, 2**31], np.uint32), adj))
    cases.append(("datetime64", capi.CH_DATETIME64, np.array([INT64_MIN + 10, INT64_MAX - 10, -1, 0], np.int64), -7))
    cases.append(("timestamp-zero", capi.CH_TIMESTAMP, np.array([5, 6, INT64_MAX], np.int64), -5))
    return cases


def py_ch_value(t, x, adj):
    """-> (type, data) of one value: TSimpleValueConverter; the time types add the adjustment and cast back to their own
    ClickHouse type before they widen."""
    x = x.item() if hasattr(x, "item") else x
    if t in (capi.CH_INT8, capi.CH_INT16, capi.CH_INT32, capi.CH_INT64):
        return T.Int64, int(x) % U64
    if t in (capi.CH_UINT8, capi.CH_UINT16, capi.CH_UINT32, capi.CH_UINT64):
        return T.Uint64, int(x)
    if t == capi.CH_FLOAT32:
        return T.Double, None  # widened as the C++ cast does: compared against the oracle only
    if t == capi.CH_FLOAT64:
        return T.Double, int(np.asarray(x).view(np.uint64))
    if t == capi.CH_BOOL:
        return T.Boolean, int(x)
    if t == capi.CH_DATE:
        return T.Uint64, (int(x) + adj) % 2**16
    if t == capi.CH_DATE32:
        return T.Int64, (((int(x) + adj + 2**31) % U32) - 2**31) % U64
    if t == capi.CH_DATETIME:
        return T.Uint64, (int(x) + adj) % U32
    if t == capi.CH_DATETIME64:
        return T.Int64, (int(x) + adj) % U64
    return T.Uint64, int(x) + adj


def test_oracle_ch_to_values_matches_the_restatement():
    for name, t, data, adj in ch_cases():
        code, vals = oracle.ch_column_to_values(t, data, time_adjustment=adj)
        assert code == 0, name
        for k, x in enumerate(data):
            wt, wd = py_ch_value(t, x, adj)
            assert vals[k]["type"] == wt and (wd is None or vals[k]["data"] == wd), (name, k)
    # float32 -> double keeps the sign of -0.0, subnormals and the NaN payload bits (x86 quiets a signalling NaN)
    _, vals = oracle.ch_column_to_values(capi.CH_FLOAT32, f32([0x80000000, 1, 0x7FC12345]))
    assert vals["data"].tolist() == [2**63, 0x36A0000000000000, 0x7FF82468A0000000]
    assert oracle.ch_column_to_values(capi.CH_TIMESTAMP, np.array([4], np.int64), time_adjustment=-5)[0] == 2
    assert oracle.ch_column_to_values(capi.CH_BOOL, np.array([2], np.uint8), null_map=np.array([1], np.uint8))[0] == 1


# ---------------------------------------------------------------------------------------------------------------- flag helpers
STARTS = (0, 1, 7, 8, 31, 32, 255, 256, 257)
LENGTHS = tuple(range(0, 34)) + (63, 64, 65, 127, 128, 129, 223, 255, 256, 257, 511, 512, 513, 1023, 1024, 1025, 1055)


def pack_bits(bits):
    return np.packbits(np.asarray(bits, np.uint8), bitorder="little")


def flag_sources(rng, n_direct):
    """(name, kind, data, data_count, rle): direct dictionary indexes / bitmap, and RLE sources of both kinds with runs of
    1, of 31 / 32 / 33 and of 10^6 rows."""
    direct_d = rng.integers(0, 3, n_direct).astype(np.uint32)
    direct_b = pack_bits(rng.integers(0, 2, n_direct))
    out = [("direct-dict", DZ, direct_d, n_direct, None), ("direct-bitmap", BM, direct_b, n_direct, None)]
    for name, lens in (("runs-1", [1] * 1400), ("runs-31-32-33", [31, 32, 33] * 16),
                       ("runs-10^6", [10**6, 1, 10**6, 33, 10**6, 2])):
        rle = run_starts(lens)
        assert int(rle[-1]) + lens[-1] >= STARTS[-1] + LENGTHS[-1]
        d = rng.integers(0, 3, len(rle)).astype(np.uint32)
        d[::2] = np.where(d[::2] == 0, 1, 0)  # neighbouring runs differ often
        b = pack_bits((np.arange(len(rle)) + rng.integers(0, 2)) % 2 | rng.integers(0, 2, len(rle)))
        out.append((name + "-dict", DZ, d, len(rle), rle))
        out.append((name + "-bitmap", BM, b, len(rle), rle))
    return out


def py_flags(kind, data, rle, s, e):
    k = np.arange(s, e, dtype=np.int64)
    if rle is not None:
        k = np.searchsorted(rle, k.astype(np.uint64), side="right").astype(np.int64) - 1
    if kind == DZ:
        return (data[k] == 0).astype(np.uint8)
    return ((data[k >> 3] >> (k & 7)) & 1).astype(np.uint8)


def test_oracle_flag_helpers_match_the_restatement():
    rng = np.random.default_rng(8)
    for name, kind, data, n, rle in flag_sources(rng, 2000):
        wins = [(s, s + ln) for s in STARTS for ln in LENGTHS[::3]]
        if name.startswith("runs-10^6"):
            wins += [(10**6 - 257, 10**6 + 300), (2 * 10**6 - 1, 2 * 10**6 + 40)]
        for s, e in wins:
            f = py_flags(kind, data, rle, s, e)
            neg = (e - s) % 2
            assert oracle.build_bytemap_from_flags(kind, data, rle, s, e, neg).tolist() == (f ^ neg).tolist(), (name, s, e)
            assert oracle.build_bitmap_from_flags(kind, data, rle, s, e, neg).tobytes() == pack_bits(f ^ neg).tobytes()
            assert oracle.count_flags(kind, data, rle, s, e) == int(f.sum())
            if kind == DZ:
                k = np.arange(s, e) if rle is None else np.searchsorted(rle, np.arange(s, e, dtype=np.uint64), side="right") - 1
                assert oracle.build_dictionary_indexes(data, rle, s, e).tolist() == ((data[k].astype(np.int64) - 1) % U32).tolist()
                if rle is not None:
                    assert oracle.build_dictionary_indexes(None, rle, s, e).tolist() == (k - (k[0] if len(k) else 0)).tolist()


def py_string_offsets(enc, avg, s, e):
    off = [0] + [((avg * k) + unzz32(int(enc[k - 1]))) % U32 for k in range(1, e + 1)]
    return [(off[k] - off[s]) % U32 for k in range(s, e + 1)]


def py_pointers_and_lengths(enc, avg):
    ends = [avg * (k + 1) + unzz32(int(z)) for k, z in enumerate(enc)]
    starts = [0] + ends[:-1]
    return [x % U32 for x in starts], [((e - b + 2**31) % U32) - 2**31 for b, e in zip(starts, ends)]


AVGS = (0, 7, 2**31 + 5, U32 - 1, 0x9E3779B9)  # avg * index wraps 32 bits for all but the first two


def test_oracle_string_offsets_match_the_restatement():
    rng = np.random.default_rng(9)
    enc = rng.integers(0, U32, 600, dtype=np.uint64).astype(np.uint32)
    for avg in AVGS:
        for s, e in ((0, 0), (0, 1), (1, 1), (0, 600), (599, 600), (600, 600), (300, 600), (3, 17)):
            assert oracle.decode_string_offsets(enc, avg, s, e).tolist() == py_string_offsets(enc, avg, s, e), (avg, s, e)
        for n in (1, 600):
            st, ln = oracle.decode_string_pointers_and_lengths(enc[:n], avg)
            assert (st.tolist(), ln.tolist()) == py_pointers_and_lengths(enc[:n], avg)


# ================================================================================================================ GPU
@pytest.fixture(scope="module")
def ctx():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from ytsaurus_b200 import GpuContext
    c = GpuContext(0)
    yield c
    c.close()


def _call(fn, *args):
    err = capi.Error()
    code = fn(*args, C.byref(err))
    return code, err.message.decode(errors="replace")


# ---- block codec ----
def gpu_encode(ctx, device, values, heap, counts=None, capacity_delta=0):
    n, c = values.shape
    mem = mem_of(device)
    v, h = Buf(device, values), Buf(device, heap)
    rc = _opt(device, None if counts is None else np.asarray(counts, np.uint32))
    view = capi.RowsetView(v.ptr, n, c, 0, h.ptr, len(heap), mem)
    need = C.c_uint64(0)
    code, msg = _call(ctx.lib.ytgpu_encode_horizontal_block, ctx.handle, C.byref(view), _p(rc), None, 0, C.byref(need), mem)
    if n == 0:
        return code, b"", 0
    if need.value == 0 or need.value >= U32 + 4 * n:
        return code, None, need.value
    out = Buf(device, nbytes=need.value)
    code, msg = _call(ctx.lib.ytgpu_encode_horizontal_block, ctx.handle, C.byref(view), _p(rc), out.ptr, need.value + capacity_delta,
                      C.byref(need), mem)
    got = out.get()
    if code != capi.OK:
        assert out.untouched(), msg
        return code, None, need.value
    return code, got.tobytes(), need.value


def gpu_decode(ctx, device, block, n, vc, shift=0):
    mem = mem_of(device)
    b = Buf(device, block, shift=shift)
    o, cnt = Buf(device, nbytes=n * vc * 16), Buf(device, nbytes=n * 4)
    code, msg = _call(ctx.lib.ytgpu_decode_horizontal_block, ctx.handle, b.ptr, len(block), n, vc, o.ptr, cnt.ptr, mem)
    return code, o.get().view(VALUE_DTYPE).reshape(n, vc), cnt.get().view(np.uint32)


def check_decode(ctx, device, block, n, vc, shift=0, what=""):
    try:
        want, wcnt = oracle.block_decode(block, n, vc)
    except oracle.OracleError:
        want = None
    code, got, cnt = gpu_decode(ctx, device, block, n, vc, shift)
    if want is None:
        assert code == capi.ERR_INVALID_ARGUMENT, what
        return
    assert code == capi.OK, what
    assert cnt.tolist() == wcnt.tolist(), what
    assert got.tobytes() == want.tobytes(), what


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
def test_gpu_block_codec_edges(ctx, device):
    for name, values, heap, counts in edge_rowsets():
        want = oracle.block_encode(values, heap, counts)
        code, got, need = gpu_encode(ctx, device, values, heap, counts)
        assert code == capi.OK and got == want.tobytes(), name
        code, got, _ = gpu_encode(ctx, device, values, heap, counts, capacity_delta=-1)  # one byte short: refused, no write
        assert code == capi.ERR_INVALID_ARGUMENT and got is None, name
        n, c = values.shape
        for vc in (1, c, c + 2):
            check_decode(ctx, device, want, n, vc, shift=4 if device else 3, what=(name, vc))


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
def test_gpu_block_decoder_hand_blocks_and_malformed(ctx, device):
    for name, block, n, vc in good_hand_blocks():
        for k in (vc, 1, vc + 1):
            check_decode(ctx, device, block, n, k, what=name)
    for name, block, n, vc in malformed_blocks():
        with pytest.raises(oracle.OracleError):
            oracle.block_decode(block, n, vc)
        code, _, _ = gpu_decode(ctx, device, block, n, vc)
        assert code == capi.ERR_INVALID_ARGUMENT, name
        # the context still works afterwards
        good = good_hand_blocks()[4][1]
        check_decode(ctx, device, good, 1, 1, what=("after", name))


@pytest.mark.gpu
def test_gpu_block_of_almost_4_gib(ctx):
    """2^16 rows of one string: the data ends one byte below the 2^32-byte row-offset limit.  Written and read back in
    device memory and checked on the device; one byte more is refused in both memory flavours."""
    import torch
    n, L = 1 << 16, 65530
    row = 3 + 3 + L  # count, id, type, 3-byte varint length, bytes
    assert row == 1 << 16 and len(py_varuint(L)) == 3
    rng = np.random.default_rng(40)
    heap = np.frombuffer(rng.bytes(L + 1), np.uint8).copy()
    values = make_values([[(0, T.String, L, r & 1)] for r in range(n)], 1)
    values["length"][-1] = L - 1  # the last row one byte shorter: data = 2^32 - 1 bytes
    for device in (False, True):
        over = values.copy()
        over["length"][-1] = L     # data = 2^32 bytes: the last row offset no longer fits
        code, got, need = gpu_encode(ctx, device, over, heap)
        assert code == capi.ERR_INVALID_ARGUMENT and got is None and need == 4 * n + U32
    dv = torch.from_numpy(values.view(np.uint8).reshape(n, 16)).cuda()
    dh = torch.from_numpy(heap).cuda()
    bytes_ = 4 * n + U32 - 1
    out = torch.empty(bytes_ + 2 * GUARD, dtype=torch.uint8, device="cuda")
    out[:GUARD] = 0xA5
    out[-GUARD:] = 0x5A
    view = capi.RowsetView(dv.data_ptr(), n, 1, 0, dh.data_ptr(), len(heap), capi.MEM_DEVICE)
    need = C.c_uint64(0)
    code, msg = _call(ctx.lib.ytgpu_encode_horizontal_block, ctx.handle, C.byref(view), None, out.data_ptr() + GUARD, bytes_,
                      C.byref(need), capi.MEM_DEVICE)
    assert code == capi.OK and need.value == bytes_, msg
    assert bool((out[:GUARD] == 0xA5).all()) and bool((out[-GUARD:] == 0x5A).all())
    blk = out[GUARD:GUARD + bytes_]
    offs = blk[:4 * n].view(torch.int32).to(torch.int64) % U32
    assert torch.equal(offs.cpu(), torch.arange(n, dtype=torch.int64) * row)
    data = blk[4 * n:]
    full = data[:(n - 1) * row].view(n - 1, row)
    hdr = torch.tensor(list(b"\x01\x00\x10" + py_varuint(L)), dtype=torch.uint8, device="cuda")
    assert torch.equal(full[:, :6], hdr.expand(n - 1, 6))
    assert torch.equal(full[0::2, 6:], dh[:L].expand((n - 1 + 1) // 2, L))
    assert torch.equal(full[1::2, 6:], dh[1:L + 1].expand((n - 1) // 2, L))
    last = data[(n - 1) * row:]
    assert last.numel() == row - 1 and last[:6].tolist() == list(b"\x01\x00\x10" + py_varuint(L - 1))
    assert torch.equal(last[6:], dh[1:L])
    del full
    # read back on the device: every string points at its bytes inside the block
    dec = torch.empty((n, 16), dtype=torch.uint8, device="cuda")
    cnt = torch.empty(n, dtype=torch.int32, device="cuda")
    code, msg = _call(ctx.lib.ytgpu_decode_horizontal_block, ctx.handle, blk.data_ptr(), bytes_, n, 1, dec.data_ptr(), cnt.data_ptr(),
                      capi.MEM_DEVICE)
    assert code == capi.OK, msg
    got = dec.cpu().numpy().reshape(-1).view(VALUE_DTYPE)
    assert (cnt.cpu().numpy() == 1).all() and (got["type"] == T.String).all()
    assert got["length"].tolist() == [L] * (n - 1) + [L - 1]
    assert got["data"].tolist() == (4 * n + np.arange(n, dtype=np.uint64) * row + 6).tolist()
    del out, blk, data
    torch.cuda.empty_cache()


# ---- string column -> ClickHouse ----
def gpu_s2ch(ctx, device, off, avg, ch, d, rle, start, count, filt=None, chars_shift=0, out_shift=0, capacity_delta=0,
             size_query=False, total=None):
    mem = mem_of(device)
    bo, bc = Buf(device, off), Buf(device, ch, shift=chars_shift)
    bd, br, bf = _opt(device, d), _opt(device, rle), _opt(device, filt)
    view = capi.StringColumnView(bo.ptr, len(off), avg, mem, bc.ptr, len(ch), _p(bd), 0 if d is None else len(d), _p(br),
                                 0 if rle is None else len(rle), start, count)
    need = C.c_uint64(0)
    fn = ctx.lib.ytgpu_convert_string_column_to_ch
    if size_query:
        code, msg = _call(fn, ctx.handle, C.byref(view), _p(bf), None, 0, None, C.byref(need), mem)
        return code, need.value, None, None
    cap = (total if total is not None else 0) + capacity_delta
    oc, oo = Buf(device, nbytes=max(cap, 0), shift=out_shift), Buf(device, nbytes=8 * count)
    code, msg = _call(fn, ctx.handle, C.byref(view), _p(bf), oc.ptr, cap, oo.ptr, C.byref(need), mem)
    chars, offs = oc.get(), oo.get().view(np.uint64)
    if code != capi.OK:
        assert oc.untouched() and oo.untouched()
        return code, need.value, None, None
    return code, need.value, chars.tobytes(), offs.tolist()


def check_s2ch(ctx, device, off, avg, ch, d, rle, start, count, filt=None, what="", **kw):
    wc, wo = oracle.string_column_to_ch(off, avg, ch, d, rle, start, count, filt)
    code, need, got_c, got_o = gpu_s2ch(ctx, device, off, avg, ch, d, rle, start, count, filt, total=len(wc), **kw)
    assert code == capi.OK and need == len(wc), what
    assert got_o == wo.tolist(), what
    assert got_c == wc.tobytes(), what


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
def test_gpu_string_to_ch_windows_and_filters(ctx, device):
    for name, off, avg, ch, d, rle, wins in string_cases():
        for start, count in wins:
            filters = (None, np.zeros(count, np.uint8), np.ones(count, np.uint8), (np.arange(count) % 2).astype(np.uint8))
            for filt in filters:
                check_s2ch(ctx, device, off, avg, ch, d, rle, start, count, filt, what=(name, start, count))
            # the size query, the exact capacity and one byte short
            wc, _ = oracle.string_column_to_ch(off, avg, ch, d, rle, start, count)
            code, need, _, _ = gpu_s2ch(ctx, device, off, avg, ch, d, rle, start, count, size_query=True)
            assert code == capi.OK and need == len(wc), (name, start, count)
            if count:
                code, need, _, _ = gpu_s2ch(ctx, device, off, avg, ch, d, rle, start, count, total=len(wc), capacity_delta=-1)
                assert code == capi.ERR_INVALID_ARGUMENT and need == len(wc)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
def test_gpu_string_to_ch_every_alignment(ctx, device):
    """Short trips staged in shared memory, mixed trips and warp-copied long values, with the source chars at every offset
    mod 16 and (DEVICE) the output chars at every offset mod 16."""
    name, off, avg, ch, d, rle, wins = string_cases()[0]
    wc, wo = oracle.string_column_to_ch(off, avg, ch, None, None, 0, len(off))
    for cs in range(ALIGN):
        for os_ in (range(ALIGN) if device else (0,)):
            code, need, got_c, got_o = gpu_s2ch(ctx, device, off, avg, ch, None, None, 0, len(off), chars_shift=cs, out_shift=os_,
                                                total=len(wc))
            assert code == capi.OK and got_o == wo.tolist() and got_c == wc.tobytes(), (cs, os_)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
def test_gpu_string_to_ch_refuses_malformed_columns(ctx, device):
    off, avg, ch = yt_strings([b"ab", b"cde", b"f"])
    bad_end = off.copy()
    bad_end[1] = zz32(-5)                     # value 1 ends before it starts
    past = off.copy()
    past[2] = zz32(len(ch) + 1 - 3 * avg)     # value 2 ends past the chars
    cases = [("end-before-start", bad_end, None, None), ("past-chars", past, None, None),
             ("dict-past-strings", off, np.array([1, 4, 2], np.uint32), None),
             ("dict-rle-past-strings", off, np.array([1, 0, 9], np.uint32), np.array([0, 1, 2], np.uint64)),
             ("rle-first-not-zero", off, None, np.array([1, 2], np.uint64)),
             ("dict-rle-first-not-zero", off, np.array([1, 2], np.uint32), np.array([2, 3], np.uint64))]
    for name, o, d, rle in cases:
        code, _, _, _ = gpu_s2ch(ctx, device, o, avg, ch, d, rle, 0, 3, total=64)
        assert code == capi.ERR_INVALID_ARGUMENT, name
        code, _, _, _ = gpu_s2ch(ctx, device, o, avg, ch, d, rle, 0, 3, size_query=True)
        assert code == capi.ERR_INVALID_ARGUMENT, name
    check_s2ch(ctx, device, off, avg, ch, None, None, 0, 3, what="after")  # the context stays usable


# ---- ClickHouse -> values ----
def gpu_ch(ctx, device, t, data, n, offsets=None, null_map=None, adj=0, data_shift=0, out_shift=0):
    mem = mem_of(device)
    bd = Buf(device, data, shift=data_shift)
    bo, bn = _opt(device, offsets), _opt(device, null_map)
    chars = len(np.asarray(data).view(np.uint8).reshape(-1)) if offsets is not None else 0
    col = capi.ChColumn(t, mem, bd.ptr, _p(bo), chars, _p(bn), adj, n)
    out = Buf(device, nbytes=16 * n, shift=out_shift)
    code, msg = _call(ctx.lib.ytgpu_convert_ch_column_to_values, ctx.handle, C.byref(col), out.ptr, mem)
    got = out.get()
    if code != capi.OK:
        return code, None
    return code, got.view(VALUE_DTYPE)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
def test_gpu_ch_to_values_limits(ctx, device):
    for name, t, data, adj in ch_cases():
        nulls = (np.arange(len(data)) % 3 == 1).astype(np.uint8)
        for nm in (None, nulls):
            wc, want = oracle.ch_column_to_values(t, data, null_map=nm, time_adjustment=adj)
            assert wc == 0
            for shift in ((0,) if device else (0, 1, 3, 7)):  # HOST inputs at any address
                code, got = gpu_ch(ctx, device, t, data, len(data), null_map=nm, adj=adj, data_shift=shift)
                assert code == capi.OK and got.tobytes() == want.tobytes(), (name, nm is None, shift)
    # TIMESTAMP exactly 0 after the adjustment passes, -1 is refused (also under a NULL)
    code, got = gpu_ch(ctx, device, capi.CH_TIMESTAMP, np.array([5, 6], np.int64), 2, adj=-5)
    assert code == capi.OK and got["data"].tolist() == [0, 1]
    for nm in (None, np.array([1, 1], np.uint8)):
        assert gpu_ch(ctx, device, capi.CH_TIMESTAMP, np.array([5, 4], np.int64), 2, null_map=nm, adj=-5)[0] == capi.ERR_INVALID_ARGUMENT
    # a Bool byte above 1 is refused, also under a NULL
    for b in (2, 0xFF):
        assert gpu_ch(ctx, device, capi.CH_BOOL, np.array([1, b], np.uint8), 2, null_map=np.array([0, 1], np.uint8))[0] != capi.OK
    # strings: offsets equal to chars_bytes pass, one past it is refused; an empty value is one terminating zero
    strings = [b"", b"x", bytes(range(1, 60)), b""]
    chars = np.frombuffer(b"".join(s + b"\0" for s in strings), np.uint8).copy()
    offs = np.cumsum([len(s) + 1 for s in strings]).astype(np.uint64)
    assert offs[-1] == len(chars)
    wc, want = oracle.ch_column_to_values(capi.CH_STRING, chars, offs, None, row_count=len(offs))
    code, got = gpu_ch(ctx, device, capi.CH_STRING, chars, len(offs), offsets=offs)
    assert wc == 0 and code == capi.OK and got.tobytes() == want.tobytes()
    bad = offs.copy()
    bad[-1] += 1
    assert gpu_ch(ctx, device, capi.CH_STRING, chars, len(offs), offsets=bad)[0] == capi.ERR_INVALID_ARGUMENT
    bad = offs.copy()
    bad[1] = bad[0]                       # a value without its terminating zero
    assert gpu_ch(ctx, device, capi.CH_STRING, chars, len(offs), offsets=bad)[0] == capi.ERR_INVALID_ARGUMENT
    # DEVICE outputs must be 16-byte aligned: refused without a write
    if device:
        for shift in (1, 4, 8):
            assert gpu_ch(ctx, device, capi.CH_INT64, np.arange(5, dtype=np.int64), 5, out_shift=shift)[0] == capi.ERR_INVALID_ARGUMENT


# ---- flag, dictionary-index and offset helpers ----
def gpu_map(ctx, device, bitmap, kind, data, n, rle, s, e, negate, data_shift=0, out_shift=0):
    mem = mem_of(device)
    bd, br = Buf(device, data, shift=data_shift), _opt(device, rle)
    src = capi.FlagSource(kind, 0, bd.ptr, n, _p(br), 0 if rle is None else len(rle))
    out = Buf(device, nbytes=(e - s + 7) // 8 if bitmap else e - s, shift=out_shift)
    fn = ctx.lib.ytgpu_build_bitmap_from_flags if bitmap else ctx.lib.ytgpu_build_bytemap_from_flags
    code, msg = _call(fn, ctx.handle, C.byref(src), s, e, int(negate), out.ptr, mem)
    assert code == capi.OK, msg
    return out.get()


def gpu_count(ctx, device, kind, data, n, rle, s, e, data_shift=0):
    mem = mem_of(device)
    bd, br = Buf(device, data, shift=data_shift), _opt(device, rle)
    src = capi.FlagSource(kind, 0, bd.ptr, n, _p(br), 0 if rle is None else len(rle))
    out = C.c_int64(-1)
    code, msg = _call(ctx.lib.ytgpu_count_flags, ctx.handle, C.byref(src), s, e, C.byref(out), mem)
    assert code == capi.OK, msg
    return out.value


def gpu_dict_indexes(ctx, device, d, rle, s, e, data_shift=0, out_shift=0):
    mem = mem_of(device)
    bd, br = _opt(device, d, data_shift), _opt(device, rle)
    out = Buf(device, nbytes=4 * (e - s), shift=out_shift)
    code, msg = _call(ctx.lib.ytgpu_build_dictionary_indexes, ctx.handle, _p(bd), 0 if d is None else len(d), _p(br),
                      0 if rle is None else len(rle), s, e, out.ptr, mem)
    assert code == capi.OK, msg
    return out.get().view(np.uint32)


def gpu_total_length(ctx, device, d, rle, lengths, s, e):
    mem = mem_of(device)
    bd, br, bl = Buf(device, d), Buf(device, rle), Buf(device, lengths)
    out = C.c_int64(-1)
    code, msg = _call(ctx.lib.ytgpu_count_total_string_length, ctx.handle, bd.ptr, br.ptr, len(rle), bl.ptr, len(lengths), s, e,
                      C.byref(out), mem)
    return code, out.value


def gpu_translate(ctx, device, rle, idx, end_flavour):
    mem = mem_of(device)
    br, bi = Buf(device, rle), Buf(device, np.asarray(idx, np.int64))
    out = Buf(device, nbytes=8 * len(idx))
    code, msg = _call(ctx.lib.ytgpu_translate_rle_indexes, ctx.handle, br.ptr, len(rle), bi.ptr, len(idx), int(end_flavour), out.ptr, mem)
    got = out.get().view(np.int64)
    return code, got.tolist() if code == capi.OK else None


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
def test_gpu_flag_helpers_windows(ctx, device):
    """Every helper over every source kind, windows starting at 0, 1, 7, 8, 31, 32, 255, 256 and 257 and ending in every
    class mod 32 and the edges of the 256-row step."""
    rng = np.random.default_rng(11)
    for name, kind, data, n, rle in flag_sources(rng, 2000):
        wins = [(s, s + ln) for s in STARTS for ln in LENGTHS]
        if name.startswith("runs-10^6"):
            total = int(rle[-1]) + 2
            wins += [(10**6 - 257, 10**6 + 300), (2 * 10**6 - 1, 2 * 10**6 + 40), (0, total), (10**6 + 1, total)]
        for s, e in wins:
            neg = (e - s) % 2
            for bitmap in (True, False):
                want = (oracle.build_bitmap_from_flags if bitmap else oracle.build_bytemap_from_flags)(kind, data, rle, s, e, neg)
                got = gpu_map(ctx, device, bitmap, kind, data, n, rle, s, e, neg, out_shift=(s + e) % 8)
                assert got.tobytes() == want.tobytes(), (name, bitmap, s, e, neg)
            assert gpu_count(ctx, device, kind, data, n, rle, s, e) == oracle.count_flags(kind, data, rle, s, e), (name, s, e)
            if kind == DZ:
                want = oracle.build_dictionary_indexes(data, rle, s, e)
                assert gpu_dict_indexes(ctx, device, data, rle, s, e).tolist() == want.tolist(), (name, s, e)
                if rle is not None:
                    want = oracle.build_dictionary_indexes(None, rle, s, e)
                    assert gpu_dict_indexes(ctx, device, None, rle, s, e).tolist() == want.tolist(), (name, "iota", s, e)


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
def test_gpu_dictionary_pointers_at_every_offset(ctx, device):
    """Direct dictionary indexes at every offset mod 16 (DEVICE: every 4-byte aligned one, the indexes are read as uint32):
    the 256-row vector step runs when the first index is 16-byte aligned, the generic kernel finishes the tail."""
    rng = np.random.default_rng(12)
    d = rng.integers(0, 2, 3000).astype(np.uint32)
    reached = set()
    for shift in (range(0, ALIGN, 4) if device else range(ALIGN)):
        for s in (0, 1, 2, 3, 4):
            for ln in (255, 256, 257, 511, 512 + 37, 1024, 2048 + 255):
                e = s + ln
                # HOST sources are staged into a fresh device buffer: there only the window start sets the alignment
                first = ((shift if device else 0) + 4 * s) % ALIGN
                reached.add((first == 0, ln >= VEC_STEP and ln % VEC_STEP != 0))
                for neg in (False, True):
                    want = oracle.build_bitmap_from_flags(DZ, d, None, s, e, neg)
                    got = gpu_map(ctx, device, True, DZ, d, len(d), None, s, e, neg, data_shift=shift, out_shift=shift % 5)
                    assert got.tobytes() == want.tobytes(), (shift, s, e, neg)
                want = oracle.build_bytemap_from_flags(DZ, d, None, s, e, False)
                assert gpu_map(ctx, device, False, DZ, d, len(d), None, s, e, False, data_shift=shift).tobytes() == want.tobytes()
                assert gpu_count(ctx, device, DZ, d, len(d), None, s, e, data_shift=shift) == oracle.count_flags(DZ, d, None, s, e)
                want = oracle.build_dictionary_indexes(d, None, s, e)
                got = gpu_dict_indexes(ctx, device, d, None, s, e, data_shift=shift, out_shift=(4 * s) % ALIGN if device else s)
                assert got.tolist() == want.tolist(), (shift, s, e)
    assert reached == {(True, True), (True, False), (False, True), (False, False)}  # vector path with and without a tail


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
def test_gpu_total_string_length_and_translate(ctx, device):
    lens = [1, 1, 31, 32, 33, 1, 10**6, 5, 1]
    rle = run_starts(lens)
    total = int(sum(lens))
    lengths = np.array([0, 7, 0, 2**20, 3], np.int32)
    d = np.array([1, 0, 2, 5, 4, 3, 2, 1, 6], np.uint32)  # the last run's id 6 is string_count + 1: past the strings
    last = len(rle) - 1
    for s, e in ((0, int(rle[last])), (1, 70), (int(rle[2]), int(rle[3])), (int(rle[3]) - 1, int(rle[4]) + 1), (5, int(rle[7])),
                 (int(rle[6]) + 17, int(rle[7]) - 3), (0, 0)):
        want = oracle.count_total_string_length(d[:last], rle[:last], lengths, s, e)
        code, got = gpu_total_length(ctx, device, d, rle, lengths, s, e)  # a window ending at the bad run's start never reads it
        assert code == capi.OK and got == want, (s, e)
    for s, e in ((int(rle[last]), total), (0, total), (int(rle[last]) - 1, int(rle[last]) + 1)):
        assert gpu_total_length(ctx, device, d, rle, lengths, s, e)[0] == capi.ERR_INVALID_ARGUMENT, (s, e)
    assert gpu_total_length(ctx, device, d[:last], rle[:last], lengths, 0, 5)[0] == capi.OK  # the context stays usable
    idx = sorted({0, total - 1, total, total + 5} | {int(x) for x in rle} | {int(x) - 1 for x in rle[1:]})
    for end_flavour in (False, True):
        f = oracle.translate_rle_end_index if end_flavour else oracle.translate_rle_index
        code, got = gpu_translate(ctx, device, rle, idx, end_flavour)
        assert code == capi.OK and got == [f(rle, i) for i in idx], end_flavour
        # index -1: the HOST flavour refuses it; the DEVICE flavour does not read its indexes on the host and maps it to
        # the run before the first (-1), or to 0 for an end index
        code, got = gpu_translate(ctx, device, rle, [3, -1], end_flavour)
        if device:
            assert code == capi.OK and got == [f(rle, 3), 0 if end_flavour else -1]
        else:
            assert code == capi.ERR_INVALID_ARGUMENT


@pytest.mark.gpu
@pytest.mark.parametrize("device", [False, True])
def test_gpu_string_offsets_wrap_like_the_oracle(ctx, device):
    rng = np.random.default_rng(13)
    enc = rng.integers(0, U32, 600, dtype=np.uint64).astype(np.uint32)
    mem = mem_of(device)
    for avg in AVGS:
        for s, e in ((0, 0), (0, 1), (1, 1), (0, 600), (599, 600), (600, 600), (300, 600), (3, 17)):
            be = Buf(device, enc[:e] if e else np.zeros(0, np.uint32))
            out = Buf(device, nbytes=4 * (e - s + 1), shift=(4 * s) % ALIGN)
            code, msg = _call(ctx.lib.ytgpu_decode_string_offsets, ctx.handle, be.ptr, avg, s, e, out.ptr, mem)
            assert code == capi.OK, msg
            assert out.get().view(np.uint32).tolist() == oracle.decode_string_offsets(enc, avg, s, e).tolist(), (avg, s, e)
        for n in (1, 2, 600):
            be, bs, bl = Buf(device, enc[:n]), Buf(device, nbytes=4 * n), Buf(device, nbytes=4 * n, shift=4)
            code, msg = _call(ctx.lib.ytgpu_decode_string_pointers_and_lengths, ctx.handle, be.ptr, avg, n, bs.ptr, bl.ptr, mem)
            assert code == capi.OK, msg
            st, ln = oracle.decode_string_pointers_and_lengths(enc[:n], avg)
            assert bs.get().view(np.uint32).tolist() == st.tolist() and bl.get().view(np.int32).tolist() == ln.tolist(), (avg, n)


# ================================================================================================================ tripwires
def _source(path):
    with open(path) as f:
        return re.sub(r"\s+", " ", f.read())


def test_restated_constants_match_the_sources():
    s2c = _source(os.path.join(CSRC, "string_to_ch.cu"))
    assert f"constexpr u32 kShortValue = {SHORT_VALUE};" in s2c
    assert "const bool is_long = valid && len > kShortValue;" in s2c  # a value of exactly 48 bytes is short
    assert f"const u32 skew = (u32)(reinterpret_cast<uintptr_t>(out + p0) & {ALIGN - 1});" in s2c
    flags = _source(os.path.join(CSRC, "columnar_flags.cu"))
    assert f"const u64 full = rows / {VEC_STEP};" in flags and f"done = rows / {VEC_STEP} * {VEC_STEP};" in flags
    assert f"if ((reinterpret_cast<uintptr_t>(first) & {ALIGN - 1}) == 0 && rows >= {VEC_STEP}) {{" in flags
    ch = _source(os.path.join(CSRC, "ch_convert.cu"))
    assert f"(reinterpret_cast<uintptr_t>(out) & {ALIGN - 1})" in ch
    # the block decoders compare a string length with the bytes left and refuse lengths and types that do not fit
    blk = _source(os.path.join(CSRC, "block_codec.cu"))
    assert "len >= (1ull << 32) || len > (u64)(end - p - n)" in blk and "type > 0xff" in blk
    orc = _source(os.path.join(HERE, "..", "oracle", "yt_oracle.cpp"))
    assert "len >= (1ull << 32) || len > (u64)(end - p)" in orc and "type > 0xff" in orc
