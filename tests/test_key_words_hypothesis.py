"""Property test (hypothesis) of the width-free key words (csrc/keys.cuh) that order rowset keys too wide for the
fixed-width normalised form: for any rowset of up to three key columns of the value kinds the reference can order, with
short strings and long ones (shared prefixes, embedded zeros, lengths around multiples of 7), ascending or descending,
required or not, declared or `type = 0`, sorting rows by their concatenated key words (ytgpu_hostcheck_key_words, the
host-compiled __host__ __device__ code the refinement sort runs) gives exactly the reference comparator's stable order."""
import ctypes as C

import numpy as np
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

import oracle
from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import EValueType, Sentinel, U64, make_rowset

DOUBLES = [0.0, -0.0, 1.5, -1.5, float("inf"), float("-inf"), float("nan"), 5e-324, -5e-324, 1.7976931348623157e308]
PREFIXES = [b"", b"x" * 300, b"http://example.com/" + b"\x00" * 250, bytes(range(256)) * 4]


def _long_string(prefix, n, fill):
    """250..2000 bytes: the prefix, then `fill` repeated."""
    return (prefix + fill * 2000)[: max(250, min(2000, len(prefix) + n))]


long_string = st.builds(_long_string, st.sampled_from(PREFIXES),
                        st.one_of(st.integers(0, 2000), st.sampled_from([7 * k + d for k in (36, 37, 143, 144) for d in (-1, 0, 1)])),
                        st.sampled_from([b"a", b"\x00", b"ab\x00", b"\xff"]))

scalar = st.one_of(
    st.none(),
    st.integers(-2**63, 2**63 - 1),
    st.integers(-3, 3),
    st.builds(U64, st.integers(0, 2**64 - 1)),
    st.sampled_from(DOUBLES),
    st.booleans(),
    st.just(Sentinel(EValueType.Min)),
    st.just(Sentinel(EValueType.Max)),
)
short_string = st.one_of(st.binary(max_size=40),
                         st.sampled_from([b"", b"\x00", b"a", b"a\x00", b"abcdefg", b"abcdefg\x00", b"abcdefgh", b"\xff"]))
any_value = st.one_of(scalar, short_string, long_string)

# a column: (declared type, descending, required, value strategy)
column = st.one_of(
    st.tuples(st.just(0), st.booleans(), st.just(False), st.just(any_value)),
    st.tuples(st.just(capi.TYPE_STRING), st.booleans(), st.booleans(), st.just(st.one_of(short_string, long_string))),
    st.tuples(st.just(capi.TYPE_INT64), st.booleans(), st.booleans(), st.just(st.integers(-3, 3))),
)


def key_words(rs, cols):
    lib = capi.load()
    lib.ytgpu_hostcheck_key_words.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint64, C.POINTER(capi.SortSpec),
                                              C.c_void_p, C.c_uint64, C.c_void_p, C.POINTER(C.c_uint32)]
    spec = capi.make_sort_spec(cols)
    n = rs.row_count
    cap = n * (len(cols) * (2000 // 7 + 3))
    words = np.zeros(cap, dtype=np.uint64)
    offs = np.zeros(n + 1, dtype=np.uint64)
    err = C.c_uint32(0)
    vals, heap = np.ascontiguousarray(rs.values), np.ascontiguousarray(rs.heap)
    code = lib.ytgpu_hostcheck_key_words(C.c_void_p(vals.ctypes.data), C.c_uint32(rs.value_count), C.c_void_p(heap.ctypes.data),
                                         C.c_uint64(n), C.byref(spec), C.c_void_p(words.ctypes.data), C.c_uint64(cap),
                                         C.c_void_p(offs.ctypes.data), C.byref(err))
    assert code == 0 and err.value == 0
    return [tuple(int(w) for w in words[offs[i]:offs[i + 1]]) for i in range(n)]


@settings(max_examples=400, deadline=None, suppress_health_check=[HealthCheck.too_slow])
@given(st.lists(column, min_size=1, max_size=3).flatmap(
    lambda cs: st.tuples(st.just(cs), st.lists(st.tuples(*[c[3] for c in cs]), min_size=1, max_size=30))))
def test_key_words_order_like_the_reference_comparator(case):
    cs, rows = case
    k = len(cs)
    rows = [list(r) for r in rows]
    # a required declared column holds no Null (that is a schema violation, not an ordering question)
    for r in rows:
        for i, (typ, _, req, _) in enumerate(cs):
            if typ and req and r[i] is None:
                r[i] = b"" if typ == capi.TYPE_STRING else 0
    rs = make_rowset(rows, ncols=k)
    cols = [dict(index=i, type=cs[i][0], width=0, descending=int(cs[i][1]), required=int(cs[i][2])) for i in range(k)]
    words = key_words(rs, cols)
    order = sorted(range(len(rows)), key=lambda i: words[i])
    perm, _ = oracle.sort_rows(rs.values, rs.heap, k, [int(c[1]) for c in cs], oracle.SORT_STABLE)
    assert order == perm.tolist()


def test_string_blocks():
    """The string payload: 7 raw bytes and a tag per block, tag 8 while the string continues."""
    rs = make_rowset([[b""], [b"abcdefg"], [b"abcdefg\x00"]], ncols=1)
    w = key_words(rs, [dict(index=0, type=capi.TYPE_STRING, required=1)])
    assert w[0] == (0,)
    assert w[1] == (int.from_bytes(b"abcdefg\x08", "big"), 0)
    assert w[2] == (int.from_bytes(b"abcdefg\x08", "big"), 1)
    # not required: the type byte first, then the tag of block k-1 in the top byte of word k
    w = key_words(rs, [dict(index=0, type=capi.TYPE_STRING)])
    assert w[0] == (0x10 << 56, 0)
    assert w[1] == (int.from_bytes(b"\x10abcdefg", "big"), 8 << 56, 0)
