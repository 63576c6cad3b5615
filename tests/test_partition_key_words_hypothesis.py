"""Property test (hypothesis) of the ordered partitioner over width-free key words (csrc/partition.cu,
ytgpu_hostcheck_partition_ordered_words: the bound encoding and the __host__ __device__ binary search the key-word
kernel runs, compiled for the host): for any rowset of up to three key columns and any list of lower bounds, sorted or
not, the partition index of every row equals the oracle's TOrderedPartitioner::GetPartitionIndex (partitioner.cpp:41-57).

The inputs mix `type = 0` columns holding every scalar kind (NaN, +-0, sentinels, Null), required and optional typed
columns whose bounds may hold another type, descending columns, strings with embedded zeros and shared prefixes (so
bounds are often proper prefixes of keys, or longer than every key), prefix lengths 0..k, inclusive and exclusive bounds,
and duplicate bounds.  Keys of every width are used: the word path does not depend on it."""
import ctypes as C
import itertools

import numpy as np
from hypothesis import HealthCheck, given, settings
from hypothesis import strategies as st

import oracle
from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import EValueType as T, Rowset, Sentinel, U64, VALUE_DTYPE, make_rowset

DOUBLES = [0.0, -0.0, 1.5, -1.5, float("inf"), float("-inf"), float("nan"), 5e-324]
PREFIXES = [b"", b"x" * 300, b"http://example.com/" + b"\x00" * 250, bytes(range(256)) * 4]
FILLS = [b"a", b"\x00", b"ab\x00", b"\xff"]

string = st.one_of(
    st.binary(max_size=20),
    st.sampled_from([b"", b"\x00", b"a", b"a\x00", b"abcdefg", b"abcdefg\x00", b"abcdefgh", b"\xff"]),
    # a cut of prefix + fill: keys and bounds share prefixes, one is often a proper prefix of the other
    st.builds(lambda p, f, n: (p + f * 2100)[:n], st.sampled_from(PREFIXES), st.sampled_from(FILLS),
              st.one_of(st.integers(0, 2100), st.sampled_from([7 * k + d for k in (36, 37, 143) for d in (-1, 0, 1)]))),
)
int64 = st.one_of(st.integers(-3, 3), st.integers(-2**63, 2**63 - 1))
scalar = st.one_of(
    st.none(), int64, st.builds(U64, st.integers(0, 2**64 - 1)), st.sampled_from(DOUBLES), st.booleans(),
    st.just(Sentinel(T.Min)), st.just(Sentinel(T.Max)),
)
any_value = st.one_of(scalar, string)

# a column: (declared type, descending, required)
column = st.one_of(
    st.tuples(st.just(0), st.booleans(), st.just(False)),
    st.tuples(st.just(T.String), st.booleans(), st.booleans()),
    st.tuples(st.just(T.Int64), st.booleans(), st.booleans()),
)


def key_value(col):
    typ, _, req = col
    if typ == 0:
        return any_value
    v = string if typ == T.String else int64
    return v if req else st.one_of(v, st.none())


def bound_value(col):
    # a bound may hold any type, the declared one or not
    return st.one_of(key_value(col), any_value)


def valid_key_value(col, x):
    typ, _, req = col
    if typ == 0:
        return True
    if x is None:
        return not req
    return isinstance(x, bytes) if typ == T.String else (isinstance(x, int) and not isinstance(x, bool))


@st.composite
def cases(draw):
    cs = draw(st.lists(column, min_size=1, max_size=3))
    k = len(cs)
    rows = draw(st.lists(st.tuples(*[key_value(c) for c in cs]), min_size=1, max_size=30))
    bounds = draw(st.lists(st.tuples(*[bound_value(c) for c in cs]), min_size=0, max_size=8))
    if bounds and draw(st.booleans()):
        bounds.append(bounds[draw(st.integers(0, len(bounds) - 1))])
    # keys equal to a bound (or to its prefix), where the bound's values are valid keys
    for b in bounds:
        if draw(st.booleans()):
            rows.append(tuple(x if valid_key_value(c, x) else draw(key_value(c)) for c, x in zip(cs, b)))
    blen = [draw(st.integers(0, k)) for _ in bounds]
    binc = [int(draw(st.booleans())) for _ in bounds]
    return cs, [list(r) for r in rows], [list(b) for b in bounds], blen, binc, draw(st.booleans())


def words_partition(rs, cols, bounds, blen, binc):
    from ytsaurus_b200.runtime import GpuContext
    lib = capi.load()
    spec = GpuContext._partition_spec(None, capi.PARTITION_ORDERED, len(blen), key_columns=cols, bounds=bounds,
                                      bound_prefix_length=blen, bound_inclusive=binc)
    out = np.zeros(rs.row_count, dtype=np.int32)
    vals, heap = np.ascontiguousarray(rs.values), np.ascontiguousarray(rs.heap)
    code = lib.ytgpu_hostcheck_partition_ordered_words(C.c_void_p(vals.ctypes.data), C.c_uint32(rs.value_count),
                                                       C.c_void_p(heap.ctypes.data), C.c_uint64(rs.row_count),
                                                       C.byref(spec), C.c_void_p(out.ctypes.data))
    return code, out


@settings(max_examples=400, deadline=None, suppress_health_check=[HealthCheck.too_slow])
@given(cases())
def test_key_word_partitioner_matches_the_oracle(case):
    cs, rows, braw, blen, binc, sort_bounds = case
    k = len(cs)
    desc = [int(c[1]) for c in cs]
    rs = make_rowset(rows, ncols=k)
    bs = make_rowset(braw, ncols=k) if braw else Rowset(np.zeros((0, k), dtype=VALUE_DTYPE), np.zeros(1, np.uint8))
    if sort_bounds and braw:
        perm, _ = oracle.sort_rows(bs.values, bs.heap, k, desc, oracle.SORT_STABLE)
        bs = bs.take(perm)
        blen = [blen[i] for i in perm]
        binc = [binc[i] for i in perm]
    # bound 0 is universal (TOrderedPartitioner needs every key at or above the first bound)
    bounds = Rowset(np.concatenate([np.zeros((1, k), dtype=VALUE_DTYPE), bs.values]), bs.heap)
    blen, binc = [0] + blen, [1] + binc
    want, _ = oracle.partition_ordered(rs.values, rs.heap, k, desc, bounds.values, bounds.heap, blen, binc)
    cols = [dict(index=i, type=cs[i][0], width=0, descending=desc[i], required=int(cs[i][2])) for i in range(k)]
    code, got = words_partition(rs, cols, bounds, blen, binc)
    assert code == 0
    assert got.tolist() == want.tolist()


# comparator_ut.cpp:110-165 (StressNewAndLegacyTestEquivalence), as test_comparator_properties.py states it: every key
# of length 3 over {Null, 0, 1} and every lower bound of prefix length 0..3, inclusive or not; TestKey holds exactly when
# key[:len] >= prefix (inclusive) or key[:len] > prefix (exclusive), in value order Null < 0 < 1.
VALUES = [None, 0, 1]
RANK = {None: (0, 0), 0: (1, 0), 1: (1, 1)}


def _expected(keys, prefix, inclusive, desc):
    out = []
    for key in keys:
        c = 0
        for i, b in enumerate(prefix):
            c = (RANK[key[i]] > RANK[b]) - (RANK[key[i]] < RANK[b])
            c = -c if desc[i] else c
            if c:
                break
        out.append(int(c >= 0 if inclusive else c > 0))
    return out


def test_comparator_stress_on_key_words():
    keys = list(itertools.product(VALUES, repeat=3))
    ks = make_rowset([list(key) for key in keys], ncols=3)
    for desc in [(0, 0, 0), (1, 0, 0), (0, 1, 1)]:
        cols = [dict(index=i, type=0, width=0, descending=desc[i]) for i in range(3)]
        for length in range(4):
            for prefix in itertools.product(VALUES, repeat=length):
                for inclusive in (True, False):
                    bounds = make_rowset([[None] * 3, list(prefix) + [None] * (3 - length)], ncols=3)
                    code, got = words_partition(ks, cols, bounds, [0, length], [1, int(inclusive)])
                    assert code == 0
                    assert got.tolist() == _expected(keys, prefix, inclusive, desc), (prefix, inclusive, desc)


def test_bound_errors():
    """The width-free rules of the normalised bound encoding: Any values and over-long prefixes are rejected."""
    rs = make_rowset([[b"k" * 300, 1]])
    cols = [dict(index=0, type=T.String), dict(index=1, type=T.Int64)]
    bounds = make_rowset([[None, None], [b"a", 1]])
    bounds.values["type"][1, 1] = T.Any
    code, _ = words_partition(rs, cols, bounds, [0, 2], [1, 1])
    assert code == capi.ERR_UNSUPPORTED
    code, _ = words_partition(rs, cols[:1], make_rowset([[None, None], [b"a", 1]]), [0, 2], [1, 1])
    assert code == capi.ERR_INVALID_ARGUMENT
    # a below-first-bound key comes back as -1 (the kernel reports it as "Partition index is out of bounds")
    code, got = words_partition(rs, cols, make_rowset([[b"z", 0]]), [1], [1])
    assert code == 0 and got.tolist() == [-1]
