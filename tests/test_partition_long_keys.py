"""Ordered partitioning of rowsets whose key does not fit the 256-byte normalised form: the key-word kernel
(csrc/partition.cu, partition_words_kernel) against the oracle's TOrderedPartitioner bit for bit, with the histogram
equal to the bincount of the indices, in the HOST and DEVICE memory flavours.  `last_partition_key_words` tells which
path ran: 1 for key words, 0 for normalised keys."""
import numpy as np
import pytest

import oracle
from ytsaurus_b200 import capi
from ytsaurus_b200.rowset import EValueType as T, Rowset, VALUE_DTYPE, make_rowset

pytestmark = pytest.mark.gpu


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


def url_rowset(rng, n, alphabet=b"abcdefghijklmnop", max_len=None, int_first=False):
    """[key: string, i: int64] (or [int64 in -2..2, key] with int_first).  A key is the start of one of 20000 pool
    chunks, each a host prefix of 28 bytes and 2000 letters of `alphabet`, 28..628 bytes long (cut to max_len): keys
    share host prefixes, keys from one chunk are prefixes of each other, and some are exact duplicates."""
    hosts = np.frombuffer(b"".join(b"https://host%03d.example.org/" % i for i in range(64)), np.uint8).reshape(64, 28)
    chunks = 20000
    pool = np.frombuffer(alphabet, np.uint8)[rng.integers(0, len(alphabet), (chunks, 28 + 2000))]
    pool[:, :28] = hosts[rng.integers(0, 64, chunks)]
    klen = 28 + rng.integers(0, 601, n)
    if max_len is not None:
        klen = np.minimum(klen, max_len)
    vals = np.zeros((n, 2), dtype=VALUE_DTYPE)
    s, i = (1, 0) if int_first else (0, 1)
    vals["id"][:, 1] = 1
    vals["type"][:, s] = T.String
    vals["length"][:, s] = klen
    vals["data"][:, s] = rng.integers(0, chunks, n) * pool.shape[1]
    vals["type"][:, i] = T.Int64
    vals["data"][:, i] = (rng.integers(-2, 3, n) if int_first else np.arange(n)).astype(np.int64).view(np.uint64)
    return Rowset(vals, pool.reshape(-1).copy())


def sample_bounds(rng, rs, k, desc, P, blens=(1,), inclusive=None):
    """Bound 0 universal; bound j = the (j*m/P)-th key of a sorted sample of m <= 10^4 rows, prefix length from `blens`,
    inclusive at random unless given."""
    m = min(rs.row_count, 10000)
    sample = rs.take(np.sort(rng.choice(rs.row_count, m, replace=False)))
    perm, _ = oracle.sort_rows(sample.values, sample.heap, k, desc, oracle.SORT_STABLE)
    picks = sample.values[perm.astype(np.int64)][[(j * m) // P for j in range(1, P)]]
    bounds = Rowset(np.concatenate([np.zeros((1, rs.value_count), dtype=VALUE_DTYPE), picks]), rs.heap)
    blen = [0] + [int(rng.choice(blens)) for _ in range(P - 1)]
    binc = [1] + [int(rng.integers(0, 2)) if inclusive is None else int(inclusive) for _ in range(P - 1)]
    return bounds, blen, binc


def spec_for(ctx, cols, bounds, blen, binc):
    return ctx._partition_spec(capi.PARTITION_ORDERED, len(blen), key_columns=cols, bounds=bounds,
                               bound_prefix_length=blen, bound_inclusive=binc)


def check_partition(ctx, rs, cols, bounds, blen, binc, key_words=True):
    k = len(cols)
    assert [c["index"] for c in cols] == list(range(k))
    want, _ = oracle.partition_ordered(rs.values, rs.heap, k, [c.get("descending", 0) for c in cols], bounds.values,
                                       bounds.heap, blen, binc)
    spec = spec_for(ctx, cols, bounds, blen, binc)
    dv, dh = _dev(rs)
    for device in (False, True):
        idx, hist = ctx.partition_rowset(*((dv, dh) if device else (rs.values, rs.heap)), spec)
        if device:
            idx, hist = idx.cpu().numpy(), hist.cpu().numpy().view(np.uint64)
        assert (idx == want).all(), device
        assert hist.tolist() == np.bincount(want, minlength=len(blen)).tolist(), device
        assert ctx.get_option("last_partition_key_words") == int(key_words)
    return want


@pytest.mark.parametrize("desc", [0, 1])
@pytest.mark.parametrize("required", [0, 1])
def test_one_long_string_column(ctx, desc, required):
    rng = np.random.default_rng(1 + 2 * desc + required)
    rs = url_rowset(rng, 20000, alphabet=b"ab\x00")
    cols = [dict(index=0, type=T.String, descending=desc, required=required)]
    bounds, blen, binc = sample_bounds(rng, rs, 1, [desc], 7)
    check_partition(ctx, rs, cols, bounds, blen, binc)


@pytest.mark.parametrize("P", [7, 1000])
def test_long_string_then_int64(ctx, P):
    rng = np.random.default_rng(10 + P)
    rs = url_rowset(rng, 30000)
    rs.values["data"][:, 1] = rng.integers(-3, 3, rs.row_count).astype(np.int64).view(np.uint64)
    cols = [dict(index=0, type=T.String), dict(index=1, type=T.Int64)]
    bounds, blen, binc = sample_bounds(rng, rs, 2, [0, 0], P, blens=(1, 2))
    check_partition(ctx, rs, cols, bounds, blen, binc)


@pytest.mark.parametrize("P", [7, 1000])
def test_int64_desc_then_long_string(ctx, P):
    rng = np.random.default_rng(20 + P)
    rs = url_rowset(rng, 30000, int_first=True)
    cols = [dict(index=0, type=T.Int64, descending=1, required=1), dict(index=1, type=T.String)]
    bounds, blen, binc = sample_bounds(rng, rs, 2, [1, 0], P, blens=(1, 2))
    check_partition(ctx, rs, cols, bounds, blen, binc)


@pytest.mark.parametrize("P", [2, 7, 1000, 5000])
def test_partition_counts(ctx, P):
    """P <= 4096 counts in shared memory, P = 5000 in global memory."""
    rng = np.random.default_rng(30 + P)
    rs = url_rowset(rng, 40000)
    bounds, blen, binc = sample_bounds(rng, rs, 1, [0], P)
    check_partition(ctx, rs, [dict(index=0, type=T.String)], bounds, blen, binc)


def test_million_rows(ctx):
    rng = np.random.default_rng(40)
    rs = url_rowset(rng, 1_000_000)
    bounds, blen, binc = sample_bounds(rng, rs, 1, [0], 1000)
    check_partition(ctx, rs, [dict(index=0, type=T.String)], bounds, blen, binc)


def test_slabs(ctx):
    rng = np.random.default_rng(50)
    rs = url_rowset(rng, 30000)
    cols = [dict(index=0, type=T.String), dict(index=1, type=T.Int64)]
    bounds, blen, binc = sample_bounds(rng, rs, 2, [0, 0], 13, blens=(1, 2))
    want, _ = oracle.partition_ordered(rs.values, rs.heap, 2, None, bounds.values, bounds.heap, blen, binc)
    order = np.argsort(want, kind="stable")
    spec = spec_for(ctx, cols, bounds, blen, binc)
    dv, dh = _dev(rs)
    for device in (False, True):
        idx, hist, slab, perm = ctx.partition_rowset_slabs(*((dv, dh) if device else (rs.values, rs.heap)), spec)
        if device:
            idx, hist, perm = idx.cpu().numpy(), hist.cpu().numpy().view(np.uint64), perm.cpu().numpy().view(np.uint32)
            slab = slab.cpu().numpy().view(VALUE_DTYPE).reshape(rs.values.shape)
        assert (idx == want).all()
        assert hist.tolist() == np.bincount(want, minlength=13).tolist()
        assert perm.tolist() == order.tolist()
        assert slab.tobytes() == rs.values[order].tobytes()
        assert ctx.get_option("last_partition_key_words") == 1


@pytest.mark.parametrize("desc", [0, 1])
def test_partitioned_sort_end_to_end(ctx, desc):
    """Partition job -> one sort per partition -> concatenation: the stable sort of the whole URL-keyed table."""
    import torch
    rng = np.random.default_rng(60 + desc)
    rs = url_rowset(rng, 50000)
    cols = [dict(index=0, type=T.String, descending=desc)]
    bounds, blen, binc = sample_bounds(rng, rs, 1, [desc], 8, inclusive=1)
    dv, dh = _dev(rs)
    _, hist, slab, perm = ctx.partition_rowset_slabs(dv, dh, spec_for(ctx, cols, bounds, blen, binc))
    assert ctx.get_option("last_partition_key_words") == 1
    perm = perm.cpu().numpy().view(np.uint32).astype(np.int64)
    got, start = [], 0
    for count in hist.cpu().numpy().view(np.uint64).tolist():
        if count:
            p = ctx.sort_rowset(slab[start:start + count], dh, cols)
            assert ctx.get_option("last_sort_refine_rounds") >= 1
            got.append(perm[start + p.cpu().numpy().view(np.uint32).astype(np.int64)])
        start += count
    torch.cuda.synchronize()
    want, _ = oracle.sort_rows(rs.values, rs.heap, 1, [desc], oracle.SORT_STABLE)
    assert np.concatenate(got).tolist() == want.tolist()


def test_short_keys_keep_the_normalised_path(ctx):
    rng = np.random.default_rng(70)
    rs = url_rowset(rng, 30000, max_len=200)
    bounds, blen, binc = sample_bounds(rng, rs, 1, [0], 100)
    check_partition(ctx, rs, [dict(index=0, type=T.String)], bounds, blen, binc, key_words=False)


def _error(ctx, rs, cols, bounds, blen, binc):
    with pytest.raises(capi.YtGpuError) as e:
        ctx.partition_rowset(rs.values, rs.heap, spec_for(ctx, cols, bounds, blen, binc))
    return e.value


@pytest.mark.parametrize("long", [False, True])
def test_errors_match_the_normalised_path(ctx, long):
    big = b"x" * (400 if long else 150)
    width = 300 if long else 100
    rs = make_rowset([[b"a" * 20, 1], [big, 2], [b"c", 3]])
    universal = make_rowset([[None, None], [b"b", 0]])
    # a string longer than the declared width
    e = _error(ctx, rs, [dict(index=0, type=T.String, width=width)], universal, [0, 1], [1, 1])
    assert e.code == capi.ERR_SCHEMA_VIOLATION and "longer than the declared" in e.message
    # an Any key value
    bad = make_rowset([[big, 1], [b"y", 2]])
    bad.values["type"][1, 0] = T.Any
    assert _error(ctx, bad, [dict(index=0, type=0)], universal, [0, 1], [1, 1]).code == capi.ERR_UNSUPPORTED
    # an Any bound value
    abound = make_rowset([[None, None], [b"b", 0]])
    abound.values["type"][1, 0] = T.Any
    assert _error(ctx, rs, [dict(index=0, type=T.String)], abound, [0, 1], [1, 1]).code == capi.ERR_UNSUPPORTED
    # no universal first bound: "a"*20 < "b"
    e = _error(ctx, rs, [dict(index=0, type=T.String)], make_rowset([[b"b", 0]]), [1], [1])
    assert e.code == capi.ERR_PARTITION_OUT_OF_BOUNDS and "Partition index is out of bounds" in e.message
    assert ctx.get_option("last_partition_key_words") == int(long)
