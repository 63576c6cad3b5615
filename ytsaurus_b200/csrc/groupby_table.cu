// groupby_table.cu — a GROUP BY table kept on the device and updated block by block (ytgpu_groupby_table_*).
//
// The one-shot GROUP BY (groupby_multi.cu) stores in each slot the row that claimed it and compares tuples by decoding
// that row again, so its state cannot outlive the call.  The table owns everything instead, indexed by a dense group id:
// the key words and null mask of each group, COUNT(*), the global first row, every aggregate's state, an open-addressing
// slot table slot -> group id, and per string key a growing dictionary (string_dict.cuh).  One update:
//   1. string keys -> dictionary ids: a read-only lookup of every row (its bounds checks are read before anything
//      changes), then the values the dictionary lacks are appended in first-row order (string_dict_append);
//   2. block-local groups: the one-shot's assign step (assign_key_slots, unchanged) over the block's tuples, the string
//      ids as UINT64 key columns, and the one-shot's per-aggregate accumulation (accumulate_scalar) into block-slot states;
//      the occupied block slots are compacted (mg_compact_kernel);
//   3. merge: every block group looks its tuple up in the table (read-only); the misses get new ids, their key words are
//      written and then inserted by CAS on empty slots only, so no probe compares against a half-written tuple; the block
//      states are folded into the group states, one thread per block group (block groups are distinct groups):
//      sums / counts add, MIN / MAX keep the bound, ARGMIN / ARGMAX move only on a strictly better block bound (the
//      block's own first attaining row, so an earlier block keeps a tie), FIRST is set once.  The selected row's value
//      is captured from the block then, so the table never reads a block again.
// String-valued aggregates (MIN / MAX / FIRST of a string, ARGMIN / ARGMAX with a string value or bound) own the bytes
// they selected: per group one or two (start, length) pairs into the aggregate's own device heap, the value and, for a
// string bound, the bound (MIN / MAX: one string, both).  Their block step is the one-shot's mg_accumulate_strings_kernel;
// the fold decides per block group whether the block's row replaces the group's (gt_string_decide_kernel, read-only, run
// with the lookup so that the bytes it needs are read in the same copy as the count of new groups), then appends the new
// values to the heap (gt_string_take_kernel).  Replaced values stay in the heap until it holds more than kReclaimFactor x
// the live bytes; it is then compacted in group-id order (gt_owned_lengths_kernel, scan, gt_owned_compact_kernel).
// The result orders the groups by first row with the radix sort and finalises them as the one-shot does.
#include <algorithm>
#include <new>
#include <vector>

#include "columnar.cuh"
#include "context.cuh"
#include "groupby_agg.cuh"
#include "key_tuple.cuh"
#include "radix_sort.cuh"
#include "scan.cuh"
#include "string_dict.cuh"

using namespace ytgpu;

namespace {

constexpr u64 kMaxUpdateRows = 1ull << 30;
constexpr u64 kMaxGroups = (1ull << 30) - 1;  // the result goes through the radix sort, which takes fewer than 2^30 rows
// An aggregate's string heap is compacted once its used bytes exceed kReclaimFactor x its live bytes and kReclaimMinBytes.
constexpr u64 kReclaimFactor = 2;
constexpr u64 kReclaimMinBytes = 1ull << 20;

// The table's key words: component k of group g at w[k][g] (NULL as 0), null mask bit k.
struct OwnedKeys {
    u64* w[kMaxGroupKeys];
    u32* nulls;
    u32 count;
};

__device__ __forceinline__ KeyTuple load_owned(const OwnedKeys& O, u32 g) {
    KeyTuple t;
    t.nulls = O.nulls[g];
#pragma unroll
    for (u32 k = 0; k < (u32)kMaxGroupKeys; ++k) t.w[k] = k < O.count ? O.w[k][g] : 0;
    return t;
}

// Merge, step 1 (read-only): gid[j] = the table's group of block group j's tuple, kNoSlot when the table lacks it.
__global__ void __launch_bounds__(256) gt_lookup_kernel(const KeyColumns K, const u64* __restrict__ bfirst, u64 gb, const OwnedKeys O,
                                                        const u32* __restrict__ slots, u64 mask, u32* __restrict__ gid) {
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < gb; j += (u64)gridDim.x * blockDim.x) {
        const KeyTuple t = load_tuple(K, bfirst[j]);
        u64 b = hash_tuple(K, t) & mask;
        u32 found = kNoSlot;
        for (u64 probes = 0; probes <= mask; ++probes) {
            const u32 s = slots[b];
            if (s == kNoSlot) break;
            if (same_tuple(K, t, load_owned(O, s))) {
                found = s;
                break;
            }
            b = (b + 1) & mask;
        }
        gid[j] = found;
    }
}

// Merge, step 2: the misses get ids groups + rank (rank: the exclusive scan of the miss flags, in compaction order), their
// key words, COUNT(*) 0 and first row; then their slots by CAS on empty slots (the tuples are distinct and new).
__global__ void __launch_bounds__(256) gt_insert_kernel(const KeyColumns K, const u64* __restrict__ bfirst, u64 gb, u64 row_base, u64 groups,
                                                        const u64* __restrict__ rank, OwnedKeys O, unsigned long long* counts,
                                                        unsigned long long* first, u32* slots, u64 mask, u32* __restrict__ gid) {
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < gb; j += (u64)gridDim.x * blockDim.x) {
        if (gid[j] != kNoSlot) continue;
        const u32 g = (u32)(groups + rank[j]);
        const KeyTuple t = load_tuple(K, bfirst[j]);
#pragma unroll
        for (u32 k = 0; k < (u32)kMaxGroupKeys; ++k)
            if (k < O.count) O.w[k][g] = t.w[k];
        O.nulls[g] = t.nulls;
        counts[g] = 0;
        first[g] = row_base + bfirst[j];
        u64 b = hash_tuple(K, t) & mask;
        while (atomicCAS(&slots[b], kNoSlot, g) != kNoSlot) b = (b + 1) & mask;
        gid[j] = g;
    }
}

__global__ void __launch_bounds__(256) gt_miss_flags_kernel(const u32* __restrict__ gid, u64 gb, u64* __restrict__ flags) {
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j <= gb; j += (u64)gridDim.x * blockDim.x) flags[j] = j < gb && gid[j] == kNoSlot;
}

// The slots of a grown table, from the owned key words.
__global__ void __launch_bounds__(256) gt_rehash_kernel(const OwnedKeys O, u64 groups, u32* slots, u64 mask) {
    KeyColumns K{};
    K.count = O.count;
    for (u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += (u64)gridDim.x * blockDim.x) {
        u64 b = hash_tuple(K, load_owned(O, (u32)g)) & mask;
        while (atomicCAS(&slots[b], kNoSlot, (u32)g) != kNoSlot) b = (b + 1) & mask;
    }
}

// A group's state for one aggregate: acc / nn as the one-shot's, row = the selected GLOBAL row (~0 = none) and val = the
// value captured there (FIRST / ARGMIN / ARGMAX).
struct GroupState {
    unsigned long long* acc;
    unsigned long long* nn;
    unsigned long long* row;
    u64* val;
};

// Merge, step 3: COUNT(*), then one aggregate's block state folded into the group state, per block group.
__global__ void __launch_bounds__(256) gt_merge_kernel(int op, const ColumnDev col, u64 gb, const u32* __restrict__ bslot,
                                                       const u32* __restrict__ gid, u64 row_base, AggState B, GroupState G) {
    const u8 vtype = col.value_type;
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < gb; j += (u64)gridDim.x * blockDim.x) {
        const u32 s = bslot[j], g = gid[j];
        switch (op) {
            case YTGPU_AGG_SUM:
            case YTGPU_AGG_AVG:
                if (vtype == YTGPU_TYPE_DOUBLE)
                    G.acc[g] = (u64)__double_as_longlong(__longlong_as_double((long long)G.acc[g]) + __longlong_as_double((long long)B.acc[s]));
                else G.acc[g] += B.acc[s];
                G.nn[g] += B.nn[s];
                break;
            case YTGPU_AGG_COUNT:
                G.nn[g] += B.nn[s];
                break;
            case YTGPU_AGG_MIN:
            case YTGPU_AGG_MAX:
                if (B.nn[s]) {
                    G.acc[g] = op == YTGPU_AGG_MIN ? min(G.acc[g], B.acc[s]) : max(G.acc[g], B.acc[s]);
                    G.nn[g] = 1;
                }
                break;
            case YTGPU_AGG_ARGMIN:
            case YTGPU_AGG_ARGMAX: {
                if (!B.nn[s]) break;
                const u64 e = B.acc[s];
                const bool better = !G.nn[g] || (op == YTGPU_AGG_ARGMIN ? e < G.acc[g] : e > G.acc[g]);  // a tie keeps the earlier block
                if (better) {
                    bool nul;
                    G.acc[g] = e;
                    G.nn[g] = 1;
                    G.row[g] = row_base + B.row[s];
                    G.val[g] = decode_at(col, (i64)B.row[s], &nul);
                }
                break;
            }
            case YTGPU_AGG_FIRST:
                if (G.row[g] == ~0ull && B.row[s] != ~0ull) {
                    bool nul;
                    G.row[g] = row_base + B.row[s];
                    G.val[g] = decode_at(col, (i64)B.row[s], &nul);
                }
                break;
            default:
                break;
        }
    }
}

__global__ void __launch_bounds__(256) gt_count_kernel(u64 gb, const u32* __restrict__ bslot, const u32* __restrict__ gid,
                                                       const unsigned long long* __restrict__ bcounts, unsigned long long* counts) {
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < gb; j += (u64)gridDim.x * blockDim.x) counts[gid[j]] += bcounts[bslot[j]];
}

// A string-valued aggregate's owned strings: string k of group g is len[k][g] bytes at heap + start[k][g].
struct OwnedStrings {
    u8* heap;
    u64* start[2];
    u32* len[2];
    // k may vary at run time: selected, not indexed, so the arrays stay out of local memory
    __device__ __forceinline__ u64* starts(u32 k) const { return k ? start[1] : start[0]; }
    __device__ __forceinline__ u32* lens(u32 k) const { return k ? len[1] : len[0]; }
};

// The same aggregate's strings in the block: owned string k of the block's row r is s[k] at r (bounds-checked before
// the update changed anything).  key: the owned string that orders the selection (MIN / MAX, ARGMIN / ARGMAX by a
// string), -1 for a scalar bound (in the group's acc, by_encode'd) or none (FIRST); value: owned string 0 is the result.
struct BlockStrings {
    StringDev s[2];
    u32 count;
    int key;
    bool value;
};

__device__ __forceinline__ ytgpu_value owned_value(const OwnedStrings& O, int k, u32 g) {
    ytgpu_value v{};
    v.type = YTGPU_TYPE_STRING;
    v.length = O.lens(k)[g];
    v.data = O.starts(k)[g];
    return v;
}

// Fold, step 1 (read-only, before the table grows): take[j] = block group j's row replaces its group's selection (a group
// new in this block, gid kNoSlot, always takes it), need[j] = the bytes that appends (need[gb] = 0 for the scan), and the
// bytes of the values it replaces added to *freed.  MIN / MAX and ARGMIN / ARGMAX replace only on a strictly better
// value or bound, so an earlier block keeps a tie; FIRST is set once.
__global__ void __launch_bounds__(256) gt_string_decide_kernel(int op, const ColumnDev by, const BlockStrings B, u64 gb, const u32* __restrict__ bslot,
                                                               const u32* __restrict__ gid, const unsigned long long* __restrict__ brow,
                                                               const GroupState G, const OwnedStrings O, u8* __restrict__ take,
                                                               u64* __restrict__ need, unsigned long long* freed) {
    const bool larger = op == YTGPU_AGG_MAX || op == YTGPU_AGG_ARGMAX;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    const u64 trips = (gb + 1 + stride - 1) / stride;  // the same for every thread: the warp sum sees whole warps
    u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    for (u64 t = 0; t < trips; ++t, j += stride) {
        u64 gone = 0;
        if (j < gb) {
            const u64 r = brow[bslot[j]];
            const u32 g = gid[j];
            const bool held = g != kNoSlot && G.row[g] != ~0ull;
            bool replace = r != ~0ull && !held;
            if (r != ~0ull && held && op != YTGPU_AGG_FIRST) {
                int c;
                if (B.key >= 0) {
                    const StringDev& k = B.key == 0 ? B.s[0] : B.s[1];
                    c = string_compare2(k.heap, string_of(k, r), O.heap, owned_value(O, B.key, g));
                } else {
                    bool nul;
                    const u64 e = by_encode(by.value_type, decode_at(by, (i64)r, &nul));
                    c = e < G.acc[g] ? -1 : (e > G.acc[g] ? 1 : 0);
                }
                replace = larger ? c > 0 : c < 0;
            }
            u64 bytes = 0;
            if (replace)
#pragma unroll
                for (int k = 0; k < 2; ++k) {
                    if ((u32)k >= B.count) break;
                    bytes += B.s[k].lengths[r];
                    if (held) gone += O.len[k][g];
                }
            take[j] = replace ? 1 : 0;
            need[j] = bytes;
        } else if (j == gb) {
            need[j] = 0;
        }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) gone += __shfl_xor_sync(0xffffffffu, gone, d);
        if ((threadIdx.x & 31) == 0 && gone) atomicAdd(freed, (unsigned long long)gone);
    }
}

// Copies up to N strings per selected item into `to`, a warp per item: item `from` (a lane of the calling warp, its
// `count` sources in heaps[k] at src[k], len[k] bytes, and its destination dst, valid in that lane only) is copied by
// the whole warp.
template <int N>
__device__ __forceinline__ void warp_copy_strings(u32 m, u32 lane, u32 count, const u8* const (&heaps)[N], const u64 (&src)[N],
                                                  const u32 (&len)[N], u64 dst, u8* to) {
    while (m) {
        const int from = __ffs(m) - 1;
        m &= m - 1;
        u64 d = __shfl_sync(0xffffffffu, dst, from);
#pragma unroll
        for (int k = 0; k < N; ++k) {
            if ((u32)k >= count) break;
            const u64 s = __shfl_sync(0xffffffffu, src[k], from);
            const u32 l = __shfl_sync(0xffffffffu, len[k], from);
            for (u32 x = lane; x < l; x += 32) to[d + x] = heaps[k][s + x];
            d += l;
        }
    }
}

// Fold, step 2 (after the heap grew and the new groups got ids): every replacing block group's strings are appended at
// heap + base + at[j] (at: the exclusive scan of need), and its group's start, length, global row and scalar part set.
__global__ void __launch_bounds__(256) gt_string_take_kernel(int op, const ColumnDev col, const ColumnDev by, const BlockStrings B, u64 gb,
                                                             const u32* __restrict__ bslot, const u32* __restrict__ gid,
                                                             const unsigned long long* __restrict__ brow, const u8* __restrict__ take,
                                                             const u64* __restrict__ at, u64 base, u64 row_base, GroupState G, OwnedStrings O) {
    const bool arg = op == YTGPU_AGG_ARGMIN || op == YTGPU_AGG_ARGMAX;
    const u32 lane = threadIdx.x & 31;
    const u64 warps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u8* heaps[2] = {B.s[0].heap, B.s[1].heap};
    for (u64 wbase = (u64)blockIdx.x * blockDim.x + threadIdx.x - lane; wbase < gb; wbase += warps * 32) {
        const u64 j = wbase + lane;
        const bool t = j < gb && take[j];
        u64 dst = 0, src[2] = {0, 0};
        u32 len[2] = {0, 0};
        if (t) {
            const u64 r = brow[bslot[j]];
            const u32 g = gid[j];
            dst = base + at[j];
            u64 o = dst;
#pragma unroll
            for (int k = 0; k < 2; ++k) {
                if ((u32)k >= B.count) break;
                src[k] = B.s[k].starts[r];
                len[k] = B.s[k].lengths[r];
                O.start[k][g] = o;
                O.len[k][g] = len[k];
                o += len[k];
            }
            G.row[g] = row_base + r;
            bool nul;
            if (arg && B.key < 0) G.acc[g] = by_encode(by.value_type, decode_at(by, (i64)r, &nul));
            if (arg && !B.value) G.val[g] = decode_at(col, (i64)r, &nul);
        }
        warp_copy_strings(__ballot_sync(0xffffffffu, t), lane, B.count, heaps, src, len, dst, O.heap);
    }
}

// Compaction: at[v] = the length of owned value v = g * count + k (at[values] = 0), then scanned to its new start.
__global__ void __launch_bounds__(256) gt_owned_lengths_kernel(u64 values, u32 count, const OwnedStrings O, u64* __restrict__ at) {
    for (u64 v = (u64)blockIdx.x * blockDim.x + threadIdx.x; v <= values; v += (u64)gridDim.x * blockDim.x)
        at[v] = v < values ? O.lens((u32)(v % count))[v / count] : 0;
}

// Compaction: every owned value copied to `to` + at[v], a warp per value, and its start moved there.
__global__ void __launch_bounds__(256) gt_owned_compact_kernel(u64 values, u32 count, OwnedStrings O, const u64* __restrict__ at, u8* __restrict__ to) {
    const u32 lane = threadIdx.x & 31;
    const u64 warps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u8* heaps[1] = {O.heap};
    for (u64 wbase = (u64)blockIdx.x * blockDim.x + threadIdx.x - lane; wbase < values; wbase += warps * 32) {
        const u64 v = wbase + lane;
        u64 src[1] = {0};
        u32 len[1] = {0};
        u64 dst = 0;
        if (v < values) {
            const u32 k = (u32)(v % count), g = (u32)(v / count);
            src[0] = O.starts(k)[g];
            len[0] = O.lens(k)[g];
            dst = at[v];
            O.starts(k)[g] = dst;
        }
        warp_copy_strings(__ballot_sync(0xffffffffu, len[0] != 0), lane, 1, heaps, src, len, dst, to);
    }
}

// Every string in the bounds of its heap, else DE_STRING_OUT_OF_HEAP: the string values an update's aggregates read,
// checked before the update changes the table.
__global__ void __launch_bounds__(256) gt_check_strings_kernel(const StringDev c, u64 n, u32* err_word) {
    u32 bad = 0;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        ytgpu_value v;
        string_at(c, i, &v, &bad);
    }
    if (bad) atomicOr(err_word, (u32)DE_STRING_OUT_OF_HEAP);
}

// Result: group ids in output order, keys, COUNT(*), first rows.
struct NumericKeyOutputs {
    u64* keys[kMaxGroupKeys];
    u8* key_null[kMaxGroupKeys];
};
__global__ void __launch_bounds__(256) gt_emit_keys_kernel(const OwnedKeys O, u32 numeric, const SortPlan* plan, const u32* pa, const u32* pb,
                                                           u64 g, const unsigned long long* counts, const unsigned long long* first,
                                                           NumericKeyOutputs out, u64* out_counts, u64* out_first, u32* gid_sorted) {
    const u64 o = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= g) return;
    const u32 id = perm_at(plan, pa, pb, o);
    gid_sorted[o] = id;
    const u32 nulls = O.nulls[id];
    for (u32 k = 0; k < numeric; ++k) {
        out.keys[k][o] = O.w[k][id];
        out.key_null[k][o] = (nulls >> k) & 1;
    }
    if (out_counts) out_counts[o] = counts[id];
    if (out_first) out_first[o] = first[id];
}

// A selecting aggregate's result: the captured value, NULL without a selected row.
__global__ void __launch_bounds__(256) gt_finalize_selected_kernel(u64 g, const u32* __restrict__ gid_sorted, GroupState G, u64* out_value,
                                                                   u8* out_null) {
    const u64 o = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= g) return;
    const u32 id = gid_sorted[o];
    const bool nul = G.row[id] == ~0ull;
    out_value[o] = nul ? 0 : G.val[id];
    out_null[o] = nul ? 1 : 0;
}

// One string per group id for the result: a string key (the group's dictionary id in ids, NULL by its null mask bit) or
// a string-valued aggregate's owned value (ids null: indexed by group id; NULL without a selected row).
struct GroupStrings {
    const u64* ids;
    const u32* nulls;
    u32 bit;
    const unsigned long long* rows;
    const u8* heap;
    const u64* starts;
    const u32* lengths;
    __device__ __forceinline__ bool null_at(u32 id) const { return ids ? (nulls[id] >> bit) & 1 : rows[id] == ~0ull; }
    __device__ __forceinline__ u64 index(u32 id) const { return ids ? ids[id] : id; }
};

// String outputs: lengths (then scanned to starts) and nulls, then the bytes.
__global__ void __launch_bounds__(256) gt_string_lengths_kernel(u64 g, const u32* __restrict__ gid_sorted, const GroupStrings S,
                                                                u64* __restrict__ at, u32* __restrict__ out_len, u8* __restrict__ out_null) {
    for (u64 o = (u64)blockIdx.x * blockDim.x + threadIdx.x; o <= g; o += (u64)gridDim.x * blockDim.x) {
        if (o == g) {
            at[o] = 0;
            continue;
        }
        const u32 id = gid_sorted[o];
        const bool nul = S.null_at(id);
        const u32 len = nul ? 0 : S.lengths[S.index(id)];
        at[o] = len;
        out_len[o] = len;
        out_null[o] = nul ? 1 : 0;
    }
}

__global__ void __launch_bounds__(256) gt_string_copy_kernel(u64 g, const u32* __restrict__ gid_sorted, const GroupStrings S,
                                                             const u64* __restrict__ at, u64* __restrict__ out_starts, u8* __restrict__ out_heap) {
    const u32 lane = threadIdx.x & 31;
    const u64 warps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u8* heaps[1] = {S.heap};
    for (u64 base = (u64)blockIdx.x * blockDim.x + threadIdx.x - lane; base < g; base += warps * 32) {
        const u64 o = base + lane;
        u64 src[1] = {0};
        u32 len[1] = {0};
        u64 dst = 0;
        if (o < g) {
            out_starts[o] = at[o];
            dst = at[o];
            len[0] = (u32)(at[o + 1] - at[o]);
            if (len[0]) src[0] = S.starts[S.index(gid_sorted[o])];
        }
        warp_copy_strings(__ballot_sync(0xffffffffu, len[0] != 0), lane, 1, heaps, src, len, dst, out_heap);
    }
}

// A string-valued aggregate's owned strings (count 1 or 2 per group, see BlockStrings) and its heap: `used` bytes
// written, of which `live` are held by a group.
struct OwnedHeap {
    u32 count = 0;
    int key = -1;
    bool value = false;
    DevBuf<u8> heap;
    DevBuf<u64> start[2];
    DevBuf<u32> len[2];
    u64 used = 0, live = 0;

    OwnedStrings view() { return OwnedStrings{heap.p, {start[0].p, start[1].p}, {len[0].p, len[1].p}}; }
};

struct GroupByTable {
    Context* ctx = nullptr;
    u32 numeric = 0, strings = 0, value_count = 0, aggregate_count = 0;
    u8 key_types[kMaxGroupKeys] = {};
    std::vector<u8> value_types;
    std::vector<ytgpu_aggregate> aggregates;
    u64 hint = 0;
    u64 rows = 0;        // rows of every update so far: the row base of the next
    u64 groups = 0;
    u64 capacity = 0;    // group-indexed arrays
    DevBuf<u64> keys[kMaxGroupKeys];
    DevBuf<u32> nulls;
    DevBuf<unsigned long long> counts, first;
    DevBuf<u32> slots;   // power of two >= 2 x groups
    std::vector<DevBuf<unsigned long long>> acc, nn, row;
    std::vector<DevBuf<u64>> val;
    StringDict dicts[kMaxGroupKeys];
    u64 dict_count[kMaxGroupKeys] = {}, dict_bytes[kMaxGroupKeys] = {};
    u32 string_value_count = 0;
    std::vector<OwnedHeap> heaps;  // per aggregate; count 0 unless string-valued

    OwnedKeys owned() {
        OwnedKeys O{};
        for (u32 k = 0; k < numeric + strings; ++k) O.w[k] = keys[k].p;
        O.nulls = nulls.p;
        O.count = numeric + strings;
        return O;
    }
    GroupState state(u32 a) { return GroupState{acc[a].p, nn[a].p, row[a].p, val[a].p}; }
    bool is_string(int32_t c) const { return (u32)c >= value_count; }
};

bool selects_row(int op) { return op == YTGPU_AGG_ARGMIN || op == YTGPU_AGG_ARGMAX || op == YTGPU_AGG_FIRST; }

// Group-indexed arrays for `want` groups: grown by doubling, the new tail filled with each state's initial value.
Status grow_groups(Context* ctx, GroupByTable* t, u64 want) {
    if (want <= t->capacity) return Status{};
    u64 cap = std::max<u64>(t->capacity, 1024);
    while (cap < want) cap <<= 1;
    const u64 keep = t->groups, tail = cap - keep;
    for (u32 k = 0; k < t->numeric + t->strings; ++k) YTGPU_TRY(grow_buf(ctx, &t->keys[k], keep, cap));
    YTGPU_TRY(grow_buf(ctx, &t->nulls, keep, cap));
    YTGPU_TRY(grow_buf(ctx, &t->counts, keep, cap));
    YTGPU_TRY(grow_buf(ctx, &t->first, keep, cap));
    for (u32 a = 0; a < t->aggregate_count; ++a) {
        const int op = t->aggregates[a].op;
        YTGPU_TRY(grow_buf(ctx, &t->acc[a], keep, cap));
        YTGPU_TRY(grow_buf(ctx, &t->nn[a], keep, cap));
        YTGPU_TRY(grow_buf(ctx, &t->row[a], keep, cap));
        YTGPU_TRY(grow_buf(ctx, &t->val[a], keep, cap));
        const int fill = (op == YTGPU_AGG_MIN || op == YTGPU_AGG_ARGMIN) ? 0xff : 0;
        YTGPU_CUDA_TRY(cudaMemsetAsync(t->acc[a].p + keep, fill, tail * 8, ctx->stream));
        YTGPU_CUDA_TRY(cudaMemsetAsync(t->nn[a].p + keep, 0, tail * 8, ctx->stream));
        YTGPU_CUDA_TRY(cudaMemsetAsync(t->row[a].p + keep, 0xff, tail * 8, ctx->stream));
        YTGPU_CUDA_TRY(cudaMemsetAsync(t->val[a].p + keep, 0, tail * 8, ctx->stream));
        OwnedHeap& H = t->heaps[a];
        for (u32 k = 0; k < H.count; ++k) {
            YTGPU_TRY(grow_buf(ctx, &H.start[k], keep, cap));
            YTGPU_TRY(grow_buf(ctx, &H.len[k], keep, cap));
            YTGPU_CUDA_TRY(cudaMemsetAsync(H.len[k].p + keep, 0, tail * 4, ctx->stream));
        }
    }
    t->capacity = cap;
    return Status{};
}

// The slot table for `want` groups (a power of two >= 2 x want, at least 2048), rehashed from the owned keys when it grows.
Status grow_slots(Context* ctx, GroupByTable* t, u64 want) {
    u64 cap = std::max<u64>(t->slots.n, 2048);
    while (cap < 2 * want) cap <<= 1;
    if (cap == t->slots.n) return Status{};
    YTGPU_TRY(t->slots.allocate(ctx, cap));
    YTGPU_CUDA_TRY(cudaMemsetAsync(t->slots.p, 0xff, cap * 4, ctx->stream));
    if (t->groups) {
        KernelTimer timer(ctx, KC_GROUPBY);
        gt_rehash_kernel<<<blocks_for(t->groups, 256, 8), 256, 0, ctx->stream>>>(t->owned(), t->groups, t->slots.p, cap - 1);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    return Status{};
}

Status create_impl(Context* ctx, const u8* key_types, u32 key_count, u32 string_key_count, const u8* value_types, u32 value_count,
                   u32 string_value_count, const ytgpu_aggregate* aggregates, u32 aggregate_count, u64 hint, GroupByTable** out) {
    if (!out || (key_count && !key_types) || (value_count && !value_types) || (aggregate_count && !aggregates))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    const u64 total = (u64)key_count + string_key_count;
    if (total == 0 || total > (u64)kMaxGroupKeys)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key column count must be in [1, %d]", kMaxGroupKeys);
    if (aggregate_count > (u32)kMaxAggregates) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "at most %d aggregates", kMaxAggregates);
    for (u32 k = 0; k < key_count; ++k)
        if (!aggregatable_type(key_types[k]))
            return make_status(YTGPU_ERR_UNSUPPORTED, "key %u: value type 0x%x is not INT64, UINT64, DOUBLE or BOOLEAN", k, key_types[k]);
    for (u32 a = 0; a < aggregate_count; ++a) {
        const ytgpu_aggregate& A = aggregates[a];
        if (A.op < YTGPU_AGG_SUM || A.op > YTGPU_AGG_FIRST) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "aggregate %u: unknown op %d", a, A.op);
        const bool arg = A.op == YTGPU_AGG_ARGMIN || A.op == YTGPU_AGG_ARGMAX;
        if (A.column < 0 || (arg && A.by_column < 0)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "aggregate %u: column out of range", a);
        // aggregate arguments index value_columns ++ string_values
        const u64 columns = (u64)value_count + string_value_count;
        if ((u64)A.column >= columns || (arg && (u64)A.by_column >= columns)) {
            if (string_value_count == 0)
                return make_status(YTGPU_ERR_UNSUPPORTED, "aggregate %u: only the value columns (no string aggregates) may be aggregated", a);
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "aggregate %u: column out of range", a);
        }
        if ((u32)A.column >= value_count) {
            if (A.op == YTGPU_AGG_SUM || A.op == YTGPU_AGG_AVG)
                return make_status(YTGPU_ERR_UNSUPPORTED, "aggregate %u: sum / avg over a string column", a);
        } else {
            const u8 t = value_types[A.column];
            if (!aggregatable_type(t)) return make_status(YTGPU_ERR_UNSUPPORTED, "aggregate %u: value type 0x%x is not a fixed-width scalar", a, t);
            if ((A.op == YTGPU_AGG_SUM || A.op == YTGPU_AGG_AVG) && t == YTGPU_TYPE_BOOLEAN)
                return make_status(YTGPU_ERR_UNSUPPORTED, "aggregate %u: sum / avg need int64, uint64 or double", a);
        }
        if (arg && (u32)A.by_column < value_count && !aggregatable_type(value_types[A.by_column]))
            return make_status(YTGPU_ERR_UNSUPPORTED, "aggregate %u: by_column is not a fixed-width scalar", a);
    }
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    GroupByTable* t = new (std::nothrow) GroupByTable();
    if (!t) return make_status(YTGPU_ERR_OUT_OF_MEMORY, "host allocation failed");
    t->ctx = ctx;
    t->numeric = key_count;
    t->strings = string_key_count;
    for (u32 k = 0; k < key_count; ++k) t->key_types[k] = key_types[k];
    t->value_count = value_count;
    t->value_types.assign(value_types, value_types + value_count);
    t->aggregate_count = aggregate_count;
    t->aggregates.assign(aggregates, aggregates + aggregate_count);
    t->hint = std::min<u64>(hint, kMaxGroups);
    t->acc = std::vector<DevBuf<unsigned long long>>(aggregate_count);
    t->nn = std::vector<DevBuf<unsigned long long>>(aggregate_count);
    t->row = std::vector<DevBuf<unsigned long long>>(aggregate_count);
    t->val = std::vector<DevBuf<u64>>(aggregate_count);
    t->string_value_count = string_value_count;
    t->heaps = std::vector<OwnedHeap>(aggregate_count);
    for (u32 a = 0; a < aggregate_count; ++a) {
        const ytgpu_aggregate& A = aggregates[a];
        const bool arg = A.op == YTGPU_AGG_ARGMIN || A.op == YTGPU_AGG_ARGMAX;
        const bool col_str = t->is_string(A.column) && A.op != YTGPU_AGG_COUNT, by_str = arg && t->is_string(A.by_column);
        OwnedHeap& H = t->heaps[a];
        H.count = (col_str ? 1 : 0) + (by_str ? 1 : 0);
        H.value = col_str;
        if (A.op == YTGPU_AGG_MIN || A.op == YTGPU_AGG_MAX) H.key = col_str ? 0 : -1;
        else if (by_str) H.key = col_str ? 1 : 0;
    }
    Status s = grow_groups(ctx, t, std::max<u64>(t->hint, 1));
    if (s.code == YTGPU_OK) s = grow_slots(ctx, t, std::max<u64>(t->hint, 1));
    for (u32 c = 0; c < string_key_count && s.code == YTGPU_OK; ++c) {
        s = t->dicts[c].slots.allocate(ctx, 8);
        if (s.code == YTGPU_OK) {
            const cudaError_t e = cudaMemsetAsync(t->dicts[c].slots.p, 0xff, 64, ctx->stream);
            if (e != cudaSuccess) s = cuda_status(e, "cudaMemsetAsync");
        }
    }
    if (s.code == YTGPU_OK) {
        const cudaError_t e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) s = cuda_status(e, "cudaStreamSynchronize");
    }
    if (s.code != YTGPU_OK) {
        delete t;
        return s;
    }
    *out = t;
    return Status{};
}

// The heap of string-valued aggregate H compacted into a buffer of its live bytes, in group-id order.
Status compact_heap(Context* ctx, OwnedHeap* H, u64 groups) {
    const u64 values = groups * H->count;
    DevBuf<u64> at, sums, total;
    DevBuf<u8> to;
    YTGPU_TRY(at.allocate(ctx, values + 1));
    YTGPU_TRY(sums.allocate(ctx, scan_block_count(values + 1)));
    YTGPU_TRY(total.allocate(ctx, 1));
    YTGPU_TRY(to.allocate(ctx, std::max<u64>(H->live, 16)));
    KernelTimer timer(ctx, KC_GROUPBY, 3);
    gt_owned_lengths_kernel<<<blocks_for(values + 1, 256, 8), 256, 0, ctx->stream>>>(values, H->count, H->view(), at.p);
    exclusive_scan_u64(ctx->stream, at.p, values + 1, sums.p, total.p);
    gt_owned_compact_kernel<<<blocks_for(values, 256, 8), 256, 0, ctx->stream>>>(values, H->count, H->view(), at.p, to.p);
    YTGPU_CUDA_TRY(cudaGetLastError());
    H->heap = static_cast<DevBuf<u8>&&>(to);
    H->used = H->live;
    return Status{};
}

Status update_impl(Context* ctx, GroupByTable* t, const ytgpu_column_view* key_columns, u32 key_count, const ytgpu_string_column* strings,
                   u32 string_count, const ytgpu_column_view* value_columns, u32 value_count, const ytgpu_string_column* string_values,
                   u32 string_value_count, const ytgpu_predicate* pred, int32_t pred_column) {
    if (!t || (key_count && !key_columns) || (string_count && !strings) || (value_count && !value_columns) ||
        (string_value_count && !string_values))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    if (t->ctx != ctx) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "the table was created on another context");
    if (key_count != t->numeric) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "%u key columns, the table has %u", key_count, t->numeric);
    if (string_count != t->strings)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "%u string key columns, the table has %u", string_count, t->strings);
    if (value_count != t->value_count)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "%u value columns, the table has %u", value_count, t->value_count);
    if (string_value_count != t->string_value_count)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "%u string value columns, the table has %u", string_value_count, t->string_value_count);
    // every length from the views, before any access
    u64 n = 0;
    bool have = false;
    auto same_length = [&](u64 rows, const char* what, u32 i) -> Status {
        if (!have) {
            n = rows;
            have = true;
        }
        if (rows != n) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "%s %u differs in length from the other columns", what, i);
        return Status{};
    };
    for (u32 k = 0; k < key_count; ++k) {
        const ytgpu_column_view& c = key_columns[k];
        if (c.value_count < 0 || c.start_index < 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key %u: negative column range", k);
        if (c.value_type != t->key_types[k])
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key %u: type 0x%x differs from the table's 0x%x", k, c.value_type, t->key_types[k]);
        YTGPU_TRY(same_length((u64)c.value_count, "key column", k));
    }
    for (u32 s = 0; s < string_count; ++s) {
        const ytgpu_string_column& c = strings[s];
        if (c.mem != YTGPU_MEM_DEVICE && c.mem != YTGPU_MEM_HOST)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string key %u: mem must be YTGPU_MEM_DEVICE or YTGPU_MEM_HOST", s);
        if ((c.row_count && (!c.starts || !c.lengths)) || (c.heap_bytes && !c.heap))
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string key %u: null heap, starts or lengths", s);
        YTGPU_TRY(same_length(c.row_count, "string key", s));
    }
    for (u32 v = 0; v < value_count; ++v) {
        const ytgpu_column_view& c = value_columns[v];
        if (c.value_count < 0 || c.start_index < 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "value %u: negative column range", v);
        if (c.value_type != t->value_types[v])
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "value %u: type 0x%x differs from the table's 0x%x", v, c.value_type, t->value_types[v]);
        YTGPU_TRY(same_length((u64)c.value_count, "value column", v));
    }
    for (u32 s = 0; s < string_value_count; ++s) {
        const ytgpu_string_column& c = string_values[s];
        if (c.mem != YTGPU_MEM_DEVICE && c.mem != YTGPU_MEM_HOST)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string value %u: mem must be YTGPU_MEM_DEVICE or YTGPU_MEM_HOST", s);
        if ((c.row_count && (!c.starts || !c.lengths)) || (c.heap_bytes && !c.heap))
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string value %u: null heap, starts or lengths", s);
        YTGPU_TRY(same_length(c.row_count, "string value", s));
    }
    if (n > kMaxUpdateRows) return make_status(YTGPU_ERR_UNSUPPORTED, "at most 2^30 rows per update (slots and rows are 32-bit)");
    const int op = pred ? pred->op : YTGPU_CMP_NONE;
    if (op != YTGPU_CMP_NONE && (pred_column < 0 || (u32)pred_column >= value_count))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "predicate column %d out of range", (int)pred_column);
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    if (n == 0) return Status{};

    std::vector<StagedColumn> sk(key_count), sv(value_count);
    KeyColumns K{};
    K.count = key_count + string_count;
    bool direct = true;
    for (u32 k = 0; k < key_count; ++k) {
        YTGPU_TRY(stage_column(ctx, &key_columns[k], &sk[k]));
        K.col[k] = sk[k].dev;
        direct = direct && is_direct64(sk[k].dev) && sk[k].dev.base == 0 && !sk[k].dev.zigzag;
    }
    for (u32 v = 0; v < value_count; ++v) YTGPU_TRY(stage_column(ctx, &value_columns[v], &sv[v]));
    const u32 A = t->aggregate_count;
    std::vector<StagedStrings> ss(string_value_count);
    std::vector<bool> read(string_value_count, false);  // the string values some aggregate reads
    for (u32 a = 0; a < A; ++a) {
        const ytgpu_aggregate& G = t->aggregates[a];
        if (t->is_string(G.column)) read[G.column - value_count] = true;
        if ((G.op == YTGPU_AGG_ARGMIN || G.op == YTGPU_AGG_ARGMAX) && t->is_string(G.by_column)) read[G.by_column - value_count] = true;
    }
    bool check = string_count != 0;
    for (u32 s = 0; s < string_value_count; ++s) {
        if (!read[s]) continue;
        YTGPU_TRY(stage_strings(ctx, string_values[s], &ss[s]));
        KernelTimer timer(ctx, KC_GROUPBY);
        gt_check_strings_kernel<<<blocks_for(n, 256, 8), 256, 0, ctx->stream>>>(ss[s].dev, n, ctx->dev_err);
        YTGPU_CUDA_TRY(cudaGetLastError());
        check = true;
    }

    // step 1: the lookups and every bounds check first, read before the table changes
    DevBuf<u64> ids[kMaxGroupKeys];
    DevBuf<u32> null_bits[kMaxGroupKeys];
    for (u32 c = 0; c < string_count; ++c) {
        YTGPU_TRY(ids[c].allocate(ctx, n));
        if (strings[c].null_bytemap) YTGPU_TRY(null_bits[c].allocate(ctx, (n + 31) / 32));
        YTGPU_TRY(string_dict_lookup(ctx, t->dicts[c], strings[c], n, ids[c].p, null_bits[c].p));
    }
    if (check) YTGPU_TRY(check_device_errors(ctx));  // synchronises
    for (u32 c = 0; c < string_count; ++c) {
        YTGPU_TRY(string_dict_append(ctx, &t->dicts[c], &t->dict_count[c], &t->dict_bytes[c], strings[c], n, ids[c].p));
        K.col[key_count + c] = id_column(ids[c].p, null_bits[c].p, n);
        direct = direct && !strings[c].null_bytemap;
    }

    // step 2
    const ColumnDev pred_dev = op != YTGPU_CMP_NONE ? sv[pred_column].dev : ColumnDev{};
    KeyTable T;
    const u64 block_hint = std::min<u64>(std::max(t->groups, t->hint), n);
    YTGPU_TRY(assign_key_slots(ctx, KC_GROUPBY, K, direct, pred_dev, op, pred ? pred->constant : 0, n, block_hint, &T));
    const u64 bcap = T.cap;
    std::vector<DevBuf<unsigned long long>> bacc(A), bnn(A), brow(A);
    std::vector<AggState> bstate(A);
    std::vector<BlockStrings> bstr(A);
    auto column = [&](int32_t c) { return t->is_string(c) ? ColumnDev{} : sv[c].dev; };
    auto strings_of = [&](int32_t c) { return t->is_string(c) ? ss[c - value_count].dev : StringDev{}; };
    for (u32 a = 0; a < A; ++a) {
        const ytgpu_aggregate& G = t->aggregates[a];
        const bool arg = G.op == YTGPU_AGG_ARGMIN || G.op == YTGPU_AGG_ARGMAX;
        if (t->is_string(G.column) || (arg && t->is_string(G.by_column))) {
            // the one-shot's string step: the selected block row, or the non-NULL count
            AggState S{nullptr, nullptr, nullptr};
            if (G.op == YTGPU_AGG_COUNT) {
                YTGPU_TRY(bnn[a].allocate(ctx, bcap));
                YTGPU_CUDA_TRY(cudaMemsetAsync(bnn[a].p, 0, bcap * 8, ctx->stream));
                S.nn = bnn[a].p;
            } else {
                YTGPU_TRY(brow[a].allocate(ctx, bcap));
                YTGPU_CUDA_TRY(cudaMemsetAsync(brow[a].p, 0xff, bcap * 8, ctx->stream));
                S.row = brow[a].p;
            }
            bstate[a] = S;
            const StringDev cs = strings_of(G.column), bs = arg ? strings_of(G.by_column) : StringDev{};
            BlockStrings& B = bstr[a];
            const OwnedHeap& H = t->heaps[a];
            B.count = H.count;
            B.key = H.key;
            B.value = H.value;
            B.s[0] = cs.present ? cs : bs;
            B.s[1] = cs.present ? bs : StringDev{};
            KernelTimer timer(ctx, KC_GROUPBY);
            mg_accumulate_strings_kernel<<<(u32)((n + 255) / 256), 256, 0, ctx->stream>>>(G.op, column(G.column), cs,
                                                                                         arg ? column(G.by_column) : ColumnDev{}, bs, n,
                                                                                         T.slot_of_row.p, S, ctx->dev_err);
            YTGPU_CUDA_TRY(cudaGetLastError());
            continue;
        }
        YTGPU_TRY(accumulate_scalar(ctx, G.op, sv[G.column].dev, arg ? sv[G.by_column].dev : ColumnDev{}, n, bcap, T.slot_of_row.p, &bacc[a],
                                    &bnn[a], &brow[a], &bstate[a]));
    }
    const u64 max_block_groups = std::min<u64>(n, bcap);
    DevBuf<u64> bfirst;
    DevBuf<u32> bslot, counter;
    YTGPU_TRY(bfirst.allocate(ctx, max_block_groups));
    YTGPU_TRY(bslot.allocate(ctx, max_block_groups));
    YTGPU_TRY(counter.allocate(ctx, 1));
    YTGPU_CUDA_TRY(cudaMemsetAsync(counter.p, 0, 4, ctx->stream));
    {
        KernelTimer timer(ctx, KC_GROUPBY);
        mg_compact_kernel<<<blocks_for(bcap, 256, 8), 256, 0, ctx->stream>>>(T.rep.p, bcap, T.first.p, bfirst.p, bslot.p, counter.p);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    u32 gb32 = 0;
    YTGPU_CUDA_TRY(cudaMemcpyAsync(&gb32, counter.p, 4, cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    const u64 gb = gb32;
    if (gb == 0) {
        t->rows += n;
        return Status{};
    }
    // step 3: the lookup runs against the table as it is; only the misses size its growth
    // total: the count of new groups, then per string-valued aggregate the bytes its replacements append and free
    std::vector<u32> owning;
    for (u32 a = 0; a < A; ++a)
        if (t->heaps[a].count) owning.push_back(a);
    const u32 O = (u32)owning.size();
    DevBuf<u32> gid;
    DevBuf<u64> rank, sums, total;
    YTGPU_TRY(gid.allocate(ctx, gb));
    YTGPU_TRY(rank.allocate(ctx, gb + 1));
    YTGPU_TRY(sums.allocate(ctx, scan_block_count(gb + 1)));
    YTGPU_TRY(total.allocate(ctx, 1 + 2 * O));
    std::vector<DevBuf<u8>> take(O);
    std::vector<DevBuf<u64>> need(O);
    const u32 gblocks = blocks_for(gb, 256, 8);
    {
        KernelTimer timer(ctx, KC_GROUPBY, 5);
        gt_lookup_kernel<<<gblocks, 256, 0, ctx->stream>>>(K, bfirst.p, gb, t->owned(), t->slots.p, t->slots.n - 1, gid.p);
        gt_miss_flags_kernel<<<blocks_for(gb + 1, 256, 8), 256, 0, ctx->stream>>>(gid.p, gb, rank.p);
        exclusive_scan_u64(ctx->stream, rank.p, gb + 1, sums.p, total.p);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    if (O) YTGPU_CUDA_TRY(cudaMemsetAsync(total.p + 1, 0, 2 * O * 8, ctx->stream));
    for (u32 i = 0; i < O; ++i) {
        const u32 a = owning[i];
        const ytgpu_aggregate& G = t->aggregates[a];
        const bool arg = G.op == YTGPU_AGG_ARGMIN || G.op == YTGPU_AGG_ARGMAX;
        YTGPU_TRY(take[i].allocate(ctx, gb));
        YTGPU_TRY(need[i].allocate(ctx, gb + 1));
        KernelTimer timer(ctx, KC_GROUPBY, 4);
        gt_string_decide_kernel<<<blocks_for(gb + 1, 256, 8), 256, 0, ctx->stream>>>(
            G.op, arg ? column(G.by_column) : ColumnDev{}, bstr[a], gb, bslot.p, gid.p, brow[a].p, t->state(a), t->heaps[a].view(), take[i].p,
            need[i].p, reinterpret_cast<unsigned long long*>(total.p + 2 + 2 * i));
        exclusive_scan_u64(ctx->stream, need[i].p, gb + 1, sums.p, total.p + 1 + 2 * i);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    std::vector<u64> totals(1 + 2 * O);
    YTGPU_CUDA_TRY(cudaMemcpyAsync(totals.data(), total.p, totals.size() * 8, cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    const u64 added = totals[0];
    if (t->groups + added > kMaxGroups)
        return make_status(YTGPU_ERR_UNSUPPORTED, "the table holds fewer than 2^30 groups (%llu, and %llu new in this block)",
                           (unsigned long long)t->groups, (unsigned long long)added);
    YTGPU_TRY(grow_groups(ctx, t, t->groups + added));
    YTGPU_TRY(grow_slots(ctx, t, t->groups + added));
    const u64 mask = t->slots.n - 1;
    {
        KernelTimer timer(ctx, KC_GROUPBY, 2);
        gt_insert_kernel<<<gblocks, 256, 0, ctx->stream>>>(K, bfirst.p, gb, t->rows, t->groups, rank.p, t->owned(), t->counts.p, t->first.p,
                                                           t->slots.p, mask, gid.p);
        gt_count_kernel<<<gblocks, 256, 0, ctx->stream>>>(gb, bslot.p, gid.p, T.counts.p, t->counts.p);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    for (u32 a = 0; a < A; ++a) {
        const ytgpu_aggregate& G = t->aggregates[a];
        if (t->heaps[a].count) continue;
        KernelTimer timer(ctx, KC_GROUPBY);
        gt_merge_kernel<<<gblocks, 256, 0, ctx->stream>>>(G.op, column(G.column), gb, bslot.p, gid.p, t->rows, bstate[a], t->state(a));
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    for (u32 i = 0; i < O; ++i) {
        const u32 a = owning[i];
        const ytgpu_aggregate& G = t->aggregates[a];
        const bool arg = G.op == YTGPU_AGG_ARGMIN || G.op == YTGPU_AGG_ARGMAX;
        OwnedHeap& H = t->heaps[a];
        const u64 appended = totals[1 + 2 * i], freed = totals[2 + 2 * i];
        YTGPU_TRY(grow_buf(ctx, &H.heap, H.used, H.used + appended));
        {
            KernelTimer timer(ctx, KC_GROUPBY);
            gt_string_take_kernel<<<gblocks, 256, 0, ctx->stream>>>(G.op, column(G.column), arg ? column(G.by_column) : ColumnDev{}, bstr[a], gb,
                                                                   bslot.p, gid.p, brow[a].p, take[i].p, need[i].p, H.used, t->rows,
                                                                   t->state(a), H.view());
            YTGPU_CUDA_TRY(cudaGetLastError());
        }
        H.used += appended;
        H.live = H.live + appended - freed;
        if (H.used > kReclaimMinBytes && H.used > kReclaimFactor * H.live) YTGPU_TRY(compact_heap(ctx, &H, t->groups + added));
    }
    // the caller may free or reuse the block's buffers once this returns
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    t->groups += added;
    t->rows += n;
    return Status{};
}

Status result_impl(Context* ctx, GroupByTable* t, ytgpu_groupby_multi_result* out, ytgpu_groupby_string_keys* string_out, u32 string_count,
                   ytgpu_groupby_string_keys* value_string_out, u32 value_string_count, int out_mem) {
    if (!t || !out) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    if (t->ctx != ctx) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "the table was created on another context");
    if (string_count != t->strings)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "%u string key outputs, the table has %u string keys", string_count, t->strings);
    if (string_count && !string_out) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null string key outputs");
    // the string outputs: the string keys, then the string-valued aggregates' values in aggregate order
    std::vector<GroupStrings> src;
    std::vector<ytgpu_groupby_string_keys*> dst;
    for (u32 s = 0; s < string_count; ++s) {
        const u32 k = t->numeric + s;
        src.push_back(GroupStrings{t->keys[k].p, t->nulls.p, k, nullptr, t->dicts[s].heap.p, t->dicts[s].starts.p, t->dicts[s].lengths.p});
        dst.push_back(&string_out[s]);
    }
    for (u32 a = 0; a < t->aggregate_count; ++a) {
        OwnedHeap& H = t->heaps[a];
        if (!H.value) continue;
        src.push_back(GroupStrings{nullptr, nullptr, 0, t->row[a].p, H.heap.p, H.start[0].p, H.len[0].p});
        dst.push_back(value_string_out ? &value_string_out[src.size() - 1 - string_count] : nullptr);
    }
    const u32 value_strings = (u32)src.size() - string_count;
    if (value_string_count != value_strings)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "%u string value outputs, the table has %u string-valued aggregates", value_string_count,
                           value_strings);
    if (value_string_count && !value_string_out) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null string value outputs");
    if (out_mem != YTGPU_MEM_DEVICE && out_mem != YTGPU_MEM_HOST)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "out_mem must be YTGPU_MEM_DEVICE or YTGPU_MEM_HOST");
    if ((t->numeric && (!out->keys || !out->key_null)) || (t->aggregate_count && (!out->values || !out->value_null)))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null output array");
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    const u64 g = t->groups;
    const u32 outputs = (u32)src.size();
    out->group_count = g;
    for (u32 s = 0; s < outputs; ++s) dst[s]->heap_bytes = 0;
    if (g == 0) return Status{};

    SortScratch scratch;
    PermRef perm;
    const u64* cptr[1] = {reinterpret_cast<const u64*>(t->first.p)};
    YTGPU_TRY(radix_sort_chunks(ctx, cptr, 1, g, &scratch, &perm));
    DevBuf<u32> gid_sorted;
    YTGPU_TRY(gid_sorted.allocate(ctx, g));
    const u32 threads = 256;
    const u32 gblocks = (u32)((g + threads - 1) / threads);
    gt_emit_keys_kernel<<<gblocks, threads, 0, ctx->stream>>>(t->owned(), 0, perm.plan, perm.idx[0], perm.idx[1], g, t->counts.p, t->first.p,
                                                              NumericKeyOutputs{}, nullptr, nullptr, gid_sorted.p);
    ctx->count_launch();
    // string outputs: lengths and nulls (scratch until the capacities are known), their scan, and the byte totals
    std::vector<DevBuf<u64>> at(outputs);
    std::vector<DevBuf<u32>> lens(outputs);
    std::vector<DevBuf<u8>> snull(outputs);
    DevBuf<u64> totals, sums;
    if (outputs) {
        YTGPU_TRY(totals.allocate(ctx, outputs));
        YTGPU_TRY(sums.allocate(ctx, scan_block_count(g + 1)));
    }
    for (u32 s = 0; s < outputs; ++s) {
        YTGPU_TRY(at[s].allocate(ctx, g + 1));
        YTGPU_TRY(lens[s].allocate(ctx, g));
        YTGPU_TRY(snull[s].allocate(ctx, g));
        KernelTimer timer(ctx, KC_GROUPBY, 4);
        gt_string_lengths_kernel<<<blocks_for(g + 1, 256, 8), 256, 0, ctx->stream>>>(g, gid_sorted.p, src[s], at[s].p, lens[s].p, snull[s].p);
        exclusive_scan_u64(ctx->stream, at[s].p, g + 1, sums.p, totals.p + s);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    std::vector<u64> heap_bytes(outputs);
    if (outputs) YTGPU_CUDA_TRY(cudaMemcpyAsync(heap_bytes.data(), totals.p, outputs * 8, cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    for (u32 s = 0; s < outputs; ++s) dst[s]->heap_bytes = heap_bytes[s];
    if (g > out->capacity)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "result has %llu groups, capacity is %llu", (unsigned long long)g,
                           (unsigned long long)out->capacity);
    for (u32 s = 0; s < outputs; ++s) {
        const ytgpu_groupby_string_keys& S = *dst[s];
        const char* what = s < string_count ? "string key" : "string value";
        const u32 i = s < string_count ? s : s - string_count;
        if (heap_bytes[s] > S.heap_capacity)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "%s %u needs %llu heap bytes, heap_capacity is %llu", what, i,
                               (unsigned long long)heap_bytes[s], (unsigned long long)S.heap_capacity);
        if (!S.starts || !S.lengths || !S.null_bytemap || (heap_bytes[s] && !S.heap))
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "%s %u: null output", what, i);
    }
    // every check passed: nothing was written to the outputs before this point
    std::vector<OutBuf<u64>> tk(t->numeric);
    std::vector<OutBuf<u8>> tkn(t->numeric);
    OutBuf<u64> tcounts, tfirst;
    NumericKeyOutputs O{};
    for (u32 k = 0; k < t->numeric; ++k) {
        if (!out->keys[k] || !out->key_null[k]) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null key output %u", k);
        YTGPU_TRY(tk[k].prepare(ctx, out->keys[k], g, out_mem));
        YTGPU_TRY(tkn[k].prepare(ctx, out->key_null[k], g, out_mem));
        O.keys[k] = tk[k].p;
        O.key_null[k] = tkn[k].p;
    }
    YTGPU_TRY(tcounts.prepare(ctx, out->counts, g, out_mem));
    YTGPU_TRY(tfirst.prepare(ctx, out->first_rows, g, out_mem));
    gt_emit_keys_kernel<<<gblocks, threads, 0, ctx->stream>>>(t->owned(), t->numeric, perm.plan, perm.idx[0], perm.idx[1], g, t->counts.p,
                                                              t->first.p, O, tcounts.p, tfirst.p, gid_sorted.p);
    ctx->count_launch();
    std::vector<OutBuf<u64>> tv(t->aggregate_count);
    std::vector<OutBuf<u8>> tvn(t->aggregate_count);
    for (u32 a = 0; a < t->aggregate_count; ++a) {
        if (!out->values[a] || !out->value_null[a]) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null aggregate output %u", a);
        YTGPU_TRY(tv[a].prepare(ctx, out->values[a], g, out_mem));
        YTGPU_TRY(tvn[a].prepare(ctx, out->value_null[a], g, out_mem));
        const ytgpu_aggregate& A = t->aggregates[a];
        const AggState S{t->acc[a].p, t->nn[a].p, t->row[a].p};
        if (t->heaps[a].value) {  // a string-valued result: the global row that holds it, as the one-shot gives it
            mg_finalize_kernel<<<gblocks, threads, 0, ctx->stream>>>(A.op, ColumnDev{}, 0, g, gid_sorted.p, S, tv[a].p, tvn[a].p, true);
        } else if (selects_row(A.op)) {
            gt_finalize_selected_kernel<<<gblocks, threads, 0, ctx->stream>>>(g, gid_sorted.p, t->state(a), tv[a].p, tvn[a].p);
        } else {
            ColumnDev col{};
            if (!t->is_string(A.column)) col.value_type = t->value_types[A.column];
            mg_finalize_kernel<<<gblocks, threads, 0, ctx->stream>>>(A.op, col, 0, g, gid_sorted.p, S, tv[a].p, tvn[a].p, false);
        }
        ctx->count_launch();
        YTGPU_TRY(tv[a].download(ctx, g));
        YTGPU_TRY(tvn[a].download(ctx, g));
    }
    std::vector<OutBuf<u64>> ost(outputs);
    std::vector<OutBuf<u8>> oheap(outputs);
    for (u32 s = 0; s < outputs; ++s) {
        const ytgpu_groupby_string_keys& S = *dst[s];
        YTGPU_TRY(ost[s].prepare(ctx, S.starts, g, out_mem));
        YTGPU_TRY(oheap[s].prepare(ctx, S.heap, heap_bytes[s], out_mem));
        KernelTimer timer(ctx, KC_GROUPBY);
        gt_string_copy_kernel<<<blocks_for(g, 256, 8), 256, 0, ctx->stream>>>(g, gid_sorted.p, src[s], at[s].p, ost[s].p, oheap[s].p);
        YTGPU_CUDA_TRY(cudaGetLastError());
        YTGPU_TRY(ost[s].download(ctx, g));
        YTGPU_TRY(oheap[s].download(ctx, heap_bytes[s]));
        YTGPU_TRY(copy_out(ctx, S.lengths, lens[s].p, g * 4, out_mem));
        YTGPU_TRY(copy_out(ctx, S.null_bytemap, snull[s].p, g, out_mem));
    }
    YTGPU_CUDA_TRY(cudaGetLastError());
    for (u32 k = 0; k < t->numeric; ++k) {
        YTGPU_TRY(tk[k].download(ctx, g));
        YTGPU_TRY(tkn[k].download(ctx, g));
    }
    YTGPU_TRY(tcounts.download(ctx, g));
    YTGPU_TRY(tfirst.download(ctx, g));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return Status{};
}

}  // namespace

extern "C" {

int ytgpu_groupby_table_create_strings(ytgpu_context* h, const uint8_t* key_types, uint32_t key_count, uint32_t string_key_count,
                                       const uint8_t* value_types, uint32_t value_count, uint32_t string_value_count,
                                       const ytgpu_aggregate* aggregates, uint32_t aggregate_count, uint64_t group_count_hint,
                                       ytgpu_groupby_table** out, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    GroupByTable* t = nullptr;
    const int code = fill_error(err, create_impl(as_context(h), key_types, key_count, string_key_count, value_types, value_count,
                                                 string_value_count, aggregates, aggregate_count, group_count_hint, &t));
    if (out) *out = reinterpret_cast<ytgpu_groupby_table*>(t);
    return code;
}

int ytgpu_groupby_table_create(ytgpu_context* h, const uint8_t* key_types, uint32_t key_count, uint32_t string_key_count,
                               const uint8_t* value_types, uint32_t value_count, const ytgpu_aggregate* aggregates,
                               uint32_t aggregate_count, uint64_t group_count_hint, ytgpu_groupby_table** out, ytgpu_error* err) {
    return ytgpu_groupby_table_create_strings(h, key_types, key_count, string_key_count, value_types, value_count, 0, aggregates,
                                              aggregate_count, group_count_hint, out, err);
}

int ytgpu_groupby_table_update_strings(ytgpu_context* h, ytgpu_groupby_table* table, const ytgpu_column_view* key_columns,
                                       uint32_t key_count, const ytgpu_string_column* string_keys, uint32_t string_key_count,
                                       const ytgpu_column_view* value_columns, uint32_t value_count,
                                       const ytgpu_string_column* string_values, uint32_t string_value_count,
                                       const ytgpu_predicate* predicate, int32_t predicate_column, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, update_impl(as_context(h), reinterpret_cast<GroupByTable*>(table), key_columns, key_count, string_keys,
                                       string_key_count, value_columns, value_count, string_values, string_value_count, predicate,
                                       predicate_column));
}

int ytgpu_groupby_table_update(ytgpu_context* h, ytgpu_groupby_table* table, const ytgpu_column_view* key_columns, uint32_t key_count,
                               const ytgpu_string_column* string_keys, uint32_t string_key_count, const ytgpu_column_view* value_columns,
                               uint32_t value_count, const ytgpu_predicate* predicate, int32_t predicate_column, ytgpu_error* err) {
    return ytgpu_groupby_table_update_strings(h, table, key_columns, key_count, string_keys, string_key_count, value_columns, value_count,
                                              nullptr, 0, predicate, predicate_column, err);
}

int ytgpu_groupby_table_result_strings(ytgpu_context* h, const ytgpu_groupby_table* table, ytgpu_groupby_multi_result* out,
                                       ytgpu_groupby_string_keys* string_out, uint32_t string_key_count,
                                       ytgpu_groupby_string_keys* value_string_out, uint32_t string_aggregate_count, int out_mem,
                                       ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, result_impl(as_context(h), reinterpret_cast<GroupByTable*>(const_cast<ytgpu_groupby_table*>(table)), out,
                                       string_out, string_key_count, value_string_out, string_aggregate_count, out_mem));
}

int ytgpu_groupby_table_result(ytgpu_context* h, const ytgpu_groupby_table* table, ytgpu_groupby_multi_result* out,
                               ytgpu_groupby_string_keys* string_out, uint32_t string_key_count, int out_mem, ytgpu_error* err) {
    return ytgpu_groupby_table_result_strings(h, table, out, string_out, string_key_count, nullptr, 0, out_mem, err);
}

int ytgpu_groupby_table_destroy(ytgpu_groupby_table* table, ytgpu_error* err) {
    if (!table) return fill_error(err, Status{});
    GroupByTable* t = reinterpret_cast<GroupByTable*>(table);
    Context* ctx = t->ctx;
    std::unique_lock<std::mutex> lock(ctx->mu);
    const cudaError_t e = cudaSetDevice(ctx->device);
    delete t;  // stream-ordered frees on the context's stream
    return fill_error(err, e == cudaSuccess ? Status{} : cuda_status(e, "cudaSetDevice"));
}

}  // extern "C"
