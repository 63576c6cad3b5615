// groupby_multi.cu — GROUP BY over several key columns with several aggregates (the general form of the hashed path).
//
// Replaces, for tuple keys and aggregate lists, the same reference code as ytgpu_scan_filter_groupby:
//   YT QL   GroupOpHelper / InsertGroupRow (library/query/engine/cg_routines/registry.cpp:1571-1655,1783-1920) with the
//           aggregates of builtin_function_types.cpp:201-254 — sum / min / max (engine/udf/sum.c, min.c, max.c), avg and
//           argmin / argmax (builtin_function_profiler.cpp:1300-1600), first (registry.cpp:3633-3693), count;
//   CHYT    DB::Aggregator with a keys128 / serialized key and a list of aggregate functions;
//   YQL     BlockCombineHashed over tuple keys (mkql_block_agg.cpp:1234-1400).
// Three steps instead of one fused kernel (the single-key SUM/COUNT fast path stays in columnar.cu):
//   1. assign: every row that passes the predicate finds or claims the slot of its key tuple in an open-addressing
//      table.  A slot stores the index of the row that claimed it; tuples are compared by decoding that row's key
//      columns again (the inputs are immutable), so any number of key columns needs no lock and no key storage.
//      COUNT(*) and the group's first row are updated here; the slot of every row is kept (4 bytes per row).
//   2. accumulate: one pass per aggregate over its value column, atomics on per-slot state.  min / max move one way, so a
//      plain read that already bounds the value skips the atomic; argmin / argmax / first select a ROW (atomicMin of the
//      row index among the rows that attain the bound), the value is gathered at the end — exactly the reference's
//      "the first row wins a tie" (strict comparison in UpdateAggregateValue).  An aggregate over a string column (or
//      argmin / argmax by one) takes mg_accumulate_strings_kernel instead: it selects the row lock-free with a CAS on
//      the slot's row, comparing strings by the width-free key words of keys.cuh.
//   3. emit: occupied slots are compacted and ordered by first row == QL's first-seen order (InsertGroupRow appends new
//      groups), keys are decoded from the group's first row, states are finalised (avg = sum / count as double).
#include <vector>

#include "columnar.cuh"
#include "context.cuh"
#include "keys.cuh"
#include "radix_sort.cuh"

using namespace ytgpu;

namespace {

constexpr int kMaxGroupKeys = 8;
constexpr int kMaxAggregates = 32;
constexpr u32 kNoSlot = 0xffffffffu;

struct KeyColumns {
    ColumnDev col[kMaxGroupKeys];
    u32 count;
};

struct KeyTuple {
    u64 w[kMaxGroupKeys];
    u32 nulls;
};

// DIRECT: every key column is a plain 64-bit vector (no NULLs, dictionary, RLE, base or zig-zag): one load per column
// instead of the general decode (the ncu capture of the general form: 836 warp instructions per 32 rows, 14.9 active
// threads per instruction — the decode inlined into every probe step of a divergent loop).
// NK: number of key columns when known at compile time (1, 2), else 0 = K.count of them (the loops then carry a
// run-time bound through all kMaxGroupKeys unrolled steps — the second ncu capture: still 1171 warp instructions per 32 rows).
template <bool DIRECT = false, int NK = 0>
__device__ __forceinline__ KeyTuple load_tuple(const KeyColumns& K, u64 row) {
    KeyTuple t;
    t.nulls = 0;
#pragma unroll
    for (u32 k = 0; k < (u32)(NK ? NK : kMaxGroupKeys); ++k) {
        t.w[k] = 0;
        if (NK || k < K.count) {
            if (DIRECT) {
                t.w[k] = reinterpret_cast<const u64*>(K.col[k].values)[(u64)K.col[k].start + row];
            } else {
                bool nul;
                const u64 v = decode_at(K.col[k], (i64)row, &nul);
                t.w[k] = nul ? 0 : v;
                if (nul) t.nulls |= 1u << k;
            }
        }
    }
    return t;
}

template <int NK = 0>
__device__ __forceinline__ bool same_tuple(const KeyColumns& K, const KeyTuple& a, const KeyTuple& b) {
    bool same = a.nulls == b.nulls;
#pragma unroll
    for (u32 k = 0; k < (u32)(NK ? NK : kMaxGroupKeys); ++k)
        if (NK || k < K.count) same = same && a.w[k] == b.w[k];
    return same;
}

template <int NK = 0>
__device__ __forceinline__ u64 hash_tuple(const KeyColumns& K, const KeyTuple& t) {
    u64 h = 0x9E3779B97F4A7C15ull ^ t.nulls;
#pragma unroll
    for (u32 k = 0; k < (u32)(NK ? NK : kMaxGroupKeys); ++k)
        if (NK || k < K.count) {
            h = (h ^ t.w[k]) * 0xff51afd7ed558ccdull;
            h ^= h >> 33;
        }
    h *= 0xc4ceb9fe1a85ec53ull;
    return h ^ (h >> 29);
}

// Small tables (<= kSmemSlots slots, i.e. up to ~1000 expected groups): COUNT(*), the non-null counts and the sums are
// accumulated in shared memory per CTA and flushed once — 10^8 rows otherwise mean 10^8 global atomics on a thousand
// addresses.  The kernels run grid-stride with a fixed grid so that a CTA flushes once.
constexpr int kSmemSlots = 4096;

// Step 1.  rep[slot] = row that claimed the slot (kNoSlot = empty).
template <bool DIRECT, int NK>
__global__ void __launch_bounds__(256) mg_assign_kernel(const KeyColumns K, const ColumnDev pred_col, int op, u64 constant, u64 n,
                                                        u32* rep, u64 mask, u32* slot_of_row, unsigned long long* counts,
                                                        unsigned long long* first, u32* err_word) {
    __shared__ u32 s_cnt[kSmemSlots];
    __shared__ u32 s_first[kSmemSlots];
    const bool cached = mask < (u64)kSmemSlots;
    if (cached) {
        for (u32 k = threadIdx.x; k <= (u32)mask; k += blockDim.x) {
            s_cnt[k] = 0;
            s_first[k] = kNoSlot;
        }
        __syncthreads();
    }
    // Two rows per thread and trip: the probe is a chain of dependent loads (key -> table slot -> the claiming row's key);
    // with both rows' loads issued before either is used the chain's latency is paid once per pair (the third ncu capture:
    // 170 instructions per 32 rows but 26 cycles of long-scoreboard stall per issue).
    constexpr int R = NK ? 2 : 1;  // 3+ key columns: four 8-word tuples in flight would cost the occupancy
    const u64 stride = (u64)gridDim.x * blockDim.x;
    const u64 trips = (n + stride * R - 1) / (stride * R);  // the same for every thread: the warp collectives see whole warps
    u64 base = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    KeyTuple ahead[R];  // the key tuples of the NEXT trip: their DRAM latency overlaps this trip's probes
#pragma unroll
    for (int j = 0; j < R; ++j)
        if (base + (u64)j * stride < n) ahead[j] = load_tuple<DIRECT, NK>(K, base + (u64)j * stride);
    for (u64 t = 0; t < trips; ++t, base += stride * R) {
        u64 row[R], b[R];
        u32 r[R], slot[R];
        bool valid[R];
        KeyTuple mine[R], cand[R];
#pragma unroll
        for (int j = 0; j < R; ++j) {
            mine[j] = ahead[j];
            const u64 nxt = base + stride * R + (u64)j * stride;
            if (nxt < n) ahead[j] = load_tuple<DIRECT, NK>(K, nxt);
        }
#pragma unroll
        for (int j = 0; j < R; ++j) {
            row[j] = base + (u64)j * stride;
            valid[j] = row[j] < n;
            slot[j] = kNoSlot;
            if (valid[j] && op != YTGPU_CMP_NONE) {
                bool nul;
                const u64 v = decode_at(pred_col, (i64)row[j], &nul);
                valid[j] = !nul && passes(op, pred_col.value_type, v, constant);
            }
        }
#pragma unroll
        for (int j = 0; j < R; ++j) {
            b[j] = valid[j] ? hash_tuple<NK>(K, mine[j]) & mask : 0;
            r[j] = valid[j] ? rep[b[j]] : kNoSlot;
        }
#pragma unroll
        for (int j = 0; j < R; ++j)
            if (valid[j] && r[j] != kNoSlot) cand[j] = load_tuple<DIRECT, NK>(K, r[j]);
#pragma unroll
        for (int j = 0; j < R; ++j) {
            if (!valid[j]) continue;
            u32 rr = r[j];
            bool have = rr != kNoSlot;  // cand[j] holds the key of row rr
            u64 bb = b[j];
            for (u64 probes = 0; probes <= mask; ++probes) {
                if (rr == kNoSlot) {
                    const u32 old = atomicCAS(&rep[bb], kNoSlot, (u32)row[j]);
                    rr = old == kNoSlot ? (u32)row[j] : old;
                    have = false;
                }
                if (rr == (u32)row[j] || same_tuple<NK>(K, mine[j], have ? cand[j] : load_tuple<DIRECT, NK>(K, rr))) {
                    slot[j] = (u32)bb;
                    break;
                }
                bb = (bb + 1) & mask;
                rr = rep[bb];
                have = false;
            }
        }
        __syncwarp();  // the lanes leave the probe loops one by one: everything below runs once per warp, not once per exit
#pragma unroll
        for (int j = 0; j < R; ++j) {
            const u64 i = row[j];
            if (valid[j] && slot[j] == kNoSlot) atomicOr(err_word, (u32)DE_TABLE_FULL);
            if (i < n) slot_of_row[i] = slot[j];
            if (cached) {
                if (slot[j] != kNoSlot) {
                    atomicAdd(&s_cnt[slot[j]], 1u);
                    if ((u32)i < s_first[slot[j]]) atomicMin(&s_first[slot[j]], (u32)i);  // n <= 2^30: row indices fit 32 bits
                }
                continue;
            }
            // COUNT(*) and the first row: one update per warp when its 32 rows share a slot (sorted / clustered keys)
            const u32 slot0 = __shfl_sync(0xffffffffu, slot[j], 0);
            if (__all_sync(0xffffffffu, slot[j] == slot0)) {
                if ((threadIdx.x & 31) == 0 && slot[j] != kNoSlot) {
                    atomicAdd(&counts[slot[j]], 32ull);
                    atomicMin(&first[slot[j]], (unsigned long long)i);
                }
            } else if (slot[j] != kNoSlot) {
                atomicAdd(&counts[slot[j]], 1ull);
                if (i < __ldcg(&first[slot[j]])) atomicMin(&first[slot[j]], (unsigned long long)i);
            }
        }
    }
    if (cached) {
        __syncthreads();
        for (u32 k = threadIdx.x; k <= (u32)mask; k += blockDim.x)
            if (s_cnt[k]) {
                atomicAdd(&counts[k], (unsigned long long)s_cnt[k]);
                atomicMin(&first[k], (unsigned long long)s_first[k]);
            }
    }
}

struct AggState {
    unsigned long long* acc;  // sum bits / encoded min / encoded max / encoded bound of argmin-argmax
    unsigned long long* nn;   // non-null values folded in (sum, avg, count); "any" flag for the others
    unsigned long long* row;  // selected row (argmin / argmax / first)
};

// The order of an argmin / argmax `by` value: its MIN / MAX word with -0.0 taken as +0.0, so the two zeros tie and the
// first row wins, as QL's strict `new.by < state.by` has it.
__device__ __forceinline__ u64 by_encode(u8 vtype, u64 bits) {
    return minmax_encode(vtype, vtype == YTGPU_TYPE_DOUBLE && bits == 0x8000000000000000ull ? 0 : bits);
}

// Step 2.  phase 1 is the row selection of argmin / argmax (the bound is final after phase 0).
__global__ void __launch_bounds__(512) mg_accumulate_kernel(int op, int phase, const ColumnDev col, const ColumnDev by, u64 n, u32 slots,
                                                            const u32* __restrict__ slot_of_row, AggState S) {
    __shared__ u64 s_acc[kSmemSlots];
    __shared__ u32 s_nn[kSmemSlots];
    const bool additive = op == YTGPU_AGG_SUM || op == YTGPU_AGG_AVG || op == YTGPU_AGG_COUNT;
    const bool extremum = op == YTGPU_AGG_MIN || op == YTGPU_AGG_MAX;
    const bool cached = (additive || extremum) && slots <= (u32)kSmemSlots;
    if (cached) {
        for (u32 k = threadIdx.x; k < slots; k += blockDim.x) {
            s_acc[k] = op == YTGPU_AGG_MIN ? ~0ull : 0ull;
            s_nn[k] = 0;
        }
        __syncthreads();
    }
    const u8 vtype = col.value_type;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    const u64 trips = (n + stride - 1) / stride;
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    for (u64 t = 0; t < trips; ++t, i += stride) {
        const u32 slot = i < n ? slot_of_row[i] : kNoSlot;
        const bool live = slot != kNoSlot;
        bool nul = true;
        u64 v = 0;
        if (live) v = decode_at(col, (i64)i, &nul);
        switch (op) {
            case YTGPU_AGG_SUM:
            case YTGPU_AGG_AVG:
            case YTGPU_AGG_COUNT: {
                const bool add = live && !nul;
                if (cached) {
                    if (add) {
                        atomicAdd(&s_nn[slot], 1u);
                        if (op != YTGPU_AGG_COUNT) {
                            if (vtype == YTGPU_TYPE_DOUBLE) {
                                atomicAdd(reinterpret_cast<double*>(&s_acc[slot]), __longlong_as_double((long long)v));
                            } else {  // two native 32-bit adds with the carry of the low word: exact mod 2^64
                                u32* w = reinterpret_cast<u32*>(&s_acc[slot]);
                                const u32 lo = (u32)v;
                                const u32 old = atomicAdd(w, lo);
                                atomicAdd(w + 1, (u32)(v >> 32) + (u32)(old + lo < old));
                            }
                        }
                    }
                    break;
                }
                const u32 slot0 = __shfl_sync(0xffffffffu, slot, 0);
                if (__all_sync(0xffffffffu, slot == slot0)) {  // whole warp in one group: reduce first
                    const u32 cnt = __popc(__ballot_sync(0xffffffffu, add));
                    u64 x = add ? v : 0;
                    if (op != YTGPU_AGG_COUNT) {
#pragma unroll
                        for (int d = 16; d > 0; d >>= 1) {
                            const u64 o = __shfl_xor_sync(0xffffffffu, x, d);
                            if (vtype == YTGPU_TYPE_DOUBLE)
                                x = (u64)__double_as_longlong(__longlong_as_double((long long)x) + __longlong_as_double((long long)o));
                            else x += o;
                        }
                    }
                    if ((threadIdx.x & 31) == 0 && slot != kNoSlot && cnt) {
                        atomicAdd(&S.nn[slot], (unsigned long long)cnt);
                        if (op != YTGPU_AGG_COUNT) {
                            if (vtype == YTGPU_TYPE_DOUBLE) atomicAdd(reinterpret_cast<double*>(&S.acc[slot]), __longlong_as_double((long long)x));
                            else atomicAdd(&S.acc[slot], (unsigned long long)x);
                        }
                    }
                } else if (add) {
                    atomicAdd(&S.nn[slot], 1ull);
                    if (op != YTGPU_AGG_COUNT) {
                        if (vtype == YTGPU_TYPE_DOUBLE) atomicAdd(reinterpret_cast<double*>(&S.acc[slot]), __longlong_as_double((long long)v));
                        else atomicAdd(&S.acc[slot], (unsigned long long)v);
                    }
                }
                break;
            }
            case YTGPU_AGG_MIN:
            case YTGPU_AGG_MAX:
                if (cached) {  // the bound only moves one way: after a few rows per group the plain read skips the atomic
                    if (live && !nul) {
                        const u64 e = minmax_encode(vtype, v);
                        unsigned long long* a = reinterpret_cast<unsigned long long*>(&s_acc[slot]);
                        if (op == YTGPU_AGG_MIN) {
                            if (e < *reinterpret_cast<volatile u64*>(a)) atomicMin(a, (unsigned long long)e);
                        } else {
                            if (e > *reinterpret_cast<volatile u64*>(a)) atomicMax(a, (unsigned long long)e);
                        }
                        if (s_nn[slot] == 0) s_nn[slot] = 1;
                    }
                    break;
                }
                if (live && !nul) {
                    const u64 e = minmax_encode(vtype, v);
                    if (op == YTGPU_AGG_MIN) {
                        if (e < __ldcg(&S.acc[slot])) atomicMin(&S.acc[slot], (unsigned long long)e);
                    } else {
                        if (e > __ldcg(&S.acc[slot])) atomicMax(&S.acc[slot], (unsigned long long)e);
                    }
                    if (__ldcg(&S.nn[slot]) == 0) S.nn[slot] = 1;
                }
                break;
            case YTGPU_AGG_ARGMIN:
            case YTGPU_AGG_ARGMAX:
                if (live && !nul) {  // both arguments must be non-null (builtin_function_profiler.cpp:1304-1309)
                    bool bnul;
                    const u64 bv = decode_at(by, (i64)i, &bnul);
                    if (!bnul) {
                        const u64 e = by_encode(by.value_type, bv);
                        if (phase == 0) {
                            if (op == YTGPU_AGG_ARGMIN) {
                                if (e < __ldcg(&S.acc[slot])) atomicMin(&S.acc[slot], (unsigned long long)e);
                            } else {
                                if (e > __ldcg(&S.acc[slot])) atomicMax(&S.acc[slot], (unsigned long long)e);
                            }
                            if (__ldcg(&S.nn[slot]) == 0) S.nn[slot] = 1;
                        } else if (e == S.acc[slot]) {
                            if (i < __ldcg(&S.row[slot])) atomicMin(&S.row[slot], (unsigned long long)i);
                        }
                    }
                }
                break;
            case YTGPU_AGG_FIRST:
                if (live && !nul && i < __ldcg(&S.row[slot])) atomicMin(&S.row[slot], (unsigned long long)i);
                break;
            default:
                break;
        }
    }
    if (cached) {
        __syncthreads();
        for (u32 k = threadIdx.x; k < slots; k += blockDim.x) {
            const u32 c = s_nn[k];
            if (c == 0) continue;
            if (extremum) {
                if (op == YTGPU_AGG_MIN) atomicMin(&S.acc[k], (unsigned long long)s_acc[k]);
                else atomicMax(&S.acc[k], (unsigned long long)s_acc[k]);
                S.nn[k] = 1;
                continue;
            }
            atomicAdd(&S.nn[k], (unsigned long long)c);
            if (op != YTGPU_AGG_COUNT) {
                if (vtype == YTGPU_TYPE_DOUBLE) atomicAdd(reinterpret_cast<double*>(&S.acc[k]), __longlong_as_double((long long)s_acc[k]));
                else atomicAdd(&S.acc[k], (unsigned long long)s_acc[k]);
            }
        }
    }
}

// ---- string-valued aggregates (MIN / MAX / FIRST / COUNT / ARGMIN / ARGMAX with a string column or by_column) ----
struct StringDev {
    const u8* heap;
    u64 heap_bytes;
    const u64* starts;
    const u32* lengths;
    const u8* nulls;  // nullable bytemap
    u32 present;      // 0: the argument is a scalar ColumnDev
};

// Value i of a string argument: false for NULL; a value that leaves the heap sets the error bit and counts as absent, so
// no later read goes outside the heap.
__device__ __forceinline__ bool string_at(const StringDev& c, u64 i, ytgpu_value* v, u32* bad) {
    if (c.nulls && c.nulls[i]) return false;
    const u64 s = c.starts[i];
    const u32 l = c.lengths[i];
    if (s > c.heap_bytes || (u64)l > c.heap_bytes - s) {
        *bad = 1;
        return false;
    }
    v->type = YTGPU_TYPE_STRING;
    v->length = l;
    v->data = s;
    return true;
}

__device__ __forceinline__ ytgpu_value string_of(const StringDev& c, u64 row) {
    ytgpu_value v{};
    v.type = YTGPU_TYPE_STRING;
    v.length = c.lengths[row];
    v.data = c.starts[row];
    return v;
}

// QL string order through the width-free key words of keys.cuh (a one-column, required, ascending String key): the order
// the long-key sort and the ordered partitioner already use.  Words are prefix-free, so the first differing word decides.
__device__ __forceinline__ int string_compare(const u8* heap, const ytgpu_value& a, const ytgpu_value& b) {
    KeyColLayout L{};
    L.type = YTGPU_TYPE_STRING;
    const u32 na = key_string_blocks(a.length), nb = key_string_blocks(b.length);
    const u32 nw = na < nb ? na : nb;
    for (u32 w = 0; w < nw; ++w) {
        const u64 x = key_col_word(L, a, heap, w), y = key_col_word(L, b, heap, w);
        if (x != y) return x < y ? -1 : 1;
    }
    return 0;
}

// The selection key of MIN / MAX (the string column itself) or ARGMIN / ARGMAX (by_column, string or scalar).
struct Selector {
    ColumnDev by;
    StringDev bs;
    bool larger;  // MAX / ARGMAX
    // (key(a), a) better than (key(b), b): a smaller (larger) key, the smaller row on equal keys.  b holds a selected row,
    // whose value was checked when it was installed.
    __device__ __forceinline__ bool better(u64 a, u64 b) const {
        int c;
        if (bs.present) {
            c = string_compare(bs.heap, string_of(bs, a), string_of(bs, b));
        } else {
            bool nul;
            const u64 ea = by_encode(by.value_type, decode_at(by, (i64)a, &nul));
            const u64 eb = by_encode(by.value_type, decode_at(by, (i64)b, &nul));
            c = ea < eb ? -1 : (ea > eb ? 1 : 0);
        }
        if (larger) c = -c;
        return c < 0 || (c == 0 && a < b);
    }
};

// Lock-free selection: install `cand` while it beats the holder.  A CAS fails only because another thread installed a
// better row; the inputs are immutable, so comparing against the winner again is enough.
__device__ __forceinline__ void select_row(unsigned long long* state, u64 cand, const Selector& sel) {
    u64 cur = __ldcg(state);
    while (cur == ~0ull || sel.better(cand, cur)) {
        const u64 old = atomicCAS(state, (unsigned long long)cur, (unsigned long long)cand);
        if (old == cur) return;
        cur = old;
    }
}

// Step 2 for an aggregate over a string column or by a string column.  State: S.row (selected row, ~0 = none) or, for
// COUNT, S.nn.  Every non-NULL string of the arguments is bounds-checked, including rows the predicate dropped.
__global__ void __launch_bounds__(256) mg_accumulate_strings_kernel(int op, const ColumnDev col, const StringDev cs, const ColumnDev by,
                                                                    const StringDev bs, u64 n, const u32* __restrict__ slot_of_row,
                                                                    AggState S, u32* err_word) {
    const bool arg = op == YTGPU_AGG_ARGMIN || op == YTGPU_AGG_ARGMAX;
    Selector sel;
    sel.larger = op == YTGPU_AGG_MAX || op == YTGPU_AGG_ARGMAX;
    if (arg) {
        sel.by = by;
        sel.bs = bs;
    } else {  // MIN / MAX select by the column itself
        sel.by = col;
        sel.bs = cs;
    }
    const u64 stride = (u64)gridDim.x * blockDim.x;
    const u64 trips = (n + stride - 1) / stride;  // the same for every thread: the warp collectives see whole warps
    u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    u32 bad = 0;
    for (u64 t = 0; t < trips; ++t, i += stride) {
        const bool in = i < n;
        const u32 slot = in ? slot_of_row[i] : kNoSlot;
        bool have = false;
        if (in) {
            ytgpu_value v;
            bool nul = true;
            if (cs.present) have = string_at(cs, i, &v, &bad);
            else {
                decode_at(col, (i64)i, &nul);
                have = !nul;
            }
            if (arg) {  // both arguments must be non-null (builtin_function_profiler.cpp:1304-1309)
                bool bhave;
                if (bs.present) bhave = string_at(bs, i, &v, &bad);
                else {
                    decode_at(by, (i64)i, &nul);
                    bhave = !nul;
                }
                have = have && bhave;
            }
        }
        have = have && slot != kNoSlot;
        const u32 slot0 = __shfl_sync(0xffffffffu, slot, 0);
        const bool uniform = __all_sync(0xffffffffu, slot == slot0) && slot0 != kNoSlot;  // sorted / clustered keys
        if (op == YTGPU_AGG_COUNT) {
            if (uniform) {
                const u32 cnt = __popc(__ballot_sync(0xffffffffu, have));
                if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&S.nn[slot], (unsigned long long)cnt);
            } else if (have) {
                atomicAdd(&S.nn[slot], 1ull);
            }
            continue;
        }
        if (op == YTGPU_AGG_FIRST) {
            if (have && i < __ldcg(&S.row[slot])) atomicMin(&S.row[slot], (unsigned long long)i);
            continue;
        }
        u64 cand = have ? i : ~0ull;
        if (uniform) {  // the warp's best row first: one CAS loop per warp instead of 32 on one address
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) {
                const u64 o = __shfl_xor_sync(0xffffffffu, cand, d);
                if (o != ~0ull && (cand == ~0ull || sel.better(o, cand))) cand = o;
            }
            if ((threadIdx.x & 31) != 0) cand = ~0ull;
        }
        if (cand != ~0ull) select_row(&S.row[slot], cand, sel);
    }
    if (bad) atomicOr(err_word, (u32)DE_STRING_OUT_OF_HEAP);
}

// Step 3a: occupied slots -> (first row, slot) pairs, order arbitrary (one atomicAdd per warp).
__global__ void __launch_bounds__(256) mg_compact_kernel(const u32* rep, u64 cap, const unsigned long long* first, u64* out_first,
                                                         u32* out_slot, u32* counter) {
    const u32 lane = threadIdx.x & 31;
    for (u64 base = (u64)blockIdx.x * blockDim.x; base < cap; base += (u64)gridDim.x * blockDim.x) {
        const u64 s = base + threadIdx.x;
        const bool occupied = s < cap && rep[s] != kNoSlot;
        const u32 m = __ballot_sync(0xffffffffu, occupied);
        if (m == 0) continue;
        u32 o = 0;
        if (lane == 0) o = atomicAdd(counter, (u32)__popc(m));
        o = __shfl_sync(0xffffffffu, o, 0) + __popc(m & ((1u << lane) - 1));
        if (occupied) {
            out_first[o] = first[s];
            out_slot[o] = (u32)s;
        }
    }
}

// Step 3b: keys, COUNT(*) and first rows in output order.
struct KeyOutputs {
    u64* keys[kMaxGroupKeys];
    u8* key_null[kMaxGroupKeys];
};
__global__ void __launch_bounds__(256) mg_emit_keys_kernel(const KeyColumns K, const SortPlan* plan, const u32* pa, const u32* pb, u64 g,
                                                           const u32* slots, const unsigned long long* first,
                                                           const unsigned long long* counts, KeyOutputs O, u64* out_counts,
                                                           u64* out_first, u32* out_slot_sorted) {
    const u64 o = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= g) return;
    const u32 slot = slots[perm_at(plan, pa, pb, o)];
    out_slot_sorted[o] = slot;
    const u64 row = first[slot];
    const KeyTuple t = load_tuple(K, row);
#pragma unroll
    for (u32 k = 0; k < (u32)kMaxGroupKeys; ++k)
        if (k < K.count) {
            O.keys[k][o] = t.w[k];
            O.key_null[k][o] = (t.nulls >> k) & 1;
        }
    if (out_counts) out_counts[o] = counts[slot];
    if (out_first) out_first[o] = row;
}

// Step 3c: one aggregate's result column.  row_result: a string-valued result, written as the selected row.
__global__ void __launch_bounds__(256) mg_finalize_kernel(int op, const ColumnDev col, u8 by_type, u64 g, const u32* slot_sorted, AggState S,
                                                          u64* out_value, u8* out_null, bool row_result) {
    const u64 o = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= g) return;
    const u32 slot = slot_sorted[o];
    const u8 vtype = col.value_type;
    u64 v = 0;
    bool nul = false;
    if (row_result) {
        v = S.row[slot];
        nul = v == ~0ull;
        out_value[o] = nul ? 0 : v;
        out_null[o] = nul ? 1 : 0;
        return;
    }
    switch (op) {
        case YTGPU_AGG_SUM:
            nul = S.nn[slot] == 0;
            v = S.acc[slot];
            break;
        case YTGPU_AGG_COUNT:
            v = S.nn[slot];
            break;
        case YTGPU_AGG_AVG: {  // Finalize: sum / count as double; NULL without values (builtin_function_profiler.cpp:1583-1620)
            const u64 c = S.nn[slot];
            nul = c == 0;
            if (!nul) {
                double s;
                if (vtype == YTGPU_TYPE_DOUBLE) s = __longlong_as_double((long long)S.acc[slot]);
                else if (vtype == YTGPU_TYPE_INT64) s = (double)(long long)S.acc[slot];
                else s = (double)(unsigned long long)S.acc[slot];
                v = (u64)__double_as_longlong(s / (double)(long long)c);
            }
            break;
        }
        case YTGPU_AGG_MIN:
        case YTGPU_AGG_MAX:
            nul = S.nn[slot] == 0;
            if (!nul) v = minmax_decode(vtype, S.acc[slot]);
            break;
        case YTGPU_AGG_ARGMIN:
        case YTGPU_AGG_ARGMAX:
        case YTGPU_AGG_FIRST: {
            const u64 row = S.row[slot];
            nul = row == ~0ull;
            if (!nul) {
                bool vn;
                v = decode_at(col, (i64)row, &vn);
                nul = vn;
            }
            break;
        }
        default:
            break;
    }
    out_value[o] = nul ? 0 : v;
    out_null[o] = nul ? 1 : 0;
}

bool aggregatable_type(u8 t) { return t == YTGPU_TYPE_INT64 || t == YTGPU_TYPE_UINT64 || t == YTGPU_TYPE_DOUBLE || t == YTGPU_TYPE_BOOLEAN; }

// A string column on the device (HOST inputs are uploaded).
struct StagedStrings {
    StringDev dev{};
    DevBuf<u8> heap, nulls;
    DevBuf<u64> starts;
    DevBuf<u32> lengths;
};

Status stage_strings(Context* ctx, const ytgpu_string_column& c, StagedStrings* s) {
    StringDev& d = s->dev;
    d.heap_bytes = c.heap_bytes;
    d.present = 1;
    if (c.mem != YTGPU_MEM_HOST) {
        d.heap = c.heap;
        d.starts = c.starts;
        d.lengths = c.lengths;
        d.nulls = c.null_bytemap;
        return Status{};
    }
    const u64 n = c.row_count;
    YTGPU_TRY(s->heap.allocate(ctx, c.heap_bytes));
    YTGPU_TRY(copy_in(ctx, s->heap.p, c.heap, c.heap_bytes, YTGPU_MEM_HOST));
    YTGPU_TRY(s->starts.allocate(ctx, n));
    YTGPU_TRY(copy_in(ctx, s->starts.p, c.starts, n * 8, YTGPU_MEM_HOST));
    YTGPU_TRY(s->lengths.allocate(ctx, n));
    YTGPU_TRY(copy_in(ctx, s->lengths.p, c.lengths, n * 4, YTGPU_MEM_HOST));
    d.heap = s->heap.p;
    d.starts = s->starts.p;
    d.lengths = s->lengths.p;
    d.nulls = nullptr;
    if (c.null_bytemap) {
        YTGPU_TRY(s->nulls.allocate(ctx, n));
        YTGPU_TRY(copy_in(ctx, s->nulls.p, c.null_bytemap, n, YTGPU_MEM_HOST));
        d.nulls = s->nulls.p;
    }
    return Status{};
}

Status groupby_multi_impl(Context* ctx, const ytgpu_column_view* key_columns, u32 key_count, const ytgpu_column_view* value_columns,
                          u32 value_count, const ytgpu_aggregate* aggregates, u32 aggregate_count, const ytgpu_predicate* pred,
                          int32_t pred_column, u64 hint, ytgpu_groupby_multi_result* out, int out_mem,
                          const ytgpu_string_column* string_columns, u32 string_count) {
    if (!key_columns || !out || (aggregate_count && !aggregates) || (value_count && !value_columns) || (string_count && !string_columns))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    // aggregate arguments index value_columns ++ string_columns
    const u64 columns_total = (u64)value_count + string_count;
    auto is_string = [&](int32_t c) { return (u32)c >= value_count; };
    if (key_count == 0 || key_count > (u32)kMaxGroupKeys)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key column count must be in [1, %d]", kMaxGroupKeys);
    if (aggregate_count > (u32)kMaxAggregates) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "at most %d aggregates", kMaxAggregates);
    if (!out->keys || !out->key_null || (aggregate_count && (!out->values || !out->value_null)))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null output array");
    const u64 n = (u64)key_columns[0].value_count;
    for (u32 k = 0; k < key_count; ++k)
        if ((u64)key_columns[k].value_count != n) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key columns differ in length");
    for (u32 v = 0; v < value_count; ++v)
        if ((u64)value_columns[v].value_count != n) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "value column %u differs in length", v);
    for (u32 s = 0; s < string_count; ++s) {
        const ytgpu_string_column& S = string_columns[s];
        if (S.row_count != n) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string column %u differs in length", s);
        if ((S.heap_bytes && !S.heap) || !S.starts || !S.lengths)  // an empty heap (all "" / NULL) is never read
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string column %u: null heap, starts or lengths", s);
        if (S.mem != YTGPU_MEM_DEVICE && S.mem != YTGPU_MEM_HOST)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string column %u: mem must be YTGPU_MEM_DEVICE or YTGPU_MEM_HOST", s);
    }
    if (n > (1ull << 30)) return make_status(YTGPU_ERR_UNSUPPORTED, "at most 2^30 rows per call (slots and rows are 32-bit)");
    const int op = pred ? pred->op : YTGPU_CMP_NONE;
    if (op != YTGPU_CMP_NONE && (pred_column < 0 || (u32)pred_column >= value_count))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "predicate column %d out of range", (int)pred_column);
    for (u32 a = 0; a < aggregate_count; ++a) {
        const ytgpu_aggregate& A = aggregates[a];
        if (A.op < YTGPU_AGG_SUM || A.op > YTGPU_AGG_FIRST) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "aggregate %u: unknown op %d", a, A.op);
        if (A.column < 0 || (u64)A.column >= columns_total) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "aggregate %u: column out of range", a);
        if (is_string(A.column)) {
            if (A.op == YTGPU_AGG_SUM || A.op == YTGPU_AGG_AVG)
                return make_status(YTGPU_ERR_UNSUPPORTED, "aggregate %u: sum / avg over a string column", a);
        } else {
            const u8 t = value_columns[A.column].value_type;
            if (!aggregatable_type(t)) return make_status(YTGPU_ERR_UNSUPPORTED, "aggregate %u: value type 0x%x is not a fixed-width scalar", a, t);
            if ((A.op == YTGPU_AGG_SUM || A.op == YTGPU_AGG_AVG) && t == YTGPU_TYPE_BOOLEAN)
                return make_status(YTGPU_ERR_UNSUPPORTED, "aggregate %u: sum / avg need int64, uint64 or double", a);
        }
        if (A.op == YTGPU_AGG_ARGMIN || A.op == YTGPU_AGG_ARGMAX) {
            if (A.by_column < 0 || (u64)A.by_column >= columns_total)
                return make_status(YTGPU_ERR_INVALID_ARGUMENT, "aggregate %u: by_column out of range", a);
            if (!is_string(A.by_column) && !aggregatable_type(value_columns[A.by_column].value_type))
                return make_status(YTGPU_ERR_UNSUPPORTED, "aggregate %u: by_column is not a fixed-width scalar", a);
        }
    }
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    out->group_count = 0;
    if (n == 0) return Status{};

    std::vector<StagedColumn> sk(key_count), sv(value_count);
    KeyColumns K{};
    K.count = key_count;
    for (u32 k = 0; k < key_count; ++k) {
        YTGPU_TRY(stage_column(ctx, &key_columns[k], &sk[k]));
        K.col[k] = sk[k].dev;
    }
    for (u32 v = 0; v < value_count; ++v) YTGPU_TRY(stage_column(ctx, &value_columns[v], &sv[v]));
    std::vector<StagedStrings> ss(string_count);
    for (u32 s = 0; s < string_count; ++s) YTGPU_TRY(stage_strings(ctx, string_columns[s], &ss[s]));
    bool keys_direct = true;  // plain 64-bit key vectors: the probe compares with one load per column
    for (u32 k = 0; k < key_count; ++k)
        keys_direct = keys_direct && is_direct64(sk[k].dev) && sk[k].dev.base == 0 && !sk[k].dev.zigzag;
    const ColumnDev pred_dev = op != YTGPU_CMP_NONE ? sv[pred_column].dev : ColumnDev{};
    const u64 constant = pred ? pred->constant : 0;

    // step 1 (the hint sizes the table; a full table doubles it and repeats the pass)
    u64 want = hint ? hint : std::min<u64>(n, 1ull << 20);  // no hint: start at 2^20 groups, a full table doubles and repeats
    if (want > n) want = n;
    u64 cap = 1024;
    // a warp waits for its longest probe chain (p99 of linear probing: 8 steps at load 1/2, 3 at 1/4): small tables are sized
    // for a load factor <= 1/4; big ones stay at <= 1/2 so that they keep fitting L2
    while (cap < want * 4 && cap < (1u << 16)) cap <<= 1;
    while (cap < want * 2) cap <<= 1;
    DevBuf<u32> rep, slot_of_row, counter;
    DevBuf<unsigned long long> counts, first;
    YTGPU_TRY(slot_of_row.allocate(ctx, n));
    YTGPU_TRY(counter.allocate(ctx, 1));
    const u32 threads = 256;
    const u32 all_rows_blocks = (u32)((n + threads - 1) / threads);
    const u32 cached_blocks = std::min<u32>(all_rows_blocks, (u32)kNumSms * 8);  // a CTA with shared-memory caches loops over rows and flushes once
    for (;;) {
        YTGPU_TRY(rep.allocate(ctx, cap));
        YTGPU_TRY(counts.allocate(ctx, cap));
        YTGPU_TRY(first.allocate(ctx, cap));
        YTGPU_CUDA_TRY(cudaMemsetAsync(rep.p, 0xff, cap * 4, ctx->stream));
        YTGPU_CUDA_TRY(cudaMemsetAsync(counts.p, 0, cap * 8, ctx->stream));
        YTGPU_CUDA_TRY(cudaMemsetAsync(first.p, 0xff, cap * 8, ctx->stream));
        {
            KernelTimer t(ctx, KC_GROUPBY);
            const u32 blocks = cap <= (u64)kSmemSlots ? cached_blocks : all_rows_blocks;
#define YTGPU_MG_ASSIGN(D, N)                                                                                                   \
    mg_assign_kernel<D, N><<<blocks, threads, 0, ctx->stream>>>(K, pred_dev, op, constant, n, rep.p, cap - 1, slot_of_row.p, counts.p, \
                                                                first.p, ctx->dev_err)
            if (keys_direct && key_count == 1) YTGPU_MG_ASSIGN(true, 1);
            else if (keys_direct && key_count == 2) YTGPU_MG_ASSIGN(true, 2);
            else if (keys_direct) YTGPU_MG_ASSIGN(true, 0);
            else if (key_count == 1) YTGPU_MG_ASSIGN(false, 1);
            else if (key_count == 2) YTGPU_MG_ASSIGN(false, 2);
            else YTGPU_MG_ASSIGN(false, 0);
#undef YTGPU_MG_ASSIGN
            YTGPU_CUDA_TRY(cudaGetLastError());
        }
        YTGPU_CUDA_TRY(cudaMemcpyAsync(ctx->host_err, ctx->dev_err, 4, cudaMemcpyDeviceToHost, ctx->stream));
        YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
        if ((*ctx->host_err & DE_TABLE_FULL) && cap < 4 * n) {
            const u32 rest = *ctx->host_err & ~(u32)DE_TABLE_FULL;
            YTGPU_CUDA_TRY(cudaMemcpyAsync(ctx->dev_err, &rest, 4, cudaMemcpyHostToDevice, ctx->stream));
            YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
            cap <<= 1;
            continue;
        }
        break;
    }
    if (*ctx->host_err) YTGPU_TRY(check_device_errors(ctx));

    // step 2
    std::vector<DevBuf<unsigned long long>> acc(aggregate_count), nn(aggregate_count), rows(aggregate_count);
    std::vector<AggState> states(aggregate_count);
    bool any_strings = false;
    for (u32 a = 0; a < aggregate_count; ++a) {
        const ytgpu_aggregate& A = aggregates[a];
        const bool arg = A.op == YTGPU_AGG_ARGMIN || A.op == YTGPU_AGG_ARGMAX;
        if (is_string(A.column) || (arg && is_string(A.by_column))) {
            // string state: the selected row, or the non-NULL count
            AggState S{nullptr, nullptr, nullptr};
            if (A.op == YTGPU_AGG_COUNT) {
                YTGPU_TRY(nn[a].allocate(ctx, cap));
                YTGPU_CUDA_TRY(cudaMemsetAsync(nn[a].p, 0, cap * 8, ctx->stream));
                S.nn = nn[a].p;
            } else {
                YTGPU_TRY(rows[a].allocate(ctx, cap));
                YTGPU_CUDA_TRY(cudaMemsetAsync(rows[a].p, 0xff, cap * 8, ctx->stream));
                S.row = rows[a].p;
            }
            states[a] = S;
            const bool col_str = is_string(A.column), by_str = arg && is_string(A.by_column);
            const ColumnDev col = col_str ? ColumnDev{} : sv[A.column].dev;
            const StringDev cs = col_str ? ss[A.column - value_count].dev : StringDev{};
            const ColumnDev by = arg && !by_str ? sv[A.by_column].dev : ColumnDev{};
            const StringDev bs = by_str ? ss[A.by_column - value_count].dev : StringDev{};
            KernelTimer t(ctx, KC_GROUPBY);
            mg_accumulate_strings_kernel<<<all_rows_blocks, threads, 0, ctx->stream>>>(A.op, col, cs, by, bs, n, slot_of_row.p, S,
                                                                                      ctx->dev_err);
            YTGPU_CUDA_TRY(cudaGetLastError());
            any_strings = true;
            continue;
        }
        const bool select_row = A.op == YTGPU_AGG_ARGMIN || A.op == YTGPU_AGG_ARGMAX || A.op == YTGPU_AGG_FIRST;
        const bool need_acc = A.op != YTGPU_AGG_COUNT && A.op != YTGPU_AGG_FIRST;
        AggState S{nullptr, nullptr, nullptr};
        if (need_acc) {
            YTGPU_TRY(acc[a].allocate(ctx, cap));
            const int fill = (A.op == YTGPU_AGG_MIN || A.op == YTGPU_AGG_ARGMIN) ? 0xff : 0;
            YTGPU_CUDA_TRY(cudaMemsetAsync(acc[a].p, fill, cap * 8, ctx->stream));
            S.acc = acc[a].p;
        }
        if (A.op != YTGPU_AGG_FIRST) {
            YTGPU_TRY(nn[a].allocate(ctx, cap));
            YTGPU_CUDA_TRY(cudaMemsetAsync(nn[a].p, 0, cap * 8, ctx->stream));
            S.nn = nn[a].p;
        }
        if (select_row) {
            YTGPU_TRY(rows[a].allocate(ctx, cap));
            YTGPU_CUDA_TRY(cudaMemsetAsync(rows[a].p, 0xff, cap * 8, ctx->stream));
            S.row = rows[a].p;
        }
        states[a] = S;
        const ColumnDev col = sv[A.column].dev;
        const ColumnDev by = arg ? sv[A.by_column].dev : ColumnDev{};
        KernelTimer t(ctx, KC_GROUPBY, arg ? 2 : 1);
        const u32 slots = cap <= (u64)kSmemSlots ? (u32)cap : 0xffffffffu;
        const bool smem_cached = A.op == YTGPU_AGG_SUM || A.op == YTGPU_AGG_AVG || A.op == YTGPU_AGG_COUNT || A.op == YTGPU_AGG_MIN || A.op == YTGPU_AGG_MAX;
        // the cached form holds 48 KB of shared memory per CTA: 512 threads keep the SM full with 4 CTAs
        const bool use_cache = smem_cached && cap <= (u64)kSmemSlots;
        const u32 acc_threads = use_cache ? 512 : threads;
        const u32 row_blocks = use_cache ? std::min<u32>((u32)((n + 511) / 512), (u32)kNumSms * 4) : all_rows_blocks;
        mg_accumulate_kernel<<<row_blocks, acc_threads, 0, ctx->stream>>>(A.op, 0, col, by, n, slots, slot_of_row.p, S);
        if (arg) mg_accumulate_kernel<<<row_blocks, acc_threads, 0, ctx->stream>>>(A.op, 1, col, by, n, slots, slot_of_row.p, S);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    if (any_strings) YTGPU_TRY(check_device_errors(ctx));  // a string that leaves its heap

    // step 3
    const u64 max_groups = std::min<u64>(n, cap);
    DevBuf<u64> cfirst;
    DevBuf<u32> cslot, slot_sorted;
    YTGPU_TRY(cfirst.allocate(ctx, max_groups));
    YTGPU_TRY(cslot.allocate(ctx, max_groups));
    YTGPU_CUDA_TRY(cudaMemsetAsync(counter.p, 0, 4, ctx->stream));
    mg_compact_kernel<<<blocks_for(cap, 256, 8), 256, 0, ctx->stream>>>(rep.p, cap, first.p, cfirst.p, cslot.p, counter.p);
    ctx->count_launch();
    u32 g32 = 0;
    YTGPU_CUDA_TRY(cudaMemcpyAsync(&g32, counter.p, 4, cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    const u64 g = g32;
    out->group_count = g;
    if (g > out->capacity)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "result has %llu groups, capacity is %llu", (unsigned long long)g,
                           (unsigned long long)out->capacity);
    if (g == 0) return Status{};

    SortScratch scratch;
    PermRef perm;
    const u64* cptr[1] = {cfirst.p};
    YTGPU_TRY(radix_sort_chunks(ctx, cptr, 1, g, &scratch, &perm));
    YTGPU_TRY(slot_sorted.allocate(ctx, g));

    const bool host = out_mem == YTGPU_MEM_HOST;
    std::vector<DevBuf<u64>> tk(key_count), tv(aggregate_count);
    std::vector<DevBuf<u8>> tkn(key_count), tvn(aggregate_count);
    DevBuf<u64> tcounts, tfirst;
    KeyOutputs O{};
    for (u32 k = 0; k < key_count; ++k) {
        if (!out->keys[k] || !out->key_null[k]) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null key output %u", k);
        O.keys[k] = out->keys[k];
        O.key_null[k] = out->key_null[k];
        if (host) {
            YTGPU_TRY(tk[k].allocate(ctx, g));
            YTGPU_TRY(tkn[k].allocate(ctx, g));
            O.keys[k] = tk[k].p;
            O.key_null[k] = tkn[k].p;
        }
    }
    u64 *dcounts = out->counts, *dfirst = out->first_rows;
    if (host && out->counts) {
        YTGPU_TRY(tcounts.allocate(ctx, g));
        dcounts = tcounts.p;
    }
    if (host && out->first_rows) {
        YTGPU_TRY(tfirst.allocate(ctx, g));
        dfirst = tfirst.p;
    }
    const u32 gblocks = (u32)((g + threads - 1) / threads);
    mg_emit_keys_kernel<<<gblocks, threads, 0, ctx->stream>>>(K, perm.plan, perm.idx[0], perm.idx[1], g, cslot.p, first.p, counts.p, O, dcounts,
                                                             dfirst, slot_sorted.p);
    ctx->count_launch();
    for (u32 a = 0; a < aggregate_count; ++a) {
        if (!out->values[a] || !out->value_null[a]) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null aggregate output %u", a);
        u64* dv = out->values[a];
        u8* dn = out->value_null[a];
        if (host) {
            YTGPU_TRY(tv[a].allocate(ctx, g));
            YTGPU_TRY(tvn[a].allocate(ctx, g));
            dv = tv[a].p;
            dn = tvn[a].p;
        }
        const ytgpu_aggregate& A = aggregates[a];
        const bool row_result = is_string(A.column) && A.op != YTGPU_AGG_COUNT;
        const ColumnDev col = is_string(A.column) ? ColumnDev{} : sv[A.column].dev;
        mg_finalize_kernel<<<gblocks, threads, 0, ctx->stream>>>(A.op, col, 0, g, slot_sorted.p, states[a], dv, dn, row_result);
        ctx->count_launch();
        if (host) {
            YTGPU_TRY(copy_out(ctx, out->values[a], dv, g * 8, YTGPU_MEM_HOST));
            YTGPU_TRY(copy_out(ctx, out->value_null[a], dn, g, YTGPU_MEM_HOST));
        }
    }
    YTGPU_CUDA_TRY(cudaGetLastError());
    if (host) {
        for (u32 k = 0; k < key_count; ++k) {
            YTGPU_TRY(copy_out(ctx, out->keys[k], O.keys[k], g * 8, YTGPU_MEM_HOST));
            YTGPU_TRY(copy_out(ctx, out->key_null[k], O.key_null[k], g, YTGPU_MEM_HOST));
        }
        if (out->counts) YTGPU_TRY(copy_out(ctx, out->counts, dcounts, g * 8, YTGPU_MEM_HOST));
        if (out->first_rows) YTGPU_TRY(copy_out(ctx, out->first_rows, dfirst, g * 8, YTGPU_MEM_HOST));
    }
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return Status{};
}

}  // namespace

extern "C" {

int ytgpu_scan_filter_groupby_multi(ytgpu_context* h, const ytgpu_column_view* key_columns, uint32_t key_count,
                                    const ytgpu_column_view* value_columns, uint32_t value_count, const ytgpu_aggregate* aggregates,
                                    uint32_t aggregate_count, const ytgpu_predicate* predicate, int32_t predicate_column,
                                    uint64_t group_count_hint, ytgpu_groupby_multi_result* out, int out_mem, ytgpu_error* err) {
    return ytgpu_scan_filter_groupby_multi_strings(h, key_columns, key_count, value_columns, value_count, aggregates, aggregate_count,
                                                   predicate, predicate_column, group_count_hint, out, out_mem, nullptr, 0, err);
}

int ytgpu_scan_filter_groupby_multi_strings(ytgpu_context* h, const ytgpu_column_view* key_columns, uint32_t key_count,
                                            const ytgpu_column_view* value_columns, uint32_t value_count,
                                            const ytgpu_aggregate* aggregates, uint32_t aggregate_count,
                                            const ytgpu_predicate* predicate, int32_t predicate_column, uint64_t group_count_hint,
                                            ytgpu_groupby_multi_result* out, int out_mem, const ytgpu_string_column* string_columns,
                                            uint32_t string_count, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, groupby_multi_impl(as_context(h), key_columns, key_count, value_columns, value_count, aggregates,
                                              aggregate_count, predicate, predicate_column, group_count_hint, out, out_mem,
                                              string_columns, string_count));
}

}  // extern "C"
