// groupby_agg.cuh — the aggregate states and kernels of the GROUP BY over key tuples, shared by the one-shot call
// (groupby_multi.cu) and the GROUP BY table (groupby_table.cu): the per-row accumulation into slot-indexed states (over
// scalar and string columns), the compaction of occupied slots and the finalisation of one aggregate's result column.
// TU-local, as key_tuple.cuh.
#pragma once

#include <algorithm>

#include "columnar.cuh"
#include "context.cuh"
#include "key_tuple.cuh"
#include "strings.cuh"

namespace {

using namespace ytgpu;

constexpr int kMaxAggregates = 32;

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

// Step 2 for one aggregate over a scalar column: its states for `cap` slots (acc / nn / row as the op needs them, in their
// initial values) and the pass (two for argmin / argmax) over the n rows' slots.  No synchronisation.
Status accumulate_scalar(Context* ctx, int op, const ColumnDev& col, const ColumnDev& by, u64 n, u64 cap, const u32* slot_of_row,
                         DevBuf<unsigned long long>* acc, DevBuf<unsigned long long>* nn, DevBuf<unsigned long long>* rows, AggState* out) {
    const bool arg = op == YTGPU_AGG_ARGMIN || op == YTGPU_AGG_ARGMAX;
    const bool select_row = arg || op == YTGPU_AGG_FIRST;
    const bool need_acc = op != YTGPU_AGG_COUNT && op != YTGPU_AGG_FIRST;
    AggState S{nullptr, nullptr, nullptr};
    if (need_acc) {
        YTGPU_TRY(acc->allocate(ctx, cap));
        const int fill = (op == YTGPU_AGG_MIN || op == YTGPU_AGG_ARGMIN) ? 0xff : 0;
        YTGPU_CUDA_TRY(cudaMemsetAsync(acc->p, fill, cap * 8, ctx->stream));
        S.acc = acc->p;
    }
    if (op != YTGPU_AGG_FIRST) {
        YTGPU_TRY(nn->allocate(ctx, cap));
        YTGPU_CUDA_TRY(cudaMemsetAsync(nn->p, 0, cap * 8, ctx->stream));
        S.nn = nn->p;
    }
    if (select_row) {
        YTGPU_TRY(rows->allocate(ctx, cap));
        YTGPU_CUDA_TRY(cudaMemsetAsync(rows->p, 0xff, cap * 8, ctx->stream));
        S.row = rows->p;
    }
    *out = S;
    const u32 threads = 256;
    const u32 all_rows_blocks = (u32)((n + threads - 1) / threads);
    KernelTimer t(ctx, KC_GROUPBY, arg ? 2 : 1);
    const u32 slots = cap <= (u64)kSmemSlots ? (u32)cap : 0xffffffffu;
    const bool smem_cached = op == YTGPU_AGG_SUM || op == YTGPU_AGG_AVG || op == YTGPU_AGG_COUNT || op == YTGPU_AGG_MIN || op == YTGPU_AGG_MAX;
    // the cached form holds 48 KB of shared memory per CTA: 512 threads keep the SM full with 4 CTAs
    const bool use_cache = smem_cached && cap <= (u64)kSmemSlots;
    const u32 acc_threads = use_cache ? 512 : threads;
    const u32 row_blocks = use_cache ? std::min<u32>((u32)((n + 511) / 512), (u32)kNumSms * 4) : all_rows_blocks;
    mg_accumulate_kernel<<<row_blocks, acc_threads, 0, ctx->stream>>>(op, 0, col, by, n, slots, slot_of_row, S);
    if (arg) mg_accumulate_kernel<<<row_blocks, acc_threads, 0, ctx->stream>>>(op, 1, col, by, n, slots, slot_of_row, S);
    YTGPU_CUDA_TRY(cudaGetLastError());
    return Status{};
}

}  // namespace
