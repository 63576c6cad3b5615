// key_tuple.cuh — the hash table over key tuples shared by GROUP BY (groupby_multi.cu) and the hash join (join.cu): the
// tuple load / compare / hash and the assign step, in which every row finds or claims the slot of its key tuple.
// Everything is TU-local (anonymous namespace) so several .cu files may include it.
#pragma once

#include <algorithm>

#include "columnar.cuh"
#include "context.cuh"

namespace {

using namespace ytgpu;

constexpr int kMaxGroupKeys = 8;
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

// A string key's dictionary ids as a key column: plain 64-bit values, with a null bitmap only when the strings have NULLs.
ColumnDev id_column(const u64* ids, const u32* null_bits, u64 n) {
    ColumnDev c{};
    c.count = (i64)n;
    c.values = ids;
    c.values_count = n;
    c.bitmap = reinterpret_cast<const u8*>(null_bits);
    c.bit_width = 64;
    c.has_values = 1;
    c.value_type = YTGPU_TYPE_UINT64;
    return c;
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

// The assign step over n rows with its table: rep[slot] = the row that claimed it, slot_of_row[row] = its slot (kNoSlot where
// the predicate drops the row), counts[slot] = rows of the key, first[slot] = its first row.
struct KeyTable {
    DevBuf<u32> rep, slot_of_row;
    DevBuf<unsigned long long> counts, first;
    u64 cap = 0;
};

// The hint (expected number of distinct tuples, 0 = unknown) sizes the table; a full table doubles it and repeats the pass.
// Synchronises the stream after every pass to read the error word.  n >= 1.
Status assign_key_slots(Context* ctx, int timer_class, const KeyColumns& K, bool keys_direct, const ColumnDev& pred_dev, int op,
                        u64 constant, u64 n, u64 hint, KeyTable* T) {
    const u32 key_count = K.count;
    u64 want = hint ? hint : std::min<u64>(n, 1ull << 20);  // no hint: start at 2^20 groups, a full table doubles and repeats
    if (want > n) want = n;
    u64 cap = 1024;
    // a warp waits for its longest probe chain (p99 of linear probing: 8 steps at load 1/2, 3 at 1/4): small tables are sized
    // for a load factor <= 1/4; big ones stay at <= 1/2 so that they keep fitting L2
    while (cap < want * 4 && cap < (1u << 16)) cap <<= 1;
    while (cap < want * 2) cap <<= 1;
    YTGPU_TRY(T->slot_of_row.allocate(ctx, n));
    const u32 threads = 256;
    const u32 all_rows_blocks = (u32)((n + threads - 1) / threads);
    const u32 cached_blocks = std::min<u32>(all_rows_blocks, (u32)kNumSms * 8);  // a CTA with shared-memory caches loops over rows and flushes once
    for (;;) {
        YTGPU_TRY(T->rep.allocate(ctx, cap));
        YTGPU_TRY(T->counts.allocate(ctx, cap));
        YTGPU_TRY(T->first.allocate(ctx, cap));
        YTGPU_CUDA_TRY(cudaMemsetAsync(T->rep.p, 0xff, cap * 4, ctx->stream));
        YTGPU_CUDA_TRY(cudaMemsetAsync(T->counts.p, 0, cap * 8, ctx->stream));
        YTGPU_CUDA_TRY(cudaMemsetAsync(T->first.p, 0xff, cap * 8, ctx->stream));
        {
            KernelTimer t(ctx, timer_class);
            const u32 blocks = cap <= (u64)kSmemSlots ? cached_blocks : all_rows_blocks;
#define YTGPU_MG_ASSIGN(D, N)                                                                                                   \
    mg_assign_kernel<D, N><<<blocks, threads, 0, ctx->stream>>>(K, pred_dev, op, constant, n, T->rep.p, cap - 1, T->slot_of_row.p, \
                                                                T->counts.p, T->first.p, ctx->dev_err)
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
    T->cap = cap;
    if (*ctx->host_err) YTGPU_TRY(check_device_errors(ctx));
    return Status{};
}

}  // namespace
