// columnar.cu — columnar decode and the fused scan -> filter -> hash-aggregate kernels.
//
// Decode mirrors DecodeIntegerVector (yt/yt/client/table_client/columnar-inl.h:355-376 with
// :66-182,:236-247), the null bytemaps of BuildNullBytemapForCHColumn
// (yt/chyt/server/columnar_conversion.cpp:948-999; columnar.cpp:350-383,603,638) and the bit-packed
// vector reader (yt/yt/core/misc/bit_packed_unsigned_vector-inl.h:156-173).
// The aggregate replaces DB::Aggregator's key64 hash table with SUM/COUNT states
// (contrib/clickhouse/src/Interpreters/Aggregator.cpp:1006,1486; AggregateFunctionSum.h:51-103) and
// YT QL's InsertGroupRow + sum (library/query/engine/cg_routines/registry.cpp:1783-1834,
// engine/udf/sum.c:12-36): decode, predicate and hash insert happen in ONE pass over the encoded
// columns, so the algorithmic traffic is the encoded bytes in + 24 B per group out.
#include <vector>

#include "columnar.cuh"
#include "context.cuh"
#include "radix_sort.cuh"
#include "rows.cuh"

using namespace ytgpu;

namespace {

template <bool DIRECT>
__device__ __forceinline__ u64 decode_value(const ColumnDev& c, const u64* __restrict__ direct, i64 i, bool* ch_null) {
    if (DIRECT) {
        *ch_null = false;
        u64 x = ld_stream_u64(direct + i) + c.base;
        if (c.zigzag) x = (x >> 1) ^ (0 - (x & 1));
        return x;
    }
    return decode_at(c, i, ch_null);
}

// Rows of a warp trip, with the run of the trip's first row as every lane's starting point when the column is run-length
// encoded: a warp then walks a contiguous share of the rows so that each trip's run is found from the previous one
// (one binary search over the runs per WARP; a search per row is a chain of 20 dependent loads at 10^6 runs).
struct WarpRows {
    u64 base, end, prev;
    bool rle;
    __device__ __forceinline__ WarpRows(const ColumnDev& c) : prev(kNoRleHint), rle(c.rle != nullptr && c.has_values) {
        const u64 n = (u64)c.count;
        const u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5, warps = ((u64)gridDim.x * blockDim.x) >> 5;
        const u64 per_warp = ((n + warps * 32 - 1) / (warps * 32)) * 32;
        base = min(n, warp * per_warp);
        end = min(n, base + per_warp);
    }
    __device__ __forceinline__ bool more() const { return base < end; }
    // all 32 lanes call; returns the run hint of this trip and advances
    __device__ __forceinline__ u64 next_hint(const ColumnDev& c, u64* row) {
        u64 h = kNoRleHint;
        if (rle) {
            u64 k = 0;
            if (lane_id() == 0)
                k = prev == kNoRleHint ? rle_pos(c.rle, c.rle_count, (u64)c.start + base) : rle_pos_gallop(c.rle, c.rle_count, (u64)c.start + base, prev);
            prev = h = __shfl_sync(0xffffffffu, k, 0);
        }
        *row = base + lane_id();
        base += 32;
        return h;
    }
};

__global__ void __launch_bounds__(256) decode_column_kernel(const ColumnDev c, u64* __restrict__ out,
                                                            u8* __restrict__ out_null) {
    WarpRows w(c);
    while (w.more()) {
        u64 i;
        const u64 hint = w.next_hint(c, &i);
        if (i >= (u64)c.count) continue;
        bool nul;
        u64 v = decode_at(c, (i64)i, &nul, hint);
        out[i] = v;
        if (out_null) out_null[i] = nul ? 1 : 0;
    }
}

// ConvertIntegerYTColumnToCHColumnImpl (yt/chyt/server/columnar_conversion.cpp:204-234): the decoded 64-bit value is
// narrowed by assignment to the ClickHouse element type; ConvertFloatingPointYTColumnToCHColumn (:341-369): a 32-bit float
// value vector read into a Float64 column is widened value by value.
template <class T>
__global__ void __launch_bounds__(256) decode_column_typed_kernel(const ColumnDev c, T* __restrict__ out, u8* __restrict__ out_null,
                                                                  bool widen_float) {
    WarpRows w(c);
    while (w.more()) {
        u64 i;
        const u64 hint = w.next_hint(c, &i);
        if (i >= (u64)c.count) continue;
        bool nul;
        u64 v = decode_at(c, (i64)i, &nul, hint);
        if (widen_float) v = (u64)__double_as_longlong((double)__uint_as_float((u32)v));
        out[i] = (T)v;
        if (out_null) out_null[i] = nul ? 1 : 0;
    }
}

__global__ void decode_string_offsets_kernel(const u32* __restrict__ enc, u32 avg, i64 start, i64 end,
                                             u32* __restrict__ out) {
    auto off = [&](i64 k) -> u32 {
        if (k == 0) return 0u;
        u32 z = enc[k - 1];
        return avg * (u32)k + ((z >> 1) ^ (0u - (z & 1)));
    };
    const u32 base = off(start);
    for (i64 k = start + (i64)blockIdx.x * blockDim.x + threadIdx.x; k <= end; k += (i64)gridDim.x * blockDim.x)
        out[k - start] = off(k) - base;
}

__global__ void decode_string_pointers_kernel(const u32* __restrict__ enc, u32 avg, u64 n, u32* __restrict__ out_start,
                                              i32* __restrict__ out_length) {
    auto end_of = [&](u64 k) -> i64 {  // end offset of value k
        const u32 z = enc[k];
        return (i64)avg * (i64)(k + 1) + (i64)((i64)(z >> 1) ^ -(i64)(z & 1));
    };
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        const i64 start = i ? end_of(i - 1) : 0, end = end_of(i);
        out_start[i] = (u32)start;
        out_length[i] = (i32)(end - start);
    }
}

// --------------------------------------------------------------------------------------------
// Hash aggregate
// --------------------------------------------------------------------------------------------
constexpr u64 kEmptyKey = ~0ull;

struct GroupTable {
    u64* keys;      // [cap + 2]; slot cap = the key equal to kEmptyKey, slot cap+1 = NULL key
    u64* sums;      // [cap + 2]
    unsigned long long* counts;  // [cap + 2]
    u32* has;       // [cap + 2] a non-null value was added
    unsigned long long* first;   // [cap + 2] smallest row index of the group (nullable: only when the caller asks)
    unsigned long long* mins;    // [cap + 2] MIN / MAX of the non-null values in an order-preserving unsigned encoding
    unsigned long long* maxs;    //           (nullable: only when the caller asks; global path only)
    u64 mask;       // cap - 1
};

// Two 32-bit multiplies and a shift: the table index comes from the TOP bits of the product sum.
__device__ __forceinline__ u32 key_hash32(u32 lo, u32 hi) { return lo * 0x9E3779B1u + hi * 0x85EBCA6Bu; }


// HAS = false: the value column cannot hold NULLs, "a non-null value was seen" == "the group has rows" (T.has unused).
template <bool HAS>
__device__ __forceinline__ void global_accumulate(const GroupTable& T, u64 slot, bool dbl, u64 sum_bits, bool has, unsigned long long cnt,
                                                  u64 first) {
    atomicAdd(&T.counts[slot], cnt);
    if (has) {
        if (dbl) atomicAdd(reinterpret_cast<double*>(&T.sums[slot]), __longlong_as_double((long long)sum_bits));
        else atomicAdd(reinterpret_cast<unsigned long long*>(&T.sums[slot]), (unsigned long long)sum_bits);
        if (HAS && T.has[slot] == 0) T.has[slot] = 1;
    }
    if (T.first) atomicMin(&T.first[slot], (unsigned long long)first);
}
// MIN / MAX only move one way, so a (possibly stale) plain read that already bounds the value proves the atomic
// unnecessary: after the first few rows of a group nearly every row skips both atomics, heavy keys do not contend.
__device__ __forceinline__ void global_minmax(const GroupTable& T, u64 slot, u64 enc_min, u64 enc_max) {
    if (enc_min < __ldcg(&T.mins[slot])) atomicMin(&T.mins[slot], (unsigned long long)enc_min);
    if (enc_max > __ldcg(&T.maxs[slot])) atomicMax(&T.maxs[slot], (unsigned long long)enc_max);
}

// The global table is probed in two-slot buckets too: one 16-byte load (one L2 sector) shows two keys, so a chain is
// half as long and the lanes of a warp leave the probe loop closer together (the ncu capture of the one-slot version:
// 14.4 active threads per instruction, 341 instructions per 32 rows at 10^6 groups).
struct Bucket2 {
    u64 k0, k1;
};
__device__ __forceinline__ Bucket2 load_bucket(const GroupTable& T, u64 b) {
    const ulonglong2 q = *reinterpret_cast<const ulonglong2*>(T.keys + 2 * b);
    return Bucket2{q.x, q.y};
}
__device__ __forceinline__ u64 global_hash(const GroupTable& T, u64 key) {  // -> bucket index
    return ((u64)(key_hash32((u32)key, (u32)(key >> 32)) ^ (u32)(key >> 29)) * 0x9E3779B97F4A7C15ull >> 20) & (T.mask >> 1);
}

// Slot of a regular key (not NULL, not kEmptyKey) in the global table, starting at bucket b whose two keys were just
// read; T.mask + 1 + error bit when the table is full.
__device__ __forceinline__ u64 global_find_slot(const GroupTable& T, u64 key, u64 b, Bucket2 q, u32* err) {
    const u64 buckets = (T.mask + 1) >> 1;
    for (u64 probes = 0; probes < buckets;) {
        if (q.k0 == key) return 2 * b;
        if (q.k1 == key) return 2 * b + 1;
        if (q.k0 == kEmptyKey || q.k1 == kEmptyKey) {
            const u64 e = 2 * b + (q.k0 == kEmptyKey ? 0 : 1);
            const u64 old = atomicCAS(reinterpret_cast<unsigned long long*>(&T.keys[e]), (unsigned long long)kEmptyKey, (unsigned long long)key);
            if (old == kEmptyKey || old == key) return e;
            q = load_bucket(T, b);  // another key took it: look at the bucket again
            continue;
        }
        b = (b + 1) & (buckets - 1);
        q = load_bucket(T, b);
        ++probes;
    }
    *err |= DE_TABLE_FULL;
    return T.mask + 1;
}

constexpr int kAggThreads = 512;          // x 2 CTAs per SM
constexpr int kLocalSlots = 4096;         // per-CTA front table: 2048 buckets of two slots, one LDS.128 per probe
constexpr int kLocalMaxGroups = 2048;     // hints up to this take the local path
constexpr int kLocalMaxProbes = 8;        // buckets looked at before a row goes to the global table instead
constexpr int kLocalSpecialEmpty = kLocalSlots;      // accumulator slot of the key equal to kEmptyKey
constexpr int kLocalSpecialNull = kLocalSlots + 1;   // accumulator slot of the NULL key

inline size_t local_smem_bytes(bool nn, bool first) {
    return (size_t)kLocalSlots * 8 + (size_t)(kLocalSlots + 2) * 8 + (size_t)(kLocalSlots + 2) * 4 * (1 + (nn ? 1 : 0) + (first ? 1 : 0)) + 16;
}

// One kernel for both regimes.  What made the round-1 kernel slow was not the atomics but DIVERGENCE: its probe loop
// exited lane by lane and the compiler sank the update code into every exit, so a warp executed the update sequence once
// per probe length (ncu: 5.25 active threads per instruction, 332-393 instructions per 32 rows).  Here every row's probe
// is a short loop that ends in __syncwarp(), the update runs ONCE per warp, carries are branch-free, and each thread
// handles two adjacent rows per trip (one 16-byte load per column) with the next trip's loads already in flight.
//   LOCAL : rows aggregate into a shared-memory table first (<= kLocalMaxGroups groups expected); rows whose bucket
//           chain is full go to the global table; the shared table is flushed once per CTA.
//   A warp whose 32 rows hold one key (sorted / RLE / dictionary-clustered chunks, the norm for YT tables) is reduced
//   with shuffles first and updates the table once.
//   PLAIN : both columns are plain 64-bit vectors without base / zig-zag, no predicate, no first-row request — the
//           configuration of the headline benchmark; the per-row work for those features is compiled out.
template <bool LOCAL, bool KDIRECT, bool VDIRECT, bool DBL, bool PLAIN = false>
__global__ void __launch_bounds__(kAggThreads, 2) groupby_kernel(const ColumnDev kc, const ColumnDev vc, int op, u64 constant,
                                                                 const GroupTable T, u32 want_first, u32* err_word) {
    constexpr bool NN = !VDIRECT;  // values may be NULL: count the non-null ones per group (SUM is NULL without any)
    extern __shared__ __align__(16) unsigned char gb_smem[];
    u64* s_keys = reinterpret_cast<u64*>(gb_smem);
    u64* s_sum = s_keys + kLocalSlots;
    u32* s_cnt = reinterpret_cast<u32*>(s_sum + kLocalSlots + 2);
    u32* s_nn = s_cnt + (kLocalSlots + 2);
    u32* s_first = s_nn + (NN ? kLocalSlots + 2 : 0);
    if (LOCAL) {
        for (int i = threadIdx.x; i < kLocalSlots + 2; i += kAggThreads) {
            if (i < kLocalSlots) s_keys[i] = kEmptyKey;
            s_sum[i] = 0;
            s_cnt[i] = 0;
            if (NN) s_nn[i] = 0;
            if (want_first) s_first[i] = 0xffffffffu;
        }
        __syncthreads();
    }
    u32 err = 0;
    const u8 vtype = vc.value_type;
    const u32 lane = threadIdx.x & 31;
    const u64* kdirect = reinterpret_cast<const u64*>(kc.values) + kc.start;
    const u64* vdirect = reinterpret_cast<const u64*>(vc.values) + vc.start;
    const bool kvec = KDIRECT && (reinterpret_cast<uintptr_t>(kdirect) & 15) == 0;
    const bool vvec = VDIRECT && (reinterpret_cast<uintptr_t>(vdirect) & 15) == 0;
    const u64 n = (u64)kc.count;
    // Run-length encoded columns: a warp walks a CONTIGUOUS share of the rows (64 per trip) so that the run of trip t + 1
    // is found from the run of trip t; with grid-strided trips every trip paid a binary search over all runs — 20
    // dependent loads x 330 trips per warp made the RLE variant latency bound (2.9 ms per 10^8 rows at 10^6 runs).
    const bool contiguous = (!KDIRECT && kc.rle && kc.has_values) || (!VDIRECT && vc.rle && vc.has_values);
    u64 stride = (u64)gridDim.x * kAggThreads * 2;
    u64 base = ((u64)blockIdx.x * kAggThreads + threadIdx.x) * 2;
    u64 trips = (n + stride - 1) / stride;  // the same for every lane of a warp: the warp collectives below see whole warps
    if (contiguous) {
        const u64 warp = ((u64)blockIdx.x * kAggThreads + threadIdx.x) >> 5, warps = ((u64)gridDim.x * kAggThreads) >> 5;
        const u64 per_warp = ((n + warps * 64 - 1) / (warps * 64)) * 64;
        const u64 wbegin = min(n, warp * per_warp), wend = min(n, wbegin + per_warp);
        stride = 64;
        base = wbegin + (u64)lane * 2;
        trips = (wend - wbegin + 63) / 64;
    }
    u64 kprev = kNoRleHint, vprev = kNoRleHint;  // the runs of the previous trip (contiguous walks only)

    // raw 64-bit words of the two rows of the NEXT trip (direct columns only)
    u64 nkey[2] = {0, 0}, nval[2] = {0, 0};
    auto prefetch = [&](u64 i0) {
        if (KDIRECT) {
            if (kvec && i0 + 1 < n) {
                const uint4 q = ld_stream_u128(reinterpret_cast<const uint4*>(kdirect + i0));
                nkey[0] = ((u64)q.y << 32) | q.x;
                nkey[1] = ((u64)q.w << 32) | q.z;
            } else {
                if (i0 < n) nkey[0] = ld_stream_u64(kdirect + i0);
                if (i0 + 1 < n) nkey[1] = ld_stream_u64(kdirect + i0 + 1);
            }
        }
        if (VDIRECT) {
            if (vvec && i0 + 1 < n) {
                const uint4 q = ld_stream_u128(reinterpret_cast<const uint4*>(vdirect + i0));
                nval[0] = ((u64)q.y << 32) | q.x;
                nval[1] = ((u64)q.w << 32) | q.z;
            } else {
                if (i0 < n) nval[0] = ld_stream_u64(vdirect + i0);
                if (i0 + 1 < n) nval[1] = ld_stream_u64(vdirect + i0 + 1);
            }
        }
    };
    prefetch(base);
    for (u64 t = 0; t < trips; ++t, base += stride) {
        const u64 ckey[2] = {nkey[0], nkey[1]}, cval[2] = {nval[0], nval[1]};
        prefetch(base + stride);
        // RLE columns: lane 0's first row is the smallest row of the warp's trip; its run (one binary search per warp) is
        // the starting point of every lane's short forward walk
        u64 khint = kNoRleHint, vhint = kNoRleHint;
        if (!KDIRECT && kc.rle && kc.has_values) {
            const u64 row0 = __shfl_sync(0xffffffffu, base, 0);
            u64 h = 0;
            if (lane == 0 && row0 < n)
                h = kprev == kNoRleHint ? rle_pos(kc.rle, kc.rle_count, (u64)kc.start + row0)
                                        : rle_pos_gallop(kc.rle, kc.rle_count, (u64)kc.start + row0, kprev);
            khint = __shfl_sync(0xffffffffu, h, 0);
            if (contiguous) kprev = khint;
        }
        if (!VDIRECT && vc.rle && vc.has_values) {
            const u64 row0 = __shfl_sync(0xffffffffu, base, 0);
            u64 h = 0;
            if (lane == 0 && row0 < n)
                h = vprev == kNoRleHint ? rle_pos(vc.rle, vc.rle_count, (u64)vc.start + row0)
                                        : rle_pos_gallop(vc.rle, vc.rle_count, (u64)vc.start + row0, vprev);
            vhint = __shfl_sync(0xffffffffu, h, 0);
            if (contiguous) vprev = vhint;
        }
        // ---- phase A: decode, filter, whole-warp reduction; both rows' first probes are issued before either is used ----
        u64 key[2], val[2];
        bool valid[2], knull[2], has[2];
        u32 cnt[2], nnc[2];
        u64 emin[2] = {~0ull, ~0ull}, emax[2] = {0, 0};  // MIN / MAX requested: order-preserving words of the row's value
        const bool minmax = !LOCAL && !PLAIN && T.mins != nullptr;
        u64 gh[2] = {0, 0};                    // global path: first bucket probed and the two keys found there
        Bucket2 gk0[2] = {{0, 0}, {0, 0}};
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const u64 i = base + r;
            valid[r] = i < n;
            knull[r] = false;
            bool vnull = !valid[r];
            key[r] = 0;
            val[r] = 0;
            if (valid[r]) {
                if (KDIRECT) {
                    key[r] = ckey[r];
                    if (!PLAIN) {
                        key[r] += kc.base;
                        if (kc.zigzag) key[r] = (key[r] >> 1) ^ (0 - (key[r] & 1));
                    }
                } else {
                    key[r] = decode_at(kc, (i64)i, &knull[r], khint);
                }
                if (VDIRECT) {
                    val[r] = cval[r];
                    if (!PLAIN) {
                        val[r] += vc.base;
                        if (vc.zigzag) val[r] = (val[r] >> 1) ^ (0 - (val[r] & 1));
                    }
                    vnull = false;
                } else {
                    val[r] = decode_at(vc, (i64)i, &vnull, vhint);
                }
                if (!PLAIN && op != YTGPU_CMP_NONE && (vnull || !passes(op, vtype, val[r], constant))) valid[r] = false;
            }
            has[r] = valid[r] && !vnull;
            if (!has[r]) val[r] = 0;
            cnt[r] = valid[r] ? 1u : 0u;
            nnc[r] = has[r] ? 1u : 0u;
            if (minmax && has[r]) emin[r] = emax[r] = minmax_encode(vtype, val[r]);
            // whole warp on one key (sorted / RLE / clustered key columns): reduce with shuffles, lane 0 updates once
            const u64 key0 = __shfl_sync(0xffffffffu, key[r], 0);
            if (__all_sync(0xffffffffu, valid[r] && !knull[r] && key[r] == key0)) {
                nnc[r] = __popc(__ballot_sync(0xffffffffu, has[r]));
#pragma unroll
                for (int d = 16; d > 0; d >>= 1) {
                    const u64 o = __shfl_xor_sync(0xffffffffu, val[r], d);
                    if (DBL) val[r] = (u64)__double_as_longlong(__longlong_as_double((long long)val[r]) + __longlong_as_double((long long)o));
                    else val[r] += o;
                }
                if (minmax) {
#pragma unroll
                    for (int d = 16; d > 0; d >>= 1) {
                        emin[r] = min(emin[r], __shfl_xor_sync(0xffffffffu, emin[r], d));
                        emax[r] = max(emax[r], __shfl_xor_sync(0xffffffffu, emax[r], d));
                    }
                }
                cnt[r] = 32;
                has[r] = nnc[r] != 0;
                if (lane != 0) valid[r] = false;  // lane 0 holds the smallest row index of the warp's 32 rows
            }
            if (!LOCAL && valid[r] && !knull[r] && key[r] != kEmptyKey) {
                gh[r] = global_hash(T, key[r]);
                gk0[r] = load_bucket(T, gh[r]);
            }
        }
        // ---- phase B: slot lookup + update, one row after the other ----
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const u64 i = base + r;
            int slot = -1;
            bool to_global = false;
            if (valid[r]) {
                if (knull[r] || key[r] == kEmptyKey) {
                    if (LOCAL) slot = knull[r] ? kLocalSpecialNull : kLocalSpecialEmpty;
                    else to_global = true;
                } else if (LOCAL) {
                    const u32 klo = (u32)key[r], khi = (u32)(key[r] >> 32);
                    u32 b = (key_hash32(klo, khi) >> 21) * 2;
                    int probes = 0;
                    while (slot < 0 && probes < kLocalMaxProbes) {
                        const uint4 kk = *reinterpret_cast<const uint4*>(&s_keys[b]);
                        if (kk.x == klo && kk.y == khi) slot = (int)b;
                        else if (kk.z == klo && kk.w == khi) slot = (int)b + 1;
                        else if ((kk.x & kk.y) == 0xffffffffu || (kk.z & kk.w) == 0xffffffffu) {
                            const u32 e = (kk.x & kk.y) == 0xffffffffu ? b : b + 1;
                            const u64 old = atomicCAS(reinterpret_cast<unsigned long long*>(&s_keys[e]), (unsigned long long)kEmptyKey,
                                                      (unsigned long long)key[r]);
                            if (old == kEmptyKey || old == key[r]) slot = (int)e;
                            // else another key took it: look at the bucket again
                        } else {
                            b = (b + 2) & (kLocalSlots - 1);
                            ++probes;
                        }
                    }
                    to_global = slot < 0;
                    if (to_global) {
                        gh[r] = global_hash(T, key[r]);
                        gk0[r] = load_bucket(T, gh[r]);
                    }
                } else {
                    to_global = true;
                }
            }
            u64 gslot = 0;
            if (valid[r] && to_global) {
                if (knull[r]) gslot = T.mask + 2;
                else if (key[r] == kEmptyKey) gslot = T.mask + 1;
                else gslot = global_find_slot(T, key[r], gh[r], gk0[r], &err);
            }
            __syncwarp();  // the updates below run once per warp, not once per probe length
            if (LOCAL && valid[r] && !to_global) {
                atomicAdd(&s_cnt[slot], cnt[r]);
                if (has[r]) {
                    if (DBL) {
                        atomicAdd(reinterpret_cast<double*>(&s_sum[slot]), __longlong_as_double((long long)val[r]));
                    } else {
                        // a 64-bit shared atomicAdd is a CAS loop; two native 32-bit adds with the carry of the low word
                        // are exact mod 2^64
                        u32* w = reinterpret_cast<u32*>(&s_sum[slot]);
                        const u32 lo = (u32)val[r];
                        const u32 old = atomicAdd(w, lo);
                        atomicAdd(w + 1, (u32)(val[r] >> 32) + (u32)(old + lo < old));
                    }
                    if (NN) atomicAdd(&s_nn[slot], nnc[r]);
                }
                if (!PLAIN && want_first) atomicMin(&s_first[slot], (u32)i);  // the local path runs for n < 2^32 only
            }
            if (valid[r] && to_global) {
                global_accumulate<NN>(T, gslot, DBL, val[r], has[r], (unsigned long long)cnt[r], i);
                if (minmax && has[r]) global_minmax(T, gslot, emin[r], emax[r]);
            }
        }
    }
    if (LOCAL) {
        __syncthreads();
        for (int i = threadIdx.x; i < kLocalSlots + 2; i += kAggThreads) {
            const u32 c = s_cnt[i];
            u64 gslot;
            if (i < kLocalSlots) {
                const u64 k = s_keys[i];
                if (k == kEmptyKey) continue;
                const u64 h = global_hash(T, k);
                gslot = global_find_slot(T, k, h, load_bucket(T, h), &err);
            } else {
                if (c == 0) continue;
                gslot = T.mask + 1 + (u64)(i - kLocalSlots);
            }
            const bool has = NN ? s_nn[i] != 0 : c != 0;
            // first rows travel as 32-bit offsets inside the chunk (the host only takes this path for n < 2^32)
            global_accumulate<NN>(T, gslot, DBL, s_sum[i], has, (unsigned long long)c, want_first ? (u64)s_first[i] : 0);
        }
    }
    if (err) atomicOr(err_word, err);
}

// Compacts occupied slots (order arbitrary); NULL-key group is appended by the host logic via slot cap+1.
// One atomicAdd per WARP reserves the output slots of its occupied lanes (a per-slot atomic on the single counter
// serialises: 10^6 groups cost 2 ms that way, 6*10^7 groups 24 ms).
__global__ void __launch_bounds__(256) compact_groups_kernel(const GroupTable T, u64* out_keys, u64* out_sums,
                                                             u64* out_counts, u8* out_sum_null, u64* out_first, u64* out_min, u64* out_max, u8 vtype,
                                                             u32* counter) {
    const u64 total = T.mask + 2;  // regular slots + the kEmptyKey slot
    const u32 lane = threadIdx.x & 31;
    for (u64 base = (u64)blockIdx.x * blockDim.x; base < total; base += (u64)gridDim.x * blockDim.x) {  // warp-uniform trips
        const u64 s = base + threadIdx.x;
        const bool occupied = s < total && (s <= T.mask ? T.keys[s] != kEmptyKey : T.counts[s] != 0);
        const u32 m = __ballot_sync(0xffffffffu, occupied);
        if (m == 0) continue;
        u32 o = 0;
        if (lane == 0) o = atomicAdd(counter, (u32)__popc(m));
        o = __shfl_sync(0xffffffffu, o, 0) + __popc(m & ((1u << lane) - 1));
        if (!occupied) continue;
        const bool has = T.has ? T.has[s] != 0 : T.counts[s] != 0;
        out_keys[o] = s <= T.mask ? T.keys[s] : kEmptyKey;
        out_sums[o] = has ? T.sums[s] : 0;
        out_counts[o] = T.counts[s];
        out_sum_null[o] = has ? 0 : 1;
        if (out_first) out_first[o] = T.first[s];
        if (out_min) {
            out_min[o] = has ? minmax_decode(vtype, T.mins[s]) : 0;
            out_max[o] = has ? minmax_decode(vtype, T.maxs[s]) : 0;
        }
    }
}

// Small results (the common case of the shared-memory regime): one CTA orders the compacted groups by key with a
// bitonic sort in shared memory and writes the output columns — instead of the general radix sort's ~20 launches.
constexpr int kSmallSortMax = 4096;
__global__ void __launch_bounds__(1024) small_sort_groups_kernel(u32 g, const u64* k, const u64* s, const u64* c, const u8* sn, const u64* f,
                                                                 const u64* mn, const u64* mx, u64* ok, u64* os, u64* oc, u8* osn, u8* okn,
                                                                 u64* of, u64* omn, u64* omx) {
    __shared__ u64 sk[kSmallSortMax];
    __shared__ u16 si[kSmallSortMax];
    u32 m = 1;
    while (m < g) m <<= 1;
    for (u32 i = threadIdx.x; i < m; i += blockDim.x) {
        sk[i] = i < g ? k[i] : ~0ull;
        si[i] = (u16)i;
    }
    __syncthreads();
    // keys are distinct except for padding (~0 may also be a real key: padding entries carry indices >= g and compare
    // greater through the index tie-break)
    for (u32 size = 2; size <= m; size <<= 1) {
        for (u32 stride = size >> 1; stride > 0; stride >>= 1) {
            for (u32 t = threadIdx.x; t < m / 2; t += blockDim.x) {
                const u32 lo = 2 * t - (t & (stride - 1));
                const u32 hi = lo + stride;
                const bool up = (lo & size) == 0;
                const u64 a = sk[lo], b = sk[hi];
                const u16 ia = si[lo], ib = si[hi];
                const bool gt = a > b || (a == b && ia > ib);
                if (gt == up) {
                    sk[lo] = b; sk[hi] = a;
                    si[lo] = ib; si[hi] = ia;
                }
            }
            __syncthreads();
        }
    }
    for (u32 i = threadIdx.x; i < g; i += blockDim.x) {
        const u32 j = si[i];
        ok[i] = k[j];
        os[i] = s[j];
        oc[i] = c[j];
        osn[i] = sn[j];
        okn[i] = 0;
        if (of) of[i] = f[j];
        if (omn) omn[i] = mn[j];
        if (omx) omx[i] = mx[j];
    }
}

__global__ void __launch_bounds__(256) gather_groups_kernel(const SortPlan* plan, const u32* pa, const u32* pb, u64 g,
                                                            const u64* k, const u64* s, const u64* c, const u8* sn, const u64* f,
                                                            const u64* mn, const u64* mx, u64* ok, u64* os, u64* oc, u8* osn, u8* okn,
                                                            u64* of, u64* omn, u64* omx) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < g; i += (u64)gridDim.x * blockDim.x) {
        u32 j = perm_at(plan, pa, pb, i);
        ok[i] = k[j];
        os[i] = s[j];
        oc[i] = c[j];
        osn[i] = sn[j];
        okn[i] = 0;
        if (of) of[i] = f[j];
        if (omn) omn[i] = mn[j];
        if (omx) omx[i] = mx[j];
    }
}

__global__ void append_null_group_kernel(const GroupTable T, u64 g, u8 vtype, u64* ok, u64* os, u64* oc, u8* osn, u8* okn, u64* of,
                                         u64* omn, u64* omx) {
    const u64 s = T.mask + 2;
    const bool has = T.has ? T.has[s] != 0 : T.counts[s] != 0;
    ok[g] = 0;
    os[g] = has ? T.sums[s] : 0;
    oc[g] = T.counts[s];
    osn[g] = has ? 0 : 1;
    okn[g] = 1;
    if (of) of[g] = T.first[s];
    if (omn) omn[g] = has ? minmax_decode(vtype, T.mins[s]) : 0;
    if (omx) omx[g] = has ? minmax_decode(vtype, T.maxs[s]) : 0;
}

// ---- host helpers ----

Status decode_column_impl(Context* ctx, const ytgpu_column_view* col, u64* out_values, u8* out_null, int out_mem) {
    if (!out_values) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null output");
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    StagedColumn sc;
    YTGPU_TRY(stage_column(ctx, col, &sc));
    const u64 n = (u64)col->value_count;
    if (n == 0) return Status{};
    OutBuf<u64> dv;
    OutBuf<u8> dn;
    YTGPU_TRY(dv.prepare(ctx, out_values, n, out_mem));
    YTGPU_TRY(dn.prepare(ctx, out_null, n, out_mem));
    {
        KernelTimer t(ctx, KC_DECODE);
        decode_column_kernel<<<blocks_for(n, 256, 8), 256, 0, ctx->stream>>>(sc.dev, dv.p, dn.p);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_TRY(dv.download(ctx, n));
    YTGPU_TRY(dn.download(ctx, n));
    if (col->mem == YTGPU_MEM_HOST || out_mem == YTGPU_MEM_HOST) YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return Status{};
}

Status decode_column_typed_impl(Context* ctx, const ytgpu_column_view* col, u32 element_bytes, void* out_values, u8* out_null, int out_mem) {
    if (!out_values || !col) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    if (element_bytes != 1 && element_bytes != 2 && element_bytes != 4 && element_bytes != 8)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "element size must be 1, 2, 4 or 8 bytes");
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    StagedColumn sc;
    YTGPU_TRY(stage_column(ctx, col, &sc));
    const u64 n = (u64)col->value_count;
    if (n == 0) return Status{};
    const bool is_float32 = col->value_type == YTGPU_TYPE_DOUBLE && col->bit_width == 32;
    if (is_float32 && element_bytes != 4 && element_bytes != 8)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "a float value vector converts to Float32 or Float64");
    OutBuf<u8> ov, on;
    YTGPU_TRY(ov.prepare(ctx, static_cast<u8*>(out_values), n * element_bytes, out_mem));
    YTGPU_TRY(on.prepare(ctx, out_null, n, out_mem));
    void* dv = ov.p;
    u8* dn = on.p;
    {
        KernelTimer t(ctx, KC_DECODE);
        const unsigned blocks = blocks_for(n, 256, 8);
        const bool widen = is_float32 && element_bytes == 8;
        switch (element_bytes) {
            case 1: decode_column_typed_kernel<u8><<<blocks, 256, 0, ctx->stream>>>(sc.dev, static_cast<u8*>(dv), dn, widen); break;
            case 2: decode_column_typed_kernel<u16><<<blocks, 256, 0, ctx->stream>>>(sc.dev, static_cast<u16*>(dv), dn, widen); break;
            case 4: decode_column_typed_kernel<u32><<<blocks, 256, 0, ctx->stream>>>(sc.dev, static_cast<u32*>(dv), dn, widen); break;
            default: decode_column_typed_kernel<u64><<<blocks, 256, 0, ctx->stream>>>(sc.dev, static_cast<u64*>(dv), dn, widen); break;
        }
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_TRY(ov.download(ctx, n * element_bytes));
    YTGPU_TRY(on.download(ctx, n));
    if (col->mem == YTGPU_MEM_HOST || out_mem == YTGPU_MEM_HOST) YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return Status{};
}

Status groupby_impl(Context* ctx, const ytgpu_column_view* kcol, const ytgpu_column_view* vcol,
                    const ytgpu_predicate* pred, u64 hint, ytgpu_groupby_result* out, int out_mem) {
    if (!kcol || !vcol || !out) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    if (kcol->value_count != vcol->value_count)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key and value columns differ in length");
    if (vcol->value_type != YTGPU_TYPE_INT64 && vcol->value_type != YTGPU_TYPE_UINT64 && vcol->value_type != YTGPU_TYPE_DOUBLE)
        return make_status(YTGPU_ERR_UNSUPPORTED, "SUM supports int64/uint64/double value columns");
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    const u64 n = (u64)kcol->value_count;
    out->group_count = 0;
    if (n == 0) return Status{};
    StagedColumn sk, sv;
    YTGPU_TRY(stage_column(ctx, kcol, &sk));
    YTGPU_TRY(stage_column(ctx, vcol, &sv));
    const bool want_first = out->first_rows != nullptr;
    const bool want_minmax = out->mins != nullptr || out->maxs != nullptr;
    const u8 vtype = vcol->value_type;
    const bool dbl = vcol->value_type == YTGPU_TYPE_DOUBLE;
    const int op = pred ? pred->op : YTGPU_CMP_NONE;
    const u64 constant = pred ? pred->constant : 0;
    const bool kd = is_direct64(sk.dev), vd = is_direct64(sv.dev);
    // the shared-memory front table serves small expected cardinalities (its first-row words are 32-bit)
    // (MIN / MAX live in the global table only)
    const bool local = hint != 0 && hint <= (u64)kLocalMaxGroups && n < (1ull << 32) && !want_minmax;

    // `hint` is a hint: when the table turns out too small the pass is repeated with a doubled table.
    u64 want = hint ? hint : n;
    if (want > n) want = n;
    u64 cap = 1024;
    while (cap < want * 2) cap <<= 1;
    DevBuf<u64> keys, sums;
    DevBuf<unsigned long long> counts, first, mins, maxs;
    DevBuf<u32> has, counter;
    DevBuf<u64> ck, cs, cc, cf, cmn, cmx;
    DevBuf<u8> csn;
    u32 g32 = 0;
    unsigned long long null_count = 0;
    YTGPU_TRY(counter.allocate(ctx, 1));
    GroupTable T{};
    for (;;) {
        YTGPU_TRY(keys.allocate(ctx, cap + 2));
        YTGPU_TRY(sums.allocate(ctx, cap + 2));
        YTGPU_TRY(counts.allocate(ctx, cap + 2));
        if (!vd) YTGPU_TRY(has.allocate(ctx, cap + 2));
        if (want_first) YTGPU_TRY(first.allocate(ctx, cap + 2));
        if (want_minmax) {
            YTGPU_TRY(mins.allocate(ctx, cap + 2));
            YTGPU_TRY(maxs.allocate(ctx, cap + 2));
            YTGPU_CUDA_TRY(cudaMemsetAsync(mins.p, 0xff, (cap + 2) * 8, ctx->stream));
            YTGPU_CUDA_TRY(cudaMemsetAsync(maxs.p, 0, (cap + 2) * 8, ctx->stream));
        }
        YTGPU_CUDA_TRY(cudaMemsetAsync(keys.p, 0xff, (cap + 2) * 8, ctx->stream));
        YTGPU_CUDA_TRY(cudaMemsetAsync(sums.p, 0, (cap + 2) * 8, ctx->stream));
        YTGPU_CUDA_TRY(cudaMemsetAsync(counts.p, 0, (cap + 2) * 8, ctx->stream));
        if (!vd) YTGPU_CUDA_TRY(cudaMemsetAsync(has.p, 0, (cap + 2) * 4, ctx->stream));
        if (want_first) YTGPU_CUDA_TRY(cudaMemsetAsync(first.p, 0xff, (cap + 2) * 8, ctx->stream));
        YTGPU_CUDA_TRY(cudaMemsetAsync(counter.p, 0, 4, ctx->stream));
        T = GroupTable{keys.p, sums.p, counts.p, vd ? nullptr : has.p, want_first ? first.p : nullptr,
                       want_minmax ? mins.p : nullptr, want_minmax ? maxs.p : nullptr, cap - 1};
        {
            KernelTimer t(ctx, KC_GROUPBY);
            const u64 pairs = (n + 1) / 2;
            const u32 grid = (u32)std::max<u64>(1, std::min<u64>((pairs + kAggThreads - 1) / kAggThreads, (u64)kNumSms * 2));
            const size_t smem = local ? local_smem_bytes(!vd, want_first) : 0;
#define YTGPU_GB(L, K, V, D)                                                                                                      \
    do {                                                                                                                          \
        if (L) cudaFuncSetAttribute(groupby_kernel<L, K, V, D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)local_smem_bytes(true, true)); \
        groupby_kernel<L, K, V, D><<<grid, kAggThreads, smem, ctx->stream>>>(sk.dev, sv.dev, op, constant, T, want_first ? 1u : 0u, ctx->dev_err); \
    } while (0)
#define YTGPU_GB_KV(L, D)                          \
    do {                                           \
        if (kd && vd) YTGPU_GB(L, true, true, D);  \
        else if (kd) YTGPU_GB(L, true, false, D);  \
        else if (vd) YTGPU_GB(L, false, true, D);  \
        else YTGPU_GB(L, false, false, D);         \
    } while (0)
            const bool plain = kd && vd && op == YTGPU_CMP_NONE && !want_first && !want_minmax && sk.dev.base == 0 && sv.dev.base == 0 && !sk.dev.zigzag &&
                               !sv.dev.zigzag;
#define YTGPU_GB_PLAIN(L, D)                                                                                                       \
    do {                                                                                                                           \
        if (L) cudaFuncSetAttribute(groupby_kernel<L, true, true, D, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)local_smem_bytes(true, true)); \
        groupby_kernel<L, true, true, D, true><<<grid, kAggThreads, smem, ctx->stream>>>(sk.dev, sv.dev, op, constant, T, 0u, ctx->dev_err);      \
    } while (0)
            if (plain) {
                if (local && dbl) YTGPU_GB_PLAIN(true, true);
                else if (local) YTGPU_GB_PLAIN(true, false);
                else if (dbl) YTGPU_GB_PLAIN(false, true);
                else YTGPU_GB_PLAIN(false, false);
            } else if (local) {
                if (dbl) YTGPU_GB_KV(true, true);
                else YTGPU_GB_KV(true, false);
            } else {
                if (dbl) YTGPU_GB_KV(false, true);
                else YTGPU_GB_KV(false, false);
            }
#undef YTGPU_GB_PLAIN
#undef YTGPU_GB_KV
#undef YTGPU_GB
            YTGPU_CUDA_TRY(cudaGetLastError());
        }
        // compact right away (cheap) so that one host round trip fetches the error word, the group count and the
        // NULL-key count together
        const u64 max_groups = std::min<u64>(n, cap + 1);
        YTGPU_TRY(ck.allocate(ctx, max_groups));
        YTGPU_TRY(cs.allocate(ctx, max_groups));
        YTGPU_TRY(cc.allocate(ctx, max_groups));
        YTGPU_TRY(csn.allocate(ctx, max_groups));
        if (want_first) YTGPU_TRY(cf.allocate(ctx, max_groups));
        if (want_minmax) {
            YTGPU_TRY(cmn.allocate(ctx, max_groups));
            YTGPU_TRY(cmx.allocate(ctx, max_groups));
        }
        compact_groups_kernel<<<blocks_for(cap + 2, 256, 8), 256, 0, ctx->stream>>>(T, ck.p, cs.p, cc.p, csn.p, want_first ? cf.p : nullptr,
                                                                                    want_minmax ? cmn.p : nullptr, want_minmax ? cmx.p : nullptr,
                                                                                    vtype, counter.p);
        ctx->count_launch();
        YTGPU_CUDA_TRY(cudaMemcpyAsync(ctx->host_err, ctx->dev_err, 4, cudaMemcpyDeviceToHost, ctx->stream));
        YTGPU_CUDA_TRY(cudaMemcpyAsync(&g32, counter.p, 4, cudaMemcpyDeviceToHost, ctx->stream));
        YTGPU_CUDA_TRY(cudaMemcpyAsync(&null_count, counts.p + cap + 1, 8, cudaMemcpyDeviceToHost, ctx->stream));
        YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
        // table full -> double it and repeat the pass (the hint was too small)
        if ((*ctx->host_err & DE_TABLE_FULL) && cap < 2 * n) {
            const u32 rest = *ctx->host_err & ~(u32)DE_TABLE_FULL;
            YTGPU_CUDA_TRY(cudaMemcpyAsync(ctx->dev_err, &rest, 4, cudaMemcpyHostToDevice, ctx->stream));
            YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
            cap <<= 1;
            continue;
        }
        break;
    }
    if (*ctx->host_err) YTGPU_TRY(check_device_errors(ctx));

    const u64 g = g32;
    const u64 total = g + (null_count ? 1 : 0);
    out->group_count = total;
    if (total > out->capacity)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "result has %llu groups, capacity is %llu",
                           (unsigned long long)total, (unsigned long long)out->capacity);
    if (total == 0) return Status{};

    OutBuf<u64> ok, os, oc, of, omn, omx;
    OutBuf<u8> osn, okn;
    YTGPU_TRY(ok.prepare(ctx, out->keys, total, out_mem));
    YTGPU_TRY(os.prepare(ctx, out->sums, total, out_mem));
    YTGPU_TRY(oc.prepare(ctx, out->counts, total, out_mem));
    YTGPU_TRY(osn.prepare(ctx, out->sum_null, total, out_mem));
    YTGPU_TRY(okn.prepare(ctx, out->key_null, total, out_mem));
    YTGPU_TRY(of.prepare(ctx, out->first_rows, total, out_mem));
    YTGPU_TRY(omn.prepare(ctx, out->mins, total, out_mem));
    YTGPU_TRY(omx.prepare(ctx, out->maxs, total, out_mem));
    u64 *dk = ok.p, *ds = os.p, *dc = oc.p, *df = of.p, *dmn = omn.p, *dmx = omx.p;
    u8 *dsn = osn.p, *dkn = okn.p;
    SortScratch scratch;
    if (g && g <= (u64)kSmallSortMax) {
        small_sort_groups_kernel<<<1, 1024, 0, ctx->stream>>>((u32)g, ck.p, cs.p, cc.p, csn.p, want_first ? cf.p : nullptr, cmn.p, cmx.p, dk, ds, dc, dsn, dkn, df,
                                                            dmn, dmx);
        ctx->count_launch();
    } else if (g) {
        PermRef perm;
        const u64* cptr[1] = {ck.p};
        YTGPU_TRY(radix_sort_chunks(ctx, cptr, 1, g, &scratch, &perm));
        gather_groups_kernel<<<blocks_for(g, 256, 8), 256, 0, ctx->stream>>>(perm.plan, perm.idx[0], perm.idx[1], g, ck.p, cs.p,
                                                                             cc.p, csn.p, want_first ? cf.p : nullptr, cmn.p, cmx.p, dk, ds, dc,
                                                                             dsn, dkn, df, dmn, dmx);
        ctx->count_launch();
    }
    if (null_count) {
        append_null_group_kernel<<<1, 1, 0, ctx->stream>>>(T, g, vtype, dk, ds, dc, dsn, dkn, df, dmn, dmx);
        ctx->count_launch();
    }
    YTGPU_CUDA_TRY(cudaGetLastError());
    YTGPU_TRY(ok.download(ctx, total));
    YTGPU_TRY(os.download(ctx, total));
    YTGPU_TRY(oc.download(ctx, total));
    YTGPU_TRY(osn.download(ctx, total));
    YTGPU_TRY(okn.download(ctx, total));
    YTGPU_TRY(of.download(ctx, total));
    YTGPU_TRY(omn.download(ctx, total));
    YTGPU_TRY(omx.download(ctx, total));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return Status{};
}

}  // namespace

extern "C" {

int ytgpu_decode_column(ytgpu_context* h, const ytgpu_column_view* column, uint64_t* out_values,
                        uint8_t* out_null_bytemap, int out_mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, decode_column_impl(as_context(h), column, out_values, out_null_bytemap, out_mem));
}

int ytgpu_decode_column_typed(ytgpu_context* h, const ytgpu_column_view* column, uint32_t element_bytes, void* out_values,
                              uint8_t* out_null_bytemap, int out_mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, decode_column_typed_impl(as_context(h), column, element_bytes, out_values, out_null_bytemap, out_mem));
}

int ytgpu_decode_string_offsets(ytgpu_context* h, const uint32_t* encoded, uint32_t avg_length, int64_t start_index,
                                int64_t end_index, uint32_t* out, int mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    Context* ctx = as_context(h);
    if (start_index < 0 || end_index < start_index || !out)
        return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "bad offset range"));
    auto run = [&]() -> Status {
        YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
        const u64 cnt = (u64)(end_index - start_index + 1);
        InBuf<u32> e;
        OutBuf<u32> o;
        YTGPU_TRY(e.stage(ctx, encoded, (size_t)end_index, mem));  // the offset of value k reads encoded[k - 1]
        YTGPU_TRY(o.prepare(ctx, out, cnt, mem));
        {
            KernelTimer t(ctx, KC_DECODE);
            decode_string_offsets_kernel<<<blocks_for(cnt, 256, 8), 256, 0, ctx->stream>>>(e.p, avg_length, start_index, end_index, o.p);
            YTGPU_CUDA_TRY(cudaGetLastError());
        }
        if (mem == YTGPU_MEM_HOST) {
            YTGPU_TRY(o.download(ctx, cnt));
            YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
        }
        return Status{};
    };
    return fill_error(err, run());
}

int ytgpu_decode_string_pointers_and_lengths(ytgpu_context* h, const uint32_t* encoded, uint32_t avg_length, uint64_t count,
                                             uint32_t* out_start, int32_t* out_length, int mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    Context* ctx = as_context(h);
    if ((!encoded && count) || !out_start || !out_length) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument"));
    auto run = [&]() -> Status {
        if (count == 0) return Status{};
        YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
        InBuf<u32> e;
        OutBuf<u32> os;
        OutBuf<i32> ol;
        YTGPU_TRY(e.stage(ctx, encoded, count, mem));
        YTGPU_TRY(os.prepare(ctx, out_start, count, mem));
        YTGPU_TRY(ol.prepare(ctx, out_length, count, mem));
        {
            KernelTimer t(ctx, KC_DECODE);
            decode_string_pointers_kernel<<<blocks_for(count, 256, 8), 256, 0, ctx->stream>>>(e.p, avg_length, count, os.p, ol.p);
            YTGPU_CUDA_TRY(cudaGetLastError());
        }
        if (mem == YTGPU_MEM_HOST) {
            YTGPU_TRY(os.download(ctx, count));
            YTGPU_TRY(ol.download(ctx, count));
            YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
        }
        return Status{};
    };
    return fill_error(err, run());
}

int ytgpu_scan_filter_groupby(ytgpu_context* h, const ytgpu_column_view* key_column, const ytgpu_column_view* value_column,
                              const ytgpu_predicate* predicate, uint64_t group_count_hint, ytgpu_groupby_result* out,
                              int out_mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, groupby_impl(as_context(h), key_column, value_column, predicate, group_count_hint, out, out_mem));
}

}  // extern "C"
