// reduce.cu — segmented SUM / COUNT over rows that are ALREADY SORTED by the group key: the aggregate stage of the
// sort -> aggregate pipeline (BASELINE.json configs[4]).
//
// Reference shape: a sorted reduce / QL GROUP BY over a sorted stream needs no hash table — consecutive rows with equal
// keys form a group (yt/yt/library/query/engine/cg_routines/registry.cpp:1838-1920 aggregates the rows of one group
// before moving on; sort_controller.cpp:3444-3456 feeds sorted partitions to the next stage).  Same results as
// ytgpu_scan_filter_groupby over the same rows (integer sums wrap mod 2^64, COUNT(*) counts rows); groups come out in key
// order, which on sorted input IS first-seen order.
//
// One pass over the rows (64 B read per row, 24 B written per group): a tile of 2048 rows counts its group heads,
// publishes the count, obtains the number of groups before it by decoupled look-back over the tile status words (the same
// chained-scan idiom as the radix passes), and every thread adds the partial (sum, count) of each run it holds to the
// group's output slot.
#include "context.cuh"

using namespace ytgpu;

namespace {

constexpr int kRedThreads = 256;
constexpr int kRedItems = 8;
constexpr int kRedTile = kRedThreads * kRedItems;
constexpr u64 kRedPartial = 1ull << 62, kRedInclusive = 2ull << 62, kRedMask = (1ull << 62) - 1;

__device__ __forceinline__ u64 ld_volatile_u64(const u64* p) {
    u64 v;
    asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ void st_volatile_u64(u64* p, u64 v) { asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(p), "l"(v)); }

template <bool DBL>
__global__ void __launch_bounds__(kRedThreads) reduce_sorted_kernel(const u8* __restrict__ rows, u64 n, u32 row_bytes, u32 key_off, u32 val_off,
                                                                    u64* __restrict__ status, u32* __restrict__ tile_counter,
                                                                    u64* __restrict__ out_keys, u64* __restrict__ out_sums,
                                                                    unsigned long long* __restrict__ out_counts, u64 capacity,
                                                                    u64* __restrict__ group_count, u32* err_word) {
    __shared__ u32 s_warp[kRedThreads / 32];
    __shared__ u32 s_tile;
    __shared__ u64 s_base;
    if (threadIdx.x == 0) s_tile = atomicAdd(tile_counter, 1u);  // tiles are numbered in start order: look-back never waits on a tile that has not started
    __syncthreads();
    const u64 tile = s_tile;
    const u64 first = tile * kRedTile + (u64)threadIdx.x * kRedItems;
    u64 key[kRedItems], val[kRedItems];
    u64 prev = 0;
    if (first < n && first > 0) prev = *reinterpret_cast<const u64*>(rows + (first - 1) * row_bytes + key_off);
#pragma unroll
    for (int j = 0; j < kRedItems; ++j) {
        const u64 r = first + j;
        if (r < n) {
            const u8* p = rows + r * row_bytes;
            key[j] = ld_stream_u64(reinterpret_cast<const u64*>(p + key_off));
            val[j] = ld_stream_u64(reinterpret_cast<const u64*>(p + val_off));
        } else {
            key[j] = 0;
            val[j] = 0;
        }
    }
    u32 heads = 0;  // bit j: row j starts a group
#pragma unroll
    for (int j = 0; j < kRedItems; ++j) {
        const u64 r = first + j;
        const bool head = r < n && (r == 0 || key[j] != (j ? key[j - 1] : prev));
        heads |= (u32)head << j;
    }
    const u32 hc = __popc(heads);
    // exclusive scan of the head counts over the block
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u32 inc = hc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const u32 t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= (u32)o) inc += t;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    u32 wp = 0, total = 0;
#pragma unroll
    for (int w = 0; w < kRedThreads / 32; ++w) {
        const u32 x = s_warp[w];
        if (w < (int)warp) wp += x;
        total += x;
    }
    const u32 hoff = inc - hc + wp;
    if (threadIdx.x == 0) {
        u64* mine = status + tile;
        st_volatile_u64(mine, (tile == 0 ? kRedInclusive : kRedPartial) | total);
        u64 excl = 0;
        for (i64 t = (i64)tile - 1; t >= 0;) {
            const u64 w = ld_volatile_u64(status + t);
            const u64 f = w >> 62;
            if (f == 0) continue;  // not published yet
            excl += w & kRedMask;
            if (f == 2) break;
            --t;
        }
        if (tile > 0) st_volatile_u64(mine, kRedInclusive | ((excl + total) & kRedMask));
        s_base = excl;
        if ((tile + 1) * kRedTile >= n) *group_count = excl + total;  // the last tile knows the number of groups
    }
    __syncthreads();
    if (first >= n) return;
    // group of the run that is open when the thread starts: (groups before the thread) - 1
    u64 g = s_base + hoff;  // == index of the NEXT group to open
    u64 sum = 0;
    unsigned long long cnt = 0;
    bool overflow = false;
    auto flush = [&](u64 group) {
        if (cnt == 0) return;
        if (group >= capacity) {
            overflow = true;
        } else {
            if (DBL) atomicAdd(reinterpret_cast<double*>(out_sums + group), __longlong_as_double((long long)sum));
            else atomicAdd(reinterpret_cast<unsigned long long*>(out_sums + group), (unsigned long long)sum);
            atomicAdd(out_counts + group, cnt);
        }
        sum = 0;
        cnt = 0;
    };
#pragma unroll
    for (int j = 0; j < kRedItems; ++j) {
        if (first + j >= n) break;
        if (heads >> j & 1) {
            flush(g - 1);
            if (g < capacity) out_keys[g] = key[j];
            else overflow = true;
            ++g;
        }
        if (DBL) sum = (u64)__double_as_longlong(__longlong_as_double((long long)sum) + __longlong_as_double((long long)val[j]));
        else sum += val[j];
        ++cnt;
    }
    flush(g - 1);
    if (overflow) atomicOr(err_word, (u32)DE_TABLE_FULL);
}

Status reduce_impl(Context* ctx, const ytgpu_fixed_rows_view* in, u32 key_off, u32 val_off, u8 vtype, u64* out_keys, u64* out_sums,
                   u64* out_counts, u64 capacity, u64* out_group_count) {
    if (!in || !out_keys || !out_sums || !out_counts || !out_group_count) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    if (in->mem != YTGPU_MEM_DEVICE) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "the sorted reduce reads device-resident rows");
    const void* words[] = {in->rows, out_keys, out_sums, out_counts};
    for (const void* w : words)
        if (reinterpret_cast<uintptr_t>(w) % 8) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "rows and outputs must be 8-byte aligned");
    const u32 rb = in->row_bytes;
    if (rb == 0 || rb % 8 || key_off % 8 || val_off % 8 || (u64)key_off + 8 > rb || (u64)val_off + 8 > rb)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key/value offsets must be 8-byte aligned and inside the row");
    if (vtype != YTGPU_TYPE_INT64 && vtype != YTGPU_TYPE_UINT64 && vtype != YTGPU_TYPE_DOUBLE)
        return make_status(YTGPU_ERR_UNSUPPORTED, "SUM supports int64/uint64/double value columns");
    *out_group_count = 0;
    const u64 n = in->row_count;
    if (n == 0) return Status{};
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    const u64 tiles = (n + kRedTile - 1) / kRedTile;
    DevBuf<u64> status, gcount;
    DevBuf<u32> counter;
    YTGPU_TRY(status.allocate(ctx, tiles));
    YTGPU_TRY(gcount.allocate(ctx, 1));
    YTGPU_TRY(counter.allocate(ctx, 1));
    YTGPU_CUDA_TRY(cudaMemsetAsync(status.p, 0, tiles * 8, ctx->stream));
    YTGPU_CUDA_TRY(cudaMemsetAsync(counter.p, 0, 4, ctx->stream));
    const u64 zero = std::min<u64>(capacity, n);
    YTGPU_CUDA_TRY(cudaMemsetAsync(out_sums, 0, zero * 8, ctx->stream));
    YTGPU_CUDA_TRY(cudaMemsetAsync(out_counts, 0, zero * 8, ctx->stream));
    {
        KernelTimer t(ctx, KC_REDUCE);
        if (vtype == YTGPU_TYPE_DOUBLE)
            reduce_sorted_kernel<true><<<(u32)tiles, kRedThreads, 0, ctx->stream>>>(in->rows, n, rb, key_off, val_off, status.p, counter.p, out_keys,
                                                                                   out_sums, reinterpret_cast<unsigned long long*>(out_counts),
                                                                                   capacity, gcount.p, ctx->dev_err);
        else
            reduce_sorted_kernel<false><<<(u32)tiles, kRedThreads, 0, ctx->stream>>>(in->rows, n, rb, key_off, val_off, status.p, counter.p, out_keys,
                                                                                    out_sums, reinterpret_cast<unsigned long long*>(out_counts),
                                                                                    capacity, gcount.p, ctx->dev_err);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_CUDA_TRY(cudaMemcpyAsync(out_group_count, gcount.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
    Status s = check_device_errors(ctx);  // synchronises the stream
    if (!s.ok() && *out_group_count > capacity)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "result has %llu groups, capacity is %llu", (unsigned long long)*out_group_count,
                           (unsigned long long)capacity);
    return s;
}

}  // namespace

extern "C" {

int ytgpu_reduce_sorted_fixed_rows(ytgpu_context* h, const ytgpu_fixed_rows_view* in, uint32_t key_offset, uint32_t value_offset,
                                   uint8_t value_type, uint64_t* out_keys, uint64_t* out_sums, uint64_t* out_counts, uint64_t capacity,
                                   uint64_t* out_group_count, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, reduce_impl(as_context(h), in, key_offset, value_offset, value_type, out_keys, out_sums, out_counts, capacity,
                                       out_group_count));
}

}  // extern "C"
