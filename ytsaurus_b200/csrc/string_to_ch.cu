// string_to_ch.cu — YT string column -> ClickHouse ColumnString: ConvertStringLikeYTColumnToCHColumn
// (yt/chyt/server/columnar_conversion.cpp:429-648), the string path of the CHYT scan.
//
// The reference appends value after value (memcpy + '\0', growing the buffer when it guessed too small).  Here:
//   1. string_ranges_kernel: every row resolves its string through the RLE runs / dictionary indexes (one run search per
//      WARP, the lanes walk from there) and decodes its byte range (DecodeStringRange); it writes the source start (u32)
//      and length + 1 (u64, the scan input); rows that are null or rejected by the filter hint are empty strings;
//   2. exclusive scan of the sizes (scan.cuh): the position of every value in the output, the total = chars size;
//      out_offsets[i] = position of value i + 1 (ColumnString offsets are END offsets);
//   3. copy_chars_kernel: row centric — a warp takes 32 consecutive values per trip; short values are copied by their own
//      lane (the lanes write one contiguous stretch of the output), longer ones by the whole warp.
// Algorithmic bytes per row: 4 (offset) [+ 4 dictionary index] + L read, L + 1 + 8 written; scratch 12 B/row.
#include "columnar.cuh"
#include "context.cuh"
#include "scan.cuh"

using namespace ytgpu;

namespace {

struct StringColumnDev {
    const u32* offsets;
    u64 string_count;
    u32 avg;
    const u8* chars;
    u64 chars_bytes;
    const u32* dict;
    u64 dict_count;
    const u64* rle;
    u64 rle_count;
    u64 start;
    u64 count;
    const u8* filter;
};

__device__ __forceinline__ i64 zigzag32_to_i64(u32 z) { return (i64)(z >> 1) ^ -(i64)(z & 1); }

// DecodeStringRange, columnar-inl.h:31-50 (32-bit arithmetic on avgLength * index, as there)
__device__ __forceinline__ void string_range(const StringColumnDev& c, u64 s, i64* begin, i64* end) {
    if (s == 0) {
        *begin = 0;
        *end = (i64)c.avg + zigzag32_to_i64(__ldg(c.offsets));
        return;
    }
    const u32 base = c.avg * (u32)s;
    *begin = (i64)base + zigzag32_to_i64(__ldg(c.offsets + s - 1));
    *end = (i64)base + (i64)c.avg + zigzag32_to_i64(__ldg(c.offsets + s));
}

__global__ void __launch_bounds__(256) string_ranges_kernel(const StringColumnDev c, u32* __restrict__ src_start, u64* __restrict__ sizes,
                                                            u32* dev_err) {
    // a warp walks a contiguous share of the rows front to back: ONE binary search over the runs per warp, afterwards
    // every search starts from the previous trip's run (a chain of full binary searches per trip made the kernel
    // latency bound: 20 dependent loads x trips, measured on the null bytemap kernels)
    const u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5, warps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u64 per_warp = ((c.count + warps * 32 - 1) / (warps * 32)) * 32;
    const u64 share_begin = min(c.count, warp * per_warp), share_end = min(c.count, share_begin + per_warp);
    u64 hint = kNoRleHint;
    for (u64 base = share_begin; base < share_end; base += 32) {
        if (c.rle) {
            u64 k = 0;
            if (lane_id() == 0)
                k = hint == kNoRleHint ? rle_pos(c.rle, c.rle_count, c.start + base) : rle_pos_gallop(c.rle, c.rle_count, c.start + base, hint);
            hint = __shfl_sync(0xffffffffu, k, 0);
        }
        const u64 i = base + lane_id();
        if (i >= c.count) continue;
        u64 v = c.start + i;  // index into the (possibly run-length encoded) index vector
        if (c.rle) v = rle_pos_gallop(c.rle, c.rle_count, v, hint);
        bool empty = c.filter && c.filter[i] == 0;
        u64 s = v;
        if (c.dict) {
            if (v >= c.dict_count) {
                atomicOr(dev_err, DE_PART_OUT_OF_BOUNDS);
                empty = true;
                s = 0;
            } else {
                const u32 d = __ldg(c.dict + v);
                if (d == 0) empty = true;  // null: `currentValue = {}` (columnar-inl.h:90-92,163-165)
                s = d ? d - 1 : 0;
            }
        }
        i64 b = 0, e = 0;
        if (!empty) {
            if (s >= c.string_count) {
                atomicOr(dev_err, DE_PART_OUT_OF_BOUNDS);
            } else {
                string_range(c, s, &b, &e);
                if (b < 0 || e < b || (u64)e > c.chars_bytes) {
                    atomicOr(dev_err, DE_PART_OUT_OF_BOUNDS);
                    b = e = 0;
                }
            }
        }
        src_start[i] = (u32)b;
        sizes[i] = (u64)(e - b) + 1;
    }
}

// pos[i] = start of value i in the output (exclusive scan of the sizes), *total = chars size.
__global__ void __launch_bounds__(256) end_offsets_kernel(const u64* __restrict__ pos, const u64* __restrict__ total, u64 n,
                                                          u64* __restrict__ out_offsets) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x)
        out_offsets[i] = i + 1 < n ? pos[i + 1] : *total;
}

// Row centric: a warp takes 32 consecutive values per trip.  Short values (<= kShortValue bytes, the norm) are assembled
// by their own lanes in a per-warp shared-memory buffer — the trip's output is one contiguous stretch — and written out
// with 16-byte stores; a longer value is copied by the whole warp, consecutive lanes -> consecutive bytes.  No lookups
// besides pos[i], pos[i + 1] and src_start[i]: the first version was OUTPUT centric (a thread per 16 output bytes finding its
// rows by binary search over the positions) and was bound by the chain of dependent search loads, 1.2 ms for 2*10^7
// values / 240 MB, i.e. 0.4 TB/s.
constexpr u32 kShortValue = 48;

__global__ void __launch_bounds__(256) copy_chars_kernel(const u8* __restrict__ chars, const u32* __restrict__ src_start,
                                                         const u64* __restrict__ pos, const u64* __restrict__ total_ptr, u64 n,
                                                         u8* __restrict__ out) {
    __shared__ __align__(16) u8 s_stage[8][32 * (kShortValue + 1) + 32];  // one staging buffer per warp (256 threads)
    const u64 total = *total_ptr;
    const u32 lane = lane_id();
    for (u64 base = ((u64)blockIdx.x * blockDim.x + threadIdx.x) & ~31ull; base < n; base += (u64)gridDim.x * blockDim.x) {
        const u64 i = base + lane;
        const bool valid = i < n;
        u64 p = 0, len = 0;
        const u8* src = chars;
        if (valid) {
            p = __ldg(pos + i);
            len = (i + 1 < n ? __ldg(pos + i + 1) : total) - p - 1;
            src = chars + __ldg(src_start + i);
        }
        const bool is_long = valid && len > kShortValue;
        u32 todo = __ballot_sync(0xffffffffu, is_long);
        if (todo == 0) {
            // Every value of the trip is short: the trip's output [p0, p1) is one contiguous stretch of at most 32 * 49 bytes.
            // The lanes assemble it in the warp's shared buffer (byte stores into shared memory are cheap; into global memory
            // one warp instruction touched ~13 sectors) and the warp writes it out with 16-byte stores.  The buffer starts at
            // the 16-byte boundary below out + p0, so buffer word w is global word w of that boundary.
            u8* buf = s_stage[threadIdx.x >> 5];
            const u64 p0 = __shfl_sync(0xffffffffu, p, 0);  // lane 0 is always valid
            const u64 last_end = valid ? p + len + 1 : 0;
            u64 p1 = last_end;
#pragma unroll
            for (int d = 16; d > 0; d >>= 1) p1 = max(p1, __shfl_xor_sync(0xffffffffu, p1, d));
            const u32 skew = (u32)(reinterpret_cast<uintptr_t>(out + p0) & 15);
            if (valid) {
                u8* dst = buf + skew + (u32)(p - p0);
                for (u32 j = 0; j < (u32)len; ++j) dst[j] = __ldg(src + j);
                dst[len] = 0;
            }
            __syncwarp();
            const u32 begin = skew, end = skew + (u32)(p1 - p0);  // valid bytes of the buffer
            u8* gbase = out + p0 - skew;                          // 16-byte aligned
            for (u32 w = lane; w * 16 < end; w += 32) {
                const u32 lo = w * 16, hi = lo + 16;
                if (lo >= begin && hi <= end) {
                    reinterpret_cast<uint4*>(gbase)[w] = reinterpret_cast<const uint4*>(buf)[w];
                } else {
                    for (u32 b = max(lo, begin); b < min(hi, end); ++b) gbase[b] = buf[b];
                }
            }
            __syncwarp();  // the buffer is reused by the next trip
            continue;
        }
        if (valid && !is_long) {
            for (u32 j = 0; j < (u32)len; ++j) out[p + j] = __ldg(src + j);
            out[p + len] = 0;
        }
        while (todo) {
            const int l = __ffs(todo) - 1;
            todo &= todo - 1;
            const u64 lp = __shfl_sync(0xffffffffu, p, l), ll = __shfl_sync(0xffffffffu, len, l);
            const u8* ls = reinterpret_cast<const u8*>(__shfl_sync(0xffffffffu, reinterpret_cast<unsigned long long>(src), l));
            // 4 bytes per lane per step when source and destination are both 4-byte aligned at this step, else 1
            const u32 head = (u32)min(ll, (u64)((4 - (reinterpret_cast<uintptr_t>(out + lp) & 3)) & 3));  // bytes before the destination is word aligned
            for (u64 j = lane; j < head; j += 32) out[lp + j] = __ldg(ls + j);
            const u64 body = (ll - head) & ~3ull;
            if (((reinterpret_cast<uintptr_t>(ls) + head) & 3) == 0) {
                const u32* s4 = reinterpret_cast<const u32*>(ls + head);
                u32* d4 = reinterpret_cast<u32*>(out + lp + head);
                for (u64 w = lane; w < body / 4; w += 32) d4[w] = __ldg(s4 + w);
            } else {
                for (u64 j = lane; j < body; j += 32) out[lp + head + j] = __ldg(ls + head + j);
            }
            for (u64 j = head + body + lane; j < ll; j += 32) out[lp + j] = __ldg(ls + j);
            if (lane == 0) out[lp + ll] = 0;
        }
    }
}

__global__ void check_rle_first_kernel(const u64* __restrict__ rle, u32* dev_err) {
    if (rle[0] != 0) atomicOr(dev_err, DE_SCHEMA_VIOLATION);
}

inline unsigned grid_for(u64 items, unsigned per_block) {
    const u64 blocks = (items + per_block - 1) / per_block;
    return (unsigned)std::max<u64>(1, std::min<u64>(blocks, (u64)kNumSms * 32));
}

Status convert_impl(Context* ctx, const ytgpu_string_column_view* col, const u8* filter_hint, u8* out_chars, u64 out_capacity,
                    u64* out_offsets, u64* out_chars_bytes, int out_mem) {
    if (!col || !out_chars_bytes) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    *out_chars_bytes = 0;
    if (col->start_index < 0 || col->value_count < 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "negative row range");
    const u64 n = (u64)col->value_count;
    if (n == 0) return Status{};  // "We can get empty column" :456-459
    if (!col->offsets || col->string_count == 0 || (!col->chars && col->chars_bytes))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "the value column has no strings");
    if (col->rle_indexes && col->rle_count == 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "empty rle_indexes");
    if (out_chars && !out_offsets) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null out_offsets");
    const u64 index_count = col->rle_indexes ? col->rle_count : (u64)col->start_index + n;  // entries of the index vector touched
    if (col->dictionary_indexes) {
        if (col->dictionary_index_count < index_count) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "row range ends past the dictionary indexes");
    } else if (col->string_count < index_count) {
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "row range ends past the strings");
    }
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));

    StringColumnDev c{};
    c.string_count = col->string_count;
    c.avg = col->avg_length;
    c.chars = col->chars;
    c.chars_bytes = col->chars_bytes;
    c.dict_count = col->dictionary_index_count;
    c.rle_count = col->rle_indexes ? col->rle_count : 0;
    c.start = (u64)col->start_index;
    c.count = n;
    if (col->mem == YTGPU_MEM_HOST) {
        if (col->rle_indexes && col->rle_indexes[0] != 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "rle_indexes[0] != 0");
    } else if (col->rle_indexes) {
        check_rle_first_kernel<<<1, 1, 0, ctx->stream>>>(col->rle_indexes, ctx->dev_err);
        ctx->count_launch();
    }
    InBuf<u32> offsets, dict;
    InBuf<u64> rle;
    InBuf<u8> chars, filter;
    YTGPU_TRY(offsets.stage(ctx, col->offsets, col->string_count, col->mem));
    c.offsets = offsets.p;
    if (out_chars) {  // the size query does not read the bytes
        YTGPU_TRY(chars.stage(ctx, col->chars, col->chars_bytes, col->mem));
        c.chars = chars.p;
    }
    YTGPU_TRY(dict.stage(ctx, col->dictionary_indexes, col->dictionary_index_count, col->mem));
    c.dict = dict.p;
    YTGPU_TRY(rle.stage(ctx, col->rle_indexes, col->rle_count, col->mem));
    c.rle = rle.p;
    YTGPU_TRY(filter.stage(ctx, filter_hint, n, col->mem));
    c.filter = filter.p;

    DevBuf<u32> src_start;
    DevBuf<u64> pos, sums, total;
    YTGPU_TRY(src_start.allocate(ctx, n));
    YTGPU_TRY(pos.allocate(ctx, n));
    YTGPU_TRY(sums.allocate(ctx, scan_block_count(n)));
    YTGPU_TRY(total.allocate(ctx, 1));
    {
        KernelTimer t(ctx, KC_DECODE, 4);
        string_ranges_kernel<<<grid_for(n, 256), 256, 0, ctx->stream>>>(c, src_start.p, pos.p, ctx->dev_err);
        exclusive_scan_u64(ctx->stream, pos.p, n, sums.p, total.p);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    u64 total_host = 0;
    YTGPU_CUDA_TRY(cudaMemcpyAsync(&total_host, total.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
    {
        Status s = check_device_errors(ctx);  // synchronises the stream
        if (!s.ok()) {
            const u32 e = *ctx->host_err;
            if (e & DE_SCHEMA_VIOLATION) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "rle_indexes[0] != 0");
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "malformed string column: an index or a string range is out of bounds");
        }
    }
    *out_chars_bytes = total_host;
    if (!out_chars) return Status{};
    if (out_capacity < total_host)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "out_chars holds %llu bytes, %llu are needed", (unsigned long long)out_capacity,
                           (unsigned long long)total_host);
    OutBuf<u8> oc;
    OutBuf<u64> oo;
    YTGPU_TRY(oc.prepare(ctx, out_chars, total_host, out_mem));
    YTGPU_TRY(oo.prepare(ctx, out_offsets, n, out_mem));
    {
        KernelTimer t(ctx, KC_GATHER, 2);
        end_offsets_kernel<<<grid_for(n, 256), 256, 0, ctx->stream>>>(pos.p, total.p, n, oo.p);
        copy_chars_kernel<<<grid_for(n, 256), 256, 0, ctx->stream>>>(c.chars, src_start.p, pos.p, total.p, n, oc.p);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_TRY(oc.download(ctx, total_host));
    YTGPU_TRY(oo.download(ctx, n));
    if (out_mem == YTGPU_MEM_HOST) YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return Status{};
}

}  // namespace

extern "C" int ytgpu_convert_string_column_to_ch(ytgpu_context* h, const ytgpu_string_column_view* column, const uint8_t* filter_hint,
                                                 uint8_t* out_chars, uint64_t out_chars_capacity, uint64_t* out_offsets,
                                                 uint64_t* out_chars_bytes, int out_mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, convert_impl(as_context(h), column, filter_hint, out_chars, out_chars_capacity, out_offsets, out_chars_bytes, out_mem));
}
