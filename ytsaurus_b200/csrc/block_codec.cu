// block_codec.cu — horizontal (schemaless) block codec on the device.
//
// The intermediate-chunk wire format on both sides of the partition and sort jobs:
//   writer  THorizontalBlockWriter::WriteRow / FlushBlock   yt/yt/ytlib/table_client/schemaless_block_writer.cpp:40-86
//           WriteRowValue                                    yt/yt/client/table_client/unversioned_row.cpp:159-206
//   reader  THorizontalBlockReader::JumpToRowIndex / GetRow  yt/yt/ytlib/table_client/schemaless_block_reader.cpp:187-246,323-349
//           ReadRowValue                                     unversioned_row.cpp:208-280
//   varints library/cpp/yt/coding/varint-inl.h (LEB128), zig_zag-inl.h
// block = ui32 offsets[row_count] ++ row data; row = varuint32 value_count, then per value varuint32 id,
// varuint32 type and the payload (Int64 zig-zag varint, Uint64 varint, Double 8 raw bytes, Boolean 1 byte,
// String/Any varuint32 length + bytes; Composite is written as Any).
// Decode: one thread per row (rows are independent thanks to the offset table); strings are NOT copied, the
// decoded value's `data` is the byte offset of the payload inside the block.  Encode: per-row sizes ->
// exclusive scan -> one thread per row writes its bytes and its offset.
#include <vector>

#include "context.cuh"
#include "scan.cuh"

using namespace ytgpu;

namespace {

constexpr u32 DE_BAD_BLOCK_LOCAL = 1u << 8;

__device__ __forceinline__ u32 varuint_size(u64 v) {
    u32 n = 1;
    while (v >= 0x80) { v >>= 7; ++n; }
    return n;
}
__device__ __forceinline__ u8* put_varuint(u8* p, u64 v) {
    while (v >= 0x80) { *p++ = (u8)(v | 0x80); v >>= 7; }
    *p++ = (u8)v;
    return p;
}
// returns bytes consumed, 0 on malformed input
__device__ __forceinline__ u32 get_varuint(const u8* p, const u8* end, u64* out) {
    u64 r = 0;
    u32 n = 0;
    int shift = 0;
    while (p + n < end) {
        const u8 b = p[n++];
        r |= (u64)(b & 0x7f) << shift;
        if (!(b & 0x80)) { *out = r; return n; }
        shift += 7;
        if (shift > 63) return 0;
    }
    return 0;
}
__device__ __forceinline__ u64 zigzag_enc(i64 n) { return ((u64)n << 1) ^ (u64)(n >> 63); }
__device__ __forceinline__ u64 zigzag_dec(u64 n) { return (n >> 1) ^ (0 - (n & 1)); }

__device__ __forceinline__ void store_value(ytgpu_value* dst, u16 id, u8 type, u32 length, u64 data) {
    uint4 raw;
    raw.x = (u32)id | ((u32)type << 16);
    raw.y = length;
    raw.z = (u32)data;
    raw.w = (u32)(data >> 32);
    *reinterpret_cast<uint4*>(dst) = raw;
}

__global__ void __launch_bounds__(256) decode_block_kernel(const u8* __restrict__ block, u64 block_bytes, u32 nrows,
                                                           u32 value_count, ytgpu_value* __restrict__ out,
                                                           u32* __restrict__ out_counts, u32* err_word) {
    const u8* data = block + (u64)nrows * 4;
    const u8* end = block + block_bytes;
    u32 err = 0;
    for (u32 r = blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += gridDim.x * blockDim.x) {
        const u32 off = reinterpret_cast<const u32*>(block)[r];
        const u8* p = data + off;
        ytgpu_value* row = out + (u64)r * value_count;
        u64 cnt = 0;
        u32 n = p < end ? get_varuint(p, end, &cnt) : 0;
        bool bad = n == 0;
        p += n;
        if (out_counts) out_counts[r] = bad ? 0u : (u32)cnt;
        for (u32 c = 0; c < value_count; ++c) {
            if (bad || c >= cnt) {
                store_value(row + c, 0xffff, YTGPU_TYPE_NULL, 0, 0);
                continue;
            }
            u64 id = 0, type = 0, payload = 0;
            u32 length = 0;
            if (!(n = get_varuint(p, end, &id))) { bad = true; --c; continue; }
            p += n;
            if (!(n = get_varuint(p, end, &type)) || type > 0xff) { bad = true; --c; continue; }
            p += n;
            switch ((u8)type) {
                case YTGPU_TYPE_INT64:
                    if (!(n = get_varuint(p, end, &payload))) bad = true;
                    p += n;
                    payload = zigzag_dec(payload);
                    break;
                case YTGPU_TYPE_UINT64:
                    if (!(n = get_varuint(p, end, &payload))) bad = true;
                    p += n;
                    break;
                case YTGPU_TYPE_DOUBLE:
                    if (p + 8 > end) { bad = true; break; }
                    for (int i = 7; i >= 0; --i) payload = (payload << 8) | p[i];
                    p += 8;
                    break;
                case YTGPU_TYPE_BOOLEAN:
                    if (p + 1 > end) { bad = true; break; }
                    payload = *p == 1;
                    p += 1;
                    break;
                case YTGPU_TYPE_STRING:
                case YTGPU_TYPE_ANY:
                case YTGPU_TYPE_COMPOSITE: {
                    // a varuint32 length; compared with the bytes left, as p + n + len wraps for a length near 2^64
                    u64 len = 0;
                    if (!(n = get_varuint(p, end, &len)) || len >= (1ull << 32) || len > (u64)(end - p - n)) { bad = true; break; }
                    p += n;
                    length = (u32)len;
                    payload = (u64)(p - block);
                    p += len;
                    break;
                }
                case YTGPU_TYPE_NULL:
                case YTGPU_TYPE_MIN:
                case YTGPU_TYPE_MAX:
                case YTGPU_TYPE_BOTTOM:
                    break;
                default:
                    bad = true;  // ThrowUnexpectedValueType
            }
            if (bad) { --c; continue; }  // re-enter: pads this and the remaining values with Null
            store_value(row + c, (u16)id, (u8)type, length, payload);
        }
        if (bad) err |= DE_BAD_BLOCK_LOCAL;
    }
    if (err) atomicOr(err_word, err);
}

__device__ __forceinline__ ytgpu_value load_val(const ytgpu_value* p) {
    uint4 raw = *reinterpret_cast<const uint4*>(p);
    ytgpu_value v;
    v.id = (u16)(raw.x & 0xffff);
    v.type = (u8)((raw.x >> 16) & 0xff);
    v.flags = (u8)(raw.x >> 24);
    v.length = raw.y;
    v.data = ((u64)raw.w << 32) | raw.z;
    return v;
}

__device__ __forceinline__ u32 value_encoded_size(const ytgpu_value& v) {
    const u8 type = v.type == YTGPU_TYPE_COMPOSITE ? (u8)YTGPU_TYPE_ANY : v.type;
    u32 s = varuint_size(v.id) + varuint_size(type);
    switch (type) {
        case YTGPU_TYPE_INT64: s += varuint_size(zigzag_enc((i64)v.data)); break;
        case YTGPU_TYPE_UINT64: s += varuint_size(v.data); break;
        case YTGPU_TYPE_DOUBLE: s += 8; break;
        case YTGPU_TYPE_BOOLEAN: s += 1; break;
        case YTGPU_TYPE_STRING:
        case YTGPU_TYPE_ANY: s += varuint_size(v.length) + v.length; break;
        default: break;
    }
    return s;
}

__global__ void __launch_bounds__(256) row_sizes_kernel(const ytgpu_value* __restrict__ values, u32 value_count,
                                                        const u32* __restrict__ row_counts, u64 nrows,
                                                        u64* __restrict__ sizes) {
    for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (u64)gridDim.x * blockDim.x) {
        const u32 cnt = row_counts ? min(row_counts[r], value_count) : value_count;
        u32 s = varuint_size(cnt);
        for (u32 c = 0; c < cnt; ++c) s += value_encoded_size(load_val(values + r * value_count + c));
        sizes[r] = s;
    }
}

// exclusive scan of u64: scan.cuh

__global__ void __launch_bounds__(256) encode_rows_kernel(const ytgpu_value* __restrict__ values, u32 value_count,
                                                          const u32* __restrict__ row_counts, const u8* __restrict__ heap,
                                                          u64 nrows, const u64* __restrict__ row_offsets, u8* __restrict__ block) {
    u8* data = block + nrows * 4;
    for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (u64)gridDim.x * blockDim.x) {
        const u64 off = row_offsets[r];
        reinterpret_cast<u32*>(block)[r] = (u32)off;
        u8* p = data + off;
        const u32 cnt = row_counts ? min(row_counts[r], value_count) : value_count;
        p = put_varuint(p, cnt);
        for (u32 c = 0; c < cnt; ++c) {
            const ytgpu_value v = load_val(values + r * value_count + c);
            const u8 type = v.type == YTGPU_TYPE_COMPOSITE ? (u8)YTGPU_TYPE_ANY : v.type;
            p = put_varuint(p, v.id);
            p = put_varuint(p, type);
            switch (type) {
                case YTGPU_TYPE_INT64: p = put_varuint(p, zigzag_enc((i64)v.data)); break;
                case YTGPU_TYPE_UINT64: p = put_varuint(p, v.data); break;
                case YTGPU_TYPE_DOUBLE:
                    for (int i = 0; i < 8; ++i) *p++ = (u8)(v.data >> (8 * i));
                    break;
                case YTGPU_TYPE_BOOLEAN: *p++ = (v.data & 0xff) ? 1 : 0; break;
                case YTGPU_TYPE_STRING:
                case YTGPU_TYPE_ANY: {
                    p = put_varuint(p, v.length);
                    const u8* s = heap + v.data;
                    for (u32 i = 0; i < v.length; ++i) p[i] = s[i];
                    p += v.length;
                    break;
                }
                default: break;
            }
        }
    }
}

inline u32 blocks_for(u64 items, int threads, int per_sm) {
    return (u32)std::max<u64>(1, std::min<u64>((items + threads - 1) / threads, (u64)kNumSms * per_sm));
}

Status decode_impl(Context* ctx, const u8* block, u64 block_bytes, u32 nrows, u32 value_count, ytgpu_value* out,
                   u32* out_counts, int mem) {
    if (!block || !out || value_count == 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument or value_count == 0");
    if ((u64)nrows * 4 > block_bytes) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "block shorter than its offset table");
    if (nrows == 0) return Status{};
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    InBuf<u8> b;
    OutBuf<ytgpu_value> o;
    OutBuf<u32> c;
    YTGPU_TRY(b.stage(ctx, block, block_bytes, mem));
    YTGPU_TRY(o.prepare(ctx, out, (size_t)nrows * value_count, mem));
    YTGPU_TRY(c.prepare(ctx, out_counts, nrows, mem));
    {
        KernelTimer t(ctx, KC_DECODE);
        decode_block_kernel<<<blocks_for(nrows, 256, 8), 256, 0, ctx->stream>>>(b.p, block_bytes, nrows, value_count, o.p, c.p, ctx->dev_err);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_TRY(o.download(ctx, (size_t)nrows * value_count));
    YTGPU_TRY(c.download(ctx, nrows));
    // malformed input is reported like ReadRowValue's ThrowUnexpectedValueType
    YTGPU_CUDA_TRY(cudaMemcpyAsync(ctx->host_err, ctx->dev_err, 4, cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_CUDA_TRY(cudaMemsetAsync(ctx->dev_err, 0, 4, ctx->stream));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (*ctx->host_err & DE_BAD_BLOCK_LOCAL) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "malformed horizontal block (bad varint, value type or offset)");
    return Status{};
}

Status encode_impl(Context* ctx, const ytgpu_rowset_view* rows, const u32* row_counts, u8* out_block, u64 capacity,
                   u64* out_bytes, int out_mem) {
    if (!rows || !out_bytes) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    const u64 n = rows->row_count;
    const u32 vc = rows->value_count;
    *out_bytes = 0;
    if (n == 0) return Status{};
    if (n >= (1ull << 32)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "a block holds fewer than 2^32 rows");
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    StagedRowset staged;
    InBuf<u32> counts;
    YTGPU_TRY(staged.stage(ctx, rows, rows->mem));
    YTGPU_TRY(counts.stage(ctx, row_counts, n, rows->mem));
    OutBuf<u8> dst;
    DevBuf<u64> sizes, sums, total;
    const u64 nblocks = (n + kScanBlock - 1) / kScanBlock;
    YTGPU_TRY(sizes.allocate(ctx, n));
    YTGPU_TRY(sums.allocate(ctx, nblocks));
    YTGPU_TRY(total.allocate(ctx, 1));
    KernelTimer t(ctx, KC_DECODE, 5);
    row_sizes_kernel<<<blocks_for(n, 256, 8), 256, 0, ctx->stream>>>(staged.values.p, vc, counts.p, n, sizes.p);
    exclusive_scan_u64(ctx->stream, sizes.p, n, sums.p, total.p);
    YTGPU_CUDA_TRY(cudaGetLastError());
    u64 data_bytes = 0;
    YTGPU_CUDA_TRY(cudaMemcpyAsync(&data_bytes, total.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    const u64 bytes = n * 4 + data_bytes;
    *out_bytes = bytes;
    if (data_bytes >= (1ull << 32)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "block data of %llu bytes does not fit ui32 row offsets", (unsigned long long)data_bytes);
    if (!out_block || bytes > capacity)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "block needs %llu bytes, capacity is %llu", (unsigned long long)bytes, (unsigned long long)capacity);
    YTGPU_TRY(dst.prepare(ctx, out_block, bytes, out_mem));
    encode_rows_kernel<<<blocks_for(n, 256, 8), 256, 0, ctx->stream>>>(staged.values.p, vc, counts.p, staged.heap.p, n, sizes.p, dst.p);
    YTGPU_CUDA_TRY(cudaGetLastError());
    YTGPU_TRY(dst.download(ctx, bytes));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return Status{};
}

}  // namespace

extern "C" {

int ytgpu_decode_horizontal_block(ytgpu_context* h, const uint8_t* block, uint64_t block_bytes, uint32_t row_count,
                                  uint32_t value_count, ytgpu_value* out_values, uint32_t* out_row_value_counts, int mem,
                                  ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, decode_impl(as_context(h), block, block_bytes, row_count, value_count, out_values, out_row_value_counts, mem));
}

int ytgpu_encode_horizontal_block(ytgpu_context* h, const ytgpu_rowset_view* rows, const uint32_t* row_value_counts,
                                  uint8_t* out_block, uint64_t out_capacity, uint64_t* out_block_bytes, int out_mem,
                                  ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, encode_impl(as_context(h), rows, row_value_counts, out_block, out_capacity, out_block_bytes, out_mem));
}

}  // extern "C"
