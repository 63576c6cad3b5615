// plain_column_writer.cu — the unversioned floating-point and boolean column writers: segments without any search for a
// layout, so one pass writes every output word.
//   TUnversionedFloatingPointColumnWriter<double>::DumpSegment  yt/yt/ytlib/table_chunk_format/floating_point_column_writer.cpp:213-240
//       data parts: SerializeFloatingPointVector (:21-31) = ui64 count | count raw doubles,  then the null bitmap
//   TUnversionedBooleanColumnWriter::DumpSegment                 boolean_column_writer.cpp:196-216, DumpBooleanValues :18-28
//       data parts: ui64 value count | value bitmap | null bitmap
// Bitmaps are TBitmapOutput: bit i of byte i/8, padded to whole 64-bit words (bitmap.h:131-200).  A NULL row stores the
// payload of a Null TUnversionedValue (zero) / a false bit, as AddValues does (:247-256, :228-238).
// One thread per OUTPUT word of the column: no atomics, no zero fill; bitmap words gather 64 bytemap bytes.
#include "common.cuh"
#include "context.cuh"

using namespace ytgpu;

namespace {

struct PlainLayout {
    u64 n;            // rows
    u64 seg_rows;     // rows per segment (the last one may be shorter)
    u64 seg_words;    // output words of a full segment
    u32 nseg;
    u32 is_boolean;
};

__host__ __device__ inline u64 bitmap_words(u64 rows) { return (rows + 63) / 64; }
__host__ __device__ inline u64 plain_segment_words(u64 rows, bool boolean) {
    return boolean ? 1 + 2 * bitmap_words(rows) : 1 + rows + bitmap_words(rows);
}

// 64 bytemap bytes -> one bitmap word (byte != 0 -> bit set); rows beyond `rows` read as 0.
__device__ __forceinline__ u64 pack_bytemap_word(const u8* __restrict__ bytemap, u64 first, u64 end) {
    u64 w = 0;
    if (!bytemap) return 0;
    if (first + 64 <= end && ((reinterpret_cast<uintptr_t>(bytemap) + first) & 7) == 0) {
        const u64* p = reinterpret_cast<const u64*>(bytemap + first);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            u64 x = p[k];
            // collapse each byte to its "non-zero" bit, then gather the 8 bits
            x |= x >> 4;
            x |= x >> 2;
            x |= x >> 1;
            x &= 0x0101010101010101ull;
            w |= ((x * 0x0102040810204080ull) >> 56) << (8 * k);
        }
        return w;
    }
    for (u64 i = first; i < end && i < first + 64; ++i)
        if (bytemap[i]) w |= 1ull << (i - first);
    return w;
}

__global__ void __launch_bounds__(256) plain_pack_kernel(const PlainLayout L, const u64* __restrict__ values, const u8* __restrict__ bools,
                                                         const u8* __restrict__ nulls, u64 total_words, u64* __restrict__ out) {
    for (u64 w = (u64)blockIdx.x * blockDim.x + threadIdx.x; w < total_words; w += (u64)gridDim.x * blockDim.x) {
        // 64-bit division costs ~100 instructions per word of a kernel that only copies: 32-bit when the column allows it
        const u64 seg = total_words <= 0xffffffffull ? (u64)((u32)w / (u32)L.seg_words) : w / L.seg_words;
        const u64 local = w - seg * L.seg_words;
        const u64 row0 = seg * L.seg_rows;
        const u64 rows = min(L.seg_rows, L.n - row0);
        const u64 bw = bitmap_words(rows);
        u64 v;
        if (local == 0) {
            v = rows;
        } else if (L.is_boolean) {
            const u64 k = local - 1;
            if (k < bw) {  // value bitmap: false for NULL rows
                u64 bits = pack_bytemap_word(bools, row0 + k * 64, row0 + rows);
                if (nulls) bits &= ~pack_bytemap_word(nulls, row0 + k * 64, row0 + rows);
                v = bits;
            } else {
                v = pack_bytemap_word(nulls, row0 + (k - bw) * 64, row0 + rows);
            }
        } else {
            const u64 k = local - 1;
            if (k < rows) v = (nulls && nulls[row0 + k]) ? 0 : values[row0 + k];
            else v = pack_bytemap_word(nulls, row0 + (k - rows) * 64, row0 + rows);
        }
        out[w] = v;
    }
}

Status encode_plain_impl(Context* ctx, bool boolean, const void* values, const u8* null_bytemap, u64 n, u32 max_values, u64 chunk_row_offset,
                         int mem, u8* out_data, u64 out_capacity, u64* out_bytes, ytgpu_plain_segment* out_segments, u32 seg_capacity,
                         u32* out_seg_count) {
    if (!out_bytes || !out_seg_count) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    *out_bytes = 0;
    *out_seg_count = 0;
    if (n == 0) return Status{};
    if (!values) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null values");
    if (max_values == 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "max_segment_value_count must be positive");
    const u64 nseg64 = (n + max_values - 1) / max_values;
    if (nseg64 > 0xffffffffull) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "too many segments");
    const u32 nseg = (u32)nseg64;
    PlainLayout L{n, std::min<u64>(max_values, n), 0, nseg, boolean ? 1u : 0u};
    L.seg_words = plain_segment_words(L.seg_rows, boolean);
    const u64 last_rows = n - (u64)(nseg - 1) * L.seg_rows;
    const u64 total_words = (u64)(nseg - 1) * L.seg_words + plain_segment_words(last_rows, boolean);
    const u64 bytes = total_words * 8;
    *out_bytes = bytes;
    *out_seg_count = nseg;
    if (!out_segments || nseg > seg_capacity)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "column needs %u segment descriptors, capacity is %u", nseg, seg_capacity);
    if (!out_data || bytes > out_capacity)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "column data needs %llu bytes, capacity is %llu", (unsigned long long)bytes,
                           (unsigned long long)out_capacity);
    for (u32 s = 0; s < nseg; ++s) {
        const u64 rows = s + 1 < nseg ? L.seg_rows : last_rows;
        ytgpu_plain_segment& d = out_segments[s];
        d = ytgpu_plain_segment{};
        d.row_count = (u32)rows;
        d.chunk_row_count = chunk_row_offset + (u64)s * L.seg_rows + rows;
        d.data_offset = (u64)s * L.seg_words * 8;
        d.data_bytes = plain_segment_words(rows, boolean) * 8;
        if (boolean) {
            d.part_bytes[0] = 8;
            d.part_bytes[1] = bitmap_words(rows) * 8;
            d.part_bytes[2] = bitmap_words(rows) * 8;
        } else {
            d.part_bytes[0] = 8 + rows * 8;
            d.part_bytes[1] = bitmap_words(rows) * 8;
            d.part_bytes[2] = 0;
        }
    }
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    InBuf<u8> dv, dn;
    YTGPU_TRY(dv.stage(ctx, static_cast<const u8*>(values), boolean ? n : n * 8, mem));
    YTGPU_TRY(dn.stage(ctx, null_bytemap, n, mem));
    if (mem != YTGPU_MEM_HOST && (reinterpret_cast<uintptr_t>(out_data) & 7))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "out_data must be 8-byte aligned");
    OutBuf<u64> dst;
    YTGPU_TRY(dst.prepare(ctx, reinterpret_cast<u64*>(out_data), total_words, mem));
    {
        KernelTimer t(ctx, KC_DECODE, 1);
        const u32 grid = (u32)std::max<u64>(1, std::min<u64>((total_words + 255) / 256, (u64)kNumSms * 8));
        plain_pack_kernel<<<grid, 256, 0, ctx->stream>>>(L, boolean ? nullptr : reinterpret_cast<const u64*>(dv.p),
                                                        boolean ? dv.p : nullptr, dn.p, total_words, dst.p);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_TRY(dst.download(ctx, total_words));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return Status{};
}

// ---- rows -> one flat column (the AddValues loops of the column converters / writers) ----
// payload: Double -> bit pattern, Boolean -> 0 / 1, Int64 / Uint64 -> the value, String -> heap offset (+ length);
// a Null value gives a zero payload / length and null_bytemap 1; any other type than `value_type` is a schema violation.
__global__ void __launch_bounds__(256) extract_column_kernel(const ytgpu_value* __restrict__ values, u64 nrows, u32 value_count, u32 column,
                                                             u8 value_type, u64* __restrict__ out_payload, u32* __restrict__ out_lengths,
                                                             u8* __restrict__ out_null, u32* __restrict__ dev_err) {
    for (u64 r = (u64)blockIdx.x * blockDim.x + threadIdx.x; r < nrows; r += (u64)gridDim.x * blockDim.x) {
        const uint4 raw = *reinterpret_cast<const uint4*>(values + r * value_count + column);
        const u8 type = (u8)((raw.x >> 16) & 0xff);
        const u32 length = raw.y;
        u64 data = ((u64)raw.w << 32) | raw.z;
        bool nl = type == YTGPU_TYPE_NULL;
        if (!nl && type != value_type) {
            atomicOr(dev_err, (u32)DE_SCHEMA_VIOLATION);
            nl = true;
        }
        if (value_type == YTGPU_TYPE_BOOLEAN) data = (data & 0xff) != 0;
        out_payload[r] = nl ? 0 : data;
        if (out_lengths) out_lengths[r] = nl ? 0 : length;
        if (out_null) out_null[r] = nl ? 1 : 0;
    }
}

Status extract_column_impl(Context* ctx, const ytgpu_rowset_view* rows, u32 column, u8 value_type, u64* out_payload, u32* out_lengths,
                           u8* out_null, int out_mem) {
    if (!rows || !out_payload) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    if (column >= rows->value_count) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "column index out of range");
    const bool is_string = value_type == YTGPU_TYPE_STRING || value_type == YTGPU_TYPE_ANY || value_type == YTGPU_TYPE_COMPOSITE;
    if (!is_string && value_type != YTGPU_TYPE_INT64 && value_type != YTGPU_TYPE_UINT64 && value_type != YTGPU_TYPE_DOUBLE &&
        value_type != YTGPU_TYPE_BOOLEAN)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "unknown value type 0x%x", value_type);
    if (is_string && !out_lengths) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string columns need out_lengths");
    const u64 n = rows->row_count;
    if (n == 0) return Status{};
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    InBuf<ytgpu_value> vals;
    OutBuf<u64> dp;
    OutBuf<u32> dl;
    OutBuf<u8> dn;
    YTGPU_TRY(vals.stage(ctx, rows->values, n * rows->value_count, rows->mem));
    YTGPU_TRY(dp.prepare(ctx, out_payload, n, out_mem));
    YTGPU_TRY(dl.prepare(ctx, out_lengths, n, out_mem));
    YTGPU_TRY(dn.prepare(ctx, out_null, n, out_mem));
    {
        KernelTimer t(ctx, KC_DECODE, 1);
        const u32 grid = (u32)std::max<u64>(1, std::min<u64>((n + 255) / 256, (u64)kNumSms * 8));
        extract_column_kernel<<<grid, 256, 0, ctx->stream>>>(vals.p, n, rows->value_count, column, value_type, dp.p, dl.p, dn.p,
                                                             ctx->dev_err);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_TRY(dp.download(ctx, n));
    YTGPU_TRY(dl.download(ctx, n));
    YTGPU_TRY(dn.download(ctx, n));
    return check_device_errors(ctx);
}

}  // namespace

extern "C" {

int ytgpu_extract_column(ytgpu_context* h, const ytgpu_rowset_view* rows, uint32_t column_index, uint8_t value_type, uint64_t* out_payload,
                         uint32_t* out_lengths, uint8_t* out_null_bytemap, int out_mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, extract_column_impl(as_context(h), rows, column_index, value_type, out_payload, out_lengths, out_null_bytemap, out_mem));
}

int ytgpu_encode_double_column(ytgpu_context* h, const uint64_t* values, const uint8_t* null_bytemap, uint64_t row_count,
                               uint32_t max_segment_value_count, uint64_t chunk_row_offset, int mem, uint8_t* out_data,
                               uint64_t out_capacity, uint64_t* out_data_bytes, ytgpu_plain_segment* out_segments,
                               uint32_t segment_capacity, uint32_t* out_segment_count, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, encode_plain_impl(as_context(h), false, values, null_bytemap, row_count, max_segment_value_count,
                                             chunk_row_offset, mem, out_data, out_capacity, out_data_bytes, out_segments,
                                             segment_capacity, out_segment_count));
}

int ytgpu_encode_boolean_column(ytgpu_context* h, const uint8_t* values, const uint8_t* null_bytemap, uint64_t row_count,
                                uint32_t max_segment_value_count, uint64_t chunk_row_offset, int mem, uint8_t* out_data,
                                uint64_t out_capacity, uint64_t* out_data_bytes, ytgpu_plain_segment* out_segments,
                                uint32_t segment_capacity, uint32_t* out_segment_count, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, encode_plain_impl(as_context(h), true, values, null_bytemap, row_count, max_segment_value_count,
                                             chunk_row_offset, mem, out_data, out_capacity, out_data_bytes, out_segments,
                                             segment_capacity, out_segment_count));
}

}  // extern "C"
