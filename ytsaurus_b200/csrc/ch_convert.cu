// ch_convert.cu — ClickHouse column -> unversioned values: TCHToYTConverter::ConvertColumnToUnversionedValues for simple
// types (yt/chyt/server/ch_to_yt_converter.cpp:131-215 TSimpleValueConverter::FillValueRange, :374-386 TNullableConverter).
//
// One thread per row, one 16-byte store per row: the kernel reads 1-8 bytes (+1 for the null map) and writes 16, so it is
// bound by the value stream it writes.  String values keep pointing into the column's chars (offsets, no copy).
#include "context.cuh"

using namespace ytgpu;

namespace {

struct ChColumnDev {
    int type;
    const void* data;
    const u64* offsets;
    u64 chars_bytes;
    const u8* null_map;
    i64 adjust;
    u64 rows;
};

__device__ __forceinline__ uint4 make_value(u32 type, u32 length, u64 data) {
    return make_uint4(type << 16, length, (u32)data, (u32)(data >> 32));  // id 0 | type | flags 0, length, data
}

__global__ void __launch_bounds__(256) ch_to_values_kernel(const ChColumnDev c, uint4* __restrict__ out, u32* dev_err) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < c.rows; i += (u64)gridDim.x * blockDim.x) {
        uint4 v;
        switch (c.type) {
            case YTGPU_CH_INT8: v = make_value(YTGPU_TYPE_INT64, 0, (u64)(i64) static_cast<const int8_t*>(c.data)[i]); break;
            case YTGPU_CH_INT16: v = make_value(YTGPU_TYPE_INT64, 0, (u64)(i64) static_cast<const int16_t*>(c.data)[i]); break;
            case YTGPU_CH_INT32: v = make_value(YTGPU_TYPE_INT64, 0, (u64)(i64) static_cast<const i32*>(c.data)[i]); break;
            case YTGPU_CH_INT64: v = make_value(YTGPU_TYPE_INT64, 0, static_cast<const u64*>(c.data)[i]); break;
            case YTGPU_CH_UINT8: v = make_value(YTGPU_TYPE_UINT64, 0, static_cast<const u8*>(c.data)[i]); break;
            case YTGPU_CH_UINT16: v = make_value(YTGPU_TYPE_UINT64, 0, static_cast<const u16*>(c.data)[i]); break;
            case YTGPU_CH_UINT32: v = make_value(YTGPU_TYPE_UINT64, 0, static_cast<const u32*>(c.data)[i]); break;
            case YTGPU_CH_UINT64: v = make_value(YTGPU_TYPE_UINT64, 0, static_cast<const u64*>(c.data)[i]); break;
            case YTGPU_CH_FLOAT32:
                v = make_value(YTGPU_TYPE_DOUBLE, 0, (u64)__double_as_longlong((double)static_cast<const float*>(c.data)[i]));
                break;
            case YTGPU_CH_FLOAT64: v = make_value(YTGPU_TYPE_DOUBLE, 0, static_cast<const u64*>(c.data)[i]); break;
            case YTGPU_CH_BOOL: {
                const u8 b = static_cast<const u8*>(c.data)[i];
                if (b > 1) atomicOr(dev_err, DE_SCHEMA_VIOLATION);
                v = make_value(YTGPU_TYPE_BOOLEAN, 0, b);
                break;
            }
            case YTGPU_CH_STRING: {
                const u64 begin = i ? c.offsets[i - 1] : 0, end = c.offsets[i];
                if (end <= begin || end > c.chars_bytes) {  // sizeAt() includes the terminating zero: never empty
                    atomicOr(dev_err, DE_PART_OUT_OF_BOUNDS);
                    v = make_value(YTGPU_TYPE_STRING, 0, 0);
                } else {
                    v = make_value(YTGPU_TYPE_STRING, (u32)(end - begin - 1), begin);
                }
                break;
            }
            case YTGPU_CH_DATE: v = make_value(YTGPU_TYPE_UINT64, 0, (u16)((i64) static_cast<const u16*>(c.data)[i] + c.adjust)); break;
            case YTGPU_CH_DATE32: v = make_value(YTGPU_TYPE_INT64, 0, (u64)(i64)(i32)((i64) static_cast<const i32*>(c.data)[i] + c.adjust)); break;
            case YTGPU_CH_DATETIME: v = make_value(YTGPU_TYPE_UINT64, 0, (u32)((i64) static_cast<const u32*>(c.data)[i] + c.adjust)); break;
            case YTGPU_CH_DATETIME64: v = make_value(YTGPU_TYPE_INT64, 0, (u64)(static_cast<const i64*>(c.data)[i] + c.adjust)); break;
            default: {  // YTGPU_CH_TIMESTAMP
                const i64 t = static_cast<const i64*>(c.data)[i] + c.adjust;
                if (t < 0) atomicOr(dev_err, DE_PART_NEGATIVE);
                v = make_value(YTGPU_TYPE_UINT64, 0, (u64)t);
                break;
            }
        }
        if (c.null_map && c.null_map[i]) v = make_value(YTGPU_TYPE_NULL, 0, 0);
        out[i] = v;
    }
}

u32 element_bytes(int type) {
    switch (type) {
        case YTGPU_CH_INT8: case YTGPU_CH_UINT8: case YTGPU_CH_BOOL: return 1;
        case YTGPU_CH_INT16: case YTGPU_CH_UINT16: case YTGPU_CH_DATE: return 2;
        case YTGPU_CH_INT32: case YTGPU_CH_UINT32: case YTGPU_CH_FLOAT32: case YTGPU_CH_DATE32: case YTGPU_CH_DATETIME: return 4;
        case YTGPU_CH_INT64: case YTGPU_CH_UINT64: case YTGPU_CH_FLOAT64: case YTGPU_CH_DATETIME64: case YTGPU_CH_TIMESTAMP: return 8;
        default: return 0;
    }
}

Status convert_impl(Context* ctx, const ytgpu_ch_column* col, ytgpu_value* out, int out_mem) {
    if (!col) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null column");
    if (col->type < YTGPU_CH_INT8 || col->type > YTGPU_CH_TIMESTAMP)
        return make_status(YTGPU_ERR_UNSUPPORTED, "Conversion of ClickHouse type %d to YT type system is not supported on the GPU path", col->type);
    const u64 n = col->row_count;
    if (n == 0) return Status{};
    if (!col->data || !out || (col->type == YTGPU_CH_STRING && !col->offsets)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    if (out_mem == YTGPU_MEM_DEVICE && (reinterpret_cast<uintptr_t>(out) & 15))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "out_values must be 16-byte aligned");
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    ChColumnDev d{};
    d.type = col->type;
    d.data = col->data;
    d.offsets = col->offsets;
    d.chars_bytes = col->chars_bytes;
    d.null_map = col->null_map;
    d.adjust = col->time_adjustment;
    d.rows = n;
    InBuf<u8> data, nulls;
    InBuf<u64> offsets;
    if (col->type == YTGPU_CH_STRING) {
        // the values only carry offsets into the chars: the bytes themselves are not needed on the device
        YTGPU_TRY(offsets.stage(ctx, col->offsets, n, col->mem));
        d.offsets = offsets.p;
    } else {
        YTGPU_TRY(data.stage(ctx, static_cast<const u8*>(col->data), (size_t)n * element_bytes(col->type), col->mem));
        d.data = data.p;
    }
    YTGPU_TRY(nulls.stage(ctx, col->null_map, n, col->mem));
    d.null_map = nulls.p;
    OutBuf<uint4> o;
    YTGPU_TRY(o.prepare(ctx, reinterpret_cast<uint4*>(out), n, out_mem));
    {
        KernelTimer t(ctx, KC_DECODE);
        const unsigned blocks = (unsigned)std::min<u64>((n + 255) / 256, (u64)kNumSms * 16);
        ch_to_values_kernel<<<blocks, 256, 0, ctx->stream>>>(d, o.p, ctx->dev_err);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_TRY(o.download(ctx, n));
    Status s = check_device_errors(ctx);  // synchronises the stream
    if (s.ok()) return s;
    const u32 e = *ctx->host_err;
    if (e & DE_SCHEMA_VIOLATION) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "Cannot convert value to YT boolean: a UInt8 above 1");
    if (e & DE_PART_NEGATIVE) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "Cannot convert value to YT timestamp: negative after the timezone adjustment");
    if (e & DE_PART_OUT_OF_BOUNDS) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string offsets are not increasing or run past the chars");
    return s;
}

}  // namespace

extern "C" int ytgpu_convert_ch_column_to_values(ytgpu_context* h, const ytgpu_ch_column* column, ytgpu_value* out_values, int out_mem,
                                                 ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, convert_impl(as_context(h), column, out_values, out_mem));
}
