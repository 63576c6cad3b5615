// string_column_reader.cu — value extraction of the four unversioned string segment layouts.
//
// Replaces the extractors of TUnversionedStringColumnReader (yt/yt/ytlib/table_chunk_format/string_column_reader.cpp):
//   TStringValueExtractorBase::GetOffset / SetStringValue :39-71  end(i) = expected_length * (i + 1) + ZigZagDecode32(offsets[i]),
//                                                                  a value spans [end(i - 1), end(i)) of the string data
//   TDictionaryStringValueExtractorBase::ExtractValue      :84-97  id 0 = NULL, else dictionary entry id - 1
//   TDirectStringValueExtractorBase::ExtractValue          :130-143 null bitmap, else value i
//   the dense / RLE readers :266-520                               RLE: the run of a row = last run start <= row
// One thread per row of the segment; every bit-packed vector is read in place (header word = size | width << 56).
#include "common.cuh"
#include "context.cuh"

using namespace ytgpu;

namespace {

struct Packed {
    const u64* words;  // header + payload
    u64 size;
    u32 width;
};

__device__ __forceinline__ u64 packed_at(const Packed& v, u64 j) {
    if (v.width == 0) return 0;
    const u64 bit = j * v.width;
    const u64* w = v.words + 1 + (bit >> 6);
    const u32 off = (u32)(bit & 63);
    u64 x = w[0] >> off;
    if (off + v.width > 64) x |= w[1] << (64 - off);
    return v.width == 64 ? x : (x & ((1ull << v.width) - 1));
}

__device__ __forceinline__ u32 end_offset(const Packed& offsets, u32 expected, u64 i) {
    const u32 z = (u32)packed_at(offsets, i);
    return expected * (u32)(i + 1) + (u32)((i32)(z >> 1) ^ -(i32)(z & 1));
}

struct SegmentDev {
    u32 type, rows, expected;
    Packed row_indexes, ids, offsets;
    const u8* bitmap;
    u32 strings_at;  // first byte of the string data inside the segment
};

__global__ void __launch_bounds__(256) decode_string_segment_kernel(const SegmentDev S, u32* __restrict__ out_start, u32* __restrict__ out_length,
                                                                    u8* __restrict__ out_null) {
    for (u32 i = blockIdx.x * blockDim.x + threadIdx.x; i < S.rows; i += gridDim.x * blockDim.x) {
        u64 k = i;  // index among the stored values: the row itself (dense) or its run (RLE)
        if (S.type == 0 || S.type == 2) {
            u64 lo = 0, hi = S.row_indexes.size;  // last run start <= i (run 0 starts at row 0)
            while (hi - lo > 1) {
                const u64 mid = (lo + hi) >> 1;
                if (packed_at(S.row_indexes, mid) <= i) lo = mid;
                else hi = mid;
            }
            k = lo;
        }
        bool nul;
        u64 entry = k;  // index into the offsets vector
        if (S.type == 0 || S.type == 1) {
            const u64 id = packed_at(S.ids, k);
            nul = id == 0;
            entry = id - 1;
        } else {
            nul = (S.bitmap[k >> 3] >> (k & 7)) & 1;
        }
        u32 start = 0, len = 0;
        if (!nul) {
            start = entry == 0 ? 0 : end_offset(S.offsets, S.expected, entry - 1);
            len = end_offset(S.offsets, S.expected, entry) - start;
        }
        out_start[i] = nul ? 0 : S.strings_at + start;
        out_length[i] = len;
        if (out_null) out_null[i] = nul ? 1 : 0;
    }
}

Status decode_string_segment_impl(Context* ctx, const ytgpu_string_segment* seg, const u8* data, u32* out_start, u32* out_length, u8* out_null,
                                  int mem) {
    if (!seg || !data || !out_start || !out_length) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    if (seg->type > 3) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "unknown string segment type %u", seg->type);
    const u64 rows = seg->row_count;
    if (rows == 0) return Status{};
    if (mem != YTGPU_MEM_HOST && (reinterpret_cast<uintptr_t>(data) & 7))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "segment data must be 8-byte aligned");
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    InBuf<u8> staged;
    YTGPU_TRY(staged.stage(ctx, data, seg->data_bytes, mem, 16));  // one readable word past the end
    const u8* dev = staged.p;
    // the structured parts, in writer order (ytgpu.h): sizes from the descriptor, checked against the vectors' own headers
    const int nstruct = seg->type == 3 || seg->type == 1 ? 2 : 3;
    u64 header[3] = {0, 0, 0};
    u64 at[4] = {0, 0, 0, 0};
    for (int p = 0; p < nstruct; ++p) at[p + 1] = at[p] + seg->part_bytes[p];
    if (at[nstruct] + seg->part_bytes[nstruct] != seg->data_bytes || (at[nstruct] & 7))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string segment: part sizes do not add up to data_bytes");
    auto is_bitmap = [&](int p) { return (seg->type == 3 && p == 1) || (seg->type == 2 && p == 2); };
    for (int p = 0; p < nstruct; ++p) {
        if (is_bitmap(p)) continue;
        if (seg->part_bytes[p] < 8) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string segment: part %d is too small for a bit-packed vector", p);
        if (mem == YTGPU_MEM_HOST) header[p] = *reinterpret_cast<const u64*>(data + at[p]);
        else YTGPU_CUDA_TRY(cudaMemcpyAsync(&header[p], dev + at[p], 8, cudaMemcpyDeviceToHost, ctx->stream));
    }
    if (mem != YTGPU_MEM_HOST) YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    auto packed = [&](int p, Packed* out) -> Status {
        out->words = reinterpret_cast<const u64*>(dev + at[p]);
        out->size = header[p] & ((1ull << 56) - 1);
        out->width = (u32)(header[p] >> 56);
        if (out->width > 64 || 8 * (1 + ((out->width * out->size + 63) >> 6)) != seg->part_bytes[p])
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string segment: bit-packed vector %d does not fit its part", p);
        return Status{};
    };
    SegmentDev S{};
    S.type = seg->type;
    S.rows = (u32)rows;
    S.expected = seg->expected_length;
    S.strings_at = (u32)at[nstruct];
    u64 stored = rows;  // values the ids / bitmap describe
    if (seg->type == 3) {
        YTGPU_TRY(packed(0, &S.offsets));
        S.bitmap = dev + at[1];
        if (S.offsets.size != rows || seg->part_bytes[1] < (rows + 7) / 8) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string segment: DirectDense sizes");
    } else if (seg->type == 1) {
        YTGPU_TRY(packed(0, &S.ids));
        YTGPU_TRY(packed(1, &S.offsets));
        if (S.ids.size != rows) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string segment: DictionaryDense sizes");
    } else if (seg->type == 2) {
        YTGPU_TRY(packed(0, &S.row_indexes));
        YTGPU_TRY(packed(1, &S.offsets));
        S.bitmap = dev + at[2];
        stored = S.row_indexes.size;
        if (stored == 0 || S.offsets.size != stored || seg->part_bytes[2] < (stored + 7) / 8)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string segment: DirectRle sizes");
    } else {
        YTGPU_TRY(packed(0, &S.row_indexes));
        YTGPU_TRY(packed(1, &S.ids));
        YTGPU_TRY(packed(2, &S.offsets));
        stored = S.row_indexes.size;
        if (stored == 0 || S.ids.size != stored) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string segment: DictionaryRle sizes");
    }
    OutBuf<u32> ds, dl;
    OutBuf<u8> dn;
    YTGPU_TRY(ds.prepare(ctx, out_start, rows, mem));
    YTGPU_TRY(dl.prepare(ctx, out_length, rows, mem));
    YTGPU_TRY(dn.prepare(ctx, out_null, rows, mem));
    {
        KernelTimer t(ctx, KC_DECODE, 1);
        const u32 grid = (u32)std::max<u64>(1, std::min<u64>((rows + 255) / 256, (u64)kNumSms * 8));
        decode_string_segment_kernel<<<grid, 256, 0, ctx->stream>>>(S, ds.p, dl.p, dn.p);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_TRY(ds.download(ctx, rows));
    YTGPU_TRY(dl.download(ctx, rows));
    YTGPU_TRY(dn.download(ctx, rows));
    if (mem == YTGPU_MEM_HOST) YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return Status{};
}

}  // namespace

extern "C" {

int ytgpu_decode_string_segment(ytgpu_context* h, const ytgpu_string_segment* segment, const uint8_t* segment_data, uint32_t* out_start,
                                uint32_t* out_length, uint8_t* out_null_bytemap, int mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, decode_string_segment_impl(as_context(h), segment, segment_data, out_start, out_length, out_null_bytemap, mem));
}

}  // extern "C"
