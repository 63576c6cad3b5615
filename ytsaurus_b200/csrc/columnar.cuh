// columnar.cuh — the device-side view of an IUnversionedColumnarRowBatch::TColumn (row_batch.h:49-191) and the per-value
// decode shared by the scan / group-by kernels (columnar.cu, groupby_multi.cu).  Everything is TU-local (anonymous
// namespace) so several .cu files may include it.
#pragma once

#include <algorithm>

#include "common.cuh"
#include "context.cuh"

namespace {

using namespace ytgpu;

struct ColumnDev {
    i64 start;
    i64 count;
    u64 base;
    const void* values;
    u64 values_count;
    const u8* bitmap;
    const u32* dict;
    const u64* rle;
    u64 rle_count;
    u8 bit_width;   // 8/16/32/64, 0 = bit-packed vector with header word
    u8 zigzag;
    u8 has_values;
    u8 value_type;
    u8 bitmap_is_validity;  // YTGPU_COLUMN_ARROW_VALIDITY: a set bit means VALID
    u32 packed_width;  // bits per value when bit_width == 0
};

__device__ __forceinline__ bool raw_bit_at(const u8* bm, u64 i) { return (bm[i >> 3] >> (i & 7)) & 1; }
// "value i of the value vector is null" for YT null bitmaps and for Arrow validity bitmaps
__device__ __forceinline__ bool null_bit_at(const ColumnDev& c, u64 i) { return raw_bit_at(c.bitmap, i) != (bool)c.bitmap_is_validity; }

__device__ __forceinline__ u64 fetch_raw(const ColumnDev& c, u64 k) {
    switch (c.bit_width) {
        case 64: return reinterpret_cast<const u64*>(c.values)[k];
        case 32: return reinterpret_cast<const u32*>(c.values)[k];
        case 16: return reinterpret_cast<const u16*>(c.values)[k];
        case 8: return reinterpret_cast<const u8*>(c.values)[k];
        case 1: return (reinterpret_cast<const u8*>(c.values)[k >> 3] >> (k & 7)) & 1;  // TBitmap of boolean values
        default: {
            const u32 w = c.packed_width;
            if (w == 0) return 0;
            const u64* data = reinterpret_cast<const u64*>(c.values) + 1;
            const u64 bit = k * w;
            const u64* word = data + (bit >> 6);
            const u32 off = (u32)(bit & 63);
            u64 v = word[0] >> off;
            if (off + w > 64) v |= word[1] << (64 - off);
            return w == 64 ? v : (v & ((1ull << w) - 1));
        }
    }
}

// largest k with rle[k] <= g  (TranslateRleIndex, columnar.cpp:737-770)
__device__ __forceinline__ u64 rle_pos(const u64* rle, u64 n, u64 g) {
    u64 lo = 0, cnt = n;
    while (cnt > 0) {
        u64 step = cnt >> 1, mid = lo + step;
        if (__ldg(rle + mid) <= g) {
            lo = mid + 1;
            cnt -= step + 1;
        } else {
            cnt = step;
        }
    }
    return lo - 1;
}

// The run holding row g found from a run `from` known to start at or before it (rle[from] <= g), whatever the distance:
// exponential steps forward, then a binary search inside the last step — 2 log2(distance) loads instead of log2(n), so a
// warp that walks a column front to back pays for the runs it crosses, not for the size of the column.
__device__ __forceinline__ u64 rle_pos_gallop(const u64* rle, u64 n, u64 g, u64 from) {
    u64 lo = from, step = 1;
    while (lo + step < n && __ldg(rle + lo + step) <= g) {
        lo += step;
        step <<= 1;
    }
    u64 hi = lo + step < n ? lo + step : n;  // rle[hi] > g, or hi == n
    while (hi - lo > 1) {
        const u64 mid = (lo + hi) >> 1;
        if (__ldg(rle + mid) <= g) lo = mid;
        else hi = mid;
    }
    return lo;
}

// The run holding row g when a run at or before it is already known (`from`: rle[from] <= g): rows handled by one warp
// are neighbours, so their runs are the same or the next few — a short forward walk instead of a binary search over all
// runs (20 dependent loads per row at 10^6 runs).  When the walk does not end quickly it continues in exponential steps.
__device__ __forceinline__ u64 rle_pos_from(const u64* rle, u64 n, u64 g, u64 from) {
    u64 pos = from;
#pragma unroll 1
    for (int step = 0; step < 8; ++step) {
        if (pos + 1 >= n || __ldg(rle + pos + 1) > g) return pos;
        ++pos;
    }
    return rle_pos_gallop(rle, n, g, pos);
}

constexpr u64 kNoRleHint = ~0ull;

// Decodes logical value i (0-based inside the batch).  *ch_null follows BuildNullBytemapForCHColumn.
// rle_hint: a run index known to start at or before row i (kNoRleHint = none).
__device__ __forceinline__ u64 decode_at(const ColumnDev& c, i64 i, bool* ch_null, u64 rle_hint = kNoRleHint) {
    const u64 g = (u64)(c.start + i);
    if (!c.has_values) {
        *ch_null = true;
        return 0;
    }
    const u64 pos = c.rle ? (rle_hint != kNoRleHint ? rle_pos_from(c.rle, c.rle_count, g, rle_hint) : rle_pos(c.rle, c.rle_count, g)) : g;
    bool is_null = false;
    u64 raw = 0;
    if (c.dict) {
        const u32 d = c.dict[pos];
        *ch_null = d == 0;
        if (d != 0) {
            if (c.bitmap && null_bit_at(c, d - 1)) is_null = true;
            else raw = fetch_raw(c, d - 1);
        }
    } else {
        const bool b = c.bitmap && null_bit_at(c, pos);
        *ch_null = b;
        if (b) is_null = true;
        else raw = fetch_raw(c, pos);
    }
    if (is_null) return 0;
    u64 x = raw + c.base;
    if (c.zigzag) x = (x >> 1) ^ (0 - (x & 1));
    return x;
}

// Value of row i of a column for interpreters that give each warp 32 consecutive rows (warp_row: the warp's first row) and
// run the same node in every lane: lane 0 finds the run of the warp's first row of an RLE column, the other lanes walk on
// from there.  A row that is not live reads nothing and is NULL.
__device__ __forceinline__ u64 scalar_value(const ColumnDev& c, u64 i, u64 warp_row, bool live, bool* nul) {
    u64 hint = kNoRleHint;
    if (c.rle && c.has_values) {
        u64 h = 0;
        if ((threadIdx.x & 31) == 0) h = rle_pos(c.rle, c.rle_count, (u64)c.start + warp_row);
        hint = __shfl_sync(0xffffffffu, h, 0);
    }
    *nul = true;
    if (!live) return 0;
    return decode_at(c, (i64)i, nul, hint);
}

// Fast path: plain 64-bit value vector (no dictionary / RLE / null bitmap); base and zig-zag still apply.
__host__ __device__ __forceinline__ bool is_direct64(const ColumnDev& c) {
    return c.has_values && c.bit_width == 64 && !c.dict && !c.rle && !c.bitmap;
}

// Values as unsigned words whose order is the value order: uint64 as is, int64 with the sign bit flipped, double with the
// usual sign transform (NaN ends up above +inf, like AggLess of the YQL aggregators).
__host__ __device__ __forceinline__ u64 minmax_encode(u8 vtype, u64 bits) {
    if (vtype == YTGPU_TYPE_INT64) return bits ^ 0x8000000000000000ull;
    if (vtype == YTGPU_TYPE_DOUBLE) {
        if ((bits & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) return ~0ull;  // NaN: the biggest (AggLess)
        return (bits >> 63) ? ~bits : (bits | 0x8000000000000000ull);
    }
    return bits;
}
__host__ __device__ __forceinline__ u64 minmax_decode(u8 vtype, u64 enc) {
    if (vtype == YTGPU_TYPE_INT64) return enc ^ 0x8000000000000000ull;
    if (vtype == YTGPU_TYPE_DOUBLE) {
        if (enc == ~0ull) return 0x7ff8000000000000ull;
        return (enc >> 63) ? (enc & 0x7fffffffffffffffull) : ~enc;
    }
    return enc;
}

// Predicate on a decoded value (a NULL never passes: callers check that first).
__device__ __forceinline__ bool passes(int op, u8 vtype, u64 v, u64 c) {
    if (op == YTGPU_CMP_NONE) return true;
    int cmp;
    if (vtype == YTGPU_TYPE_INT64) cmp = ((i64)v > (i64)c) - ((i64)v < (i64)c);
    else if (vtype == YTGPU_TYPE_DOUBLE) {
        double a = __longlong_as_double((long long)v), b = __longlong_as_double((long long)c);
        if (a != a || b != b) return op == YTGPU_CMP_NE;
        cmp = (a > b) - (a < b);
    } else cmp = (v > c) - (v < c);
    switch (op) {
        case YTGPU_CMP_LT: return cmp < 0;
        case YTGPU_CMP_LE: return cmp <= 0;
        case YTGPU_CMP_GT: return cmp > 0;
        case YTGPU_CMP_GE: return cmp >= 0;
        case YTGPU_CMP_EQ: return cmp == 0;
        default: return cmp != 0;
    }
}

// ---- host helpers ----
struct StagedColumn {
    ColumnDev dev{};
    InBuf<u8> values, bitmap;
    InBuf<u32> dict;
    InBuf<u64> rle;
};

Status stage_column(Context* ctx, const ytgpu_column_view* c, StagedColumn* s) {
    if (!c) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null column");
    if (c->start_index < 0 || c->value_count < 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "negative column range");
    if (c->bit_width != 0 && c->bit_width != 1 && c->bit_width != 8 && c->bit_width != 16 && c->bit_width != 32 && c->bit_width != 64)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "bit_width must be 0 (bit-packed), 1 (bitmap), 8, 16, 32 or 64");
    if (c->rle_indexes && c->rle_count == 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "empty RLE index vector");
    ColumnDev& d = s->dev;
    d.start = c->start_index;
    d.count = c->value_count;
    d.base = c->base_value;
    d.bit_width = c->bit_width;
    d.zigzag = c->zigzag;
    d.has_values = c->has_values && c->values;
    d.value_type = c->value_type;
    d.bitmap_is_validity = (c->reserved & YTGPU_COLUMN_ARROW_VALIDITY) ? 1 : 0;
    d.values_count = c->values_count;
    d.rle_count = c->rle_count;
    u32 packed_width = 0;
    u64 header = 0;
    if (d.has_values && c->bit_width == 0) {
        // header word: size | width << 56 (bit_packed_unsigned_vector-inl.h:115-124)
        if (c->mem == YTGPU_MEM_HOST) header = *reinterpret_cast<const u64*>(c->values);
        else YTGPU_CUDA_TRY(cudaMemcpy(&header, c->values, 8, cudaMemcpyDeviceToHost));
        packed_width = (u32)(header >> 56);
        d.values_count = header & ((1ull << 56) - 1);
        if (packed_width > 64) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "bit-packed vector width %u > 64", packed_width);
    }
    d.packed_width = packed_width;
    const size_t vbytes_exact = !d.has_values ? 0
        : (c->bit_width == 0 ? (size_t)(1 + ((packed_width * d.values_count + 63) >> 6)) * 8
                             : (c->bit_width == 1 ? (size_t)(c->values_count + 7) / 8 : (size_t)c->values_count * (c->bit_width / 8)));
    const size_t bm_entries = c->null_bitmap ? (size_t)((c->dictionary_indexes || c->rle_indexes) ? d.values_count
                                                        : (u64)(c->start_index + c->value_count)) : 0;
    YTGPU_TRY(s->values.stage(ctx, static_cast<const u8*>(c->values), vbytes_exact, c->mem, 16));  // one readable word past the end
    d.values = d.has_values ? s->values.p : nullptr;
    YTGPU_TRY(s->bitmap.stage(ctx, c->null_bitmap, (bm_entries + 7) / 8, c->mem));
    d.bitmap = s->bitmap.p;
    YTGPU_TRY(s->dict.stage(ctx, c->dictionary_indexes, c->dictionary_index_count, c->mem));
    d.dict = s->dict.p;
    YTGPU_TRY(s->rle.stage(ctx, c->rle_indexes, c->rle_count, c->mem));
    d.rle = s->rle.p;
    return Status{};
}

inline u32 blocks_for(u64 items, int threads, int per_sm) {
    return (u32)std::max<u64>(1, std::min<u64>((items + threads - 1) / threads, (u64)kNumSms * per_sm));
}

}  // namespace
