// gpu_internal.h — helpers shared by the adapter translation units (gpu_adapters.cpp, gpu_shuffle.cpp, gpu_aggregate.cpp,
// gpu_map_join.cpp).
#pragma once

#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

#include "../include/ytgpu.h"
#include "yt_query_client.h"
#include "yt_table_client.h"

namespace NYT::NTableClient::NDetail {

[[noreturn]] inline void ThrowFrom(const ytgpu_error& err) { throw TErrorException(err.code, err.message); }

//! One context per process for the adapters (private stream).  The device is the job's GPU slot: YTGPU_DEVICE
//! (set by the job proxy from the slot's CUDA_VISIBLE_DEVICES index; default 0).  The C ABI itself is
//! context-explicit and serialises the calls made on one context (ytgpu.h), so the adapters may be used from
//! the writer thread and the sort invoker pool at once; a job proxy with several GPU slots owns one context per slot.
inline ytgpu_context* GetGpuContext() {
    static ytgpu_context* ctx = nullptr;
    static std::once_flag once;
    static ytgpu_error err{};
    std::call_once(once, [] {
        const char* dev = std::getenv("YTGPU_DEVICE");
        ytgpu_context_create(dev ? std::atoi(dev) : 0, nullptr, &ctx, &err);
    });
    if (!ctx) ThrowFrom(err);
    return ctx;
}

inline bool IsStringLike(EValueType t) { return t >= EValueType::String && t <= EValueType::Composite; }

//! Rows -> flat ytgpu rowset holding the first `valueCount` values of every row (short rows padded with Null).
struct TFlatRowset {
    std::vector<ytgpu_value> Values;
    std::vector<uint8_t> Heap;
    std::vector<uint32_t> RowValueCounts;  // min(row count, valueCount) per row
    ytgpu_rowset_view View{};

    //! extraValueCount: columns appended after the copied ones (Null until the caller fills them, e.g. a stream tag).
    TFlatRowset(const std::vector<TUnversionedRow>& rows, uint32_t copiedValueCount, uint32_t extraValueCount = 0) {
        const uint32_t valueCount = copiedValueCount + extraValueCount;
        Values.resize(rows.size() * (size_t)valueCount);
        RowValueCounts.resize(rows.size());
        size_t heapBytes = 0;
        for (auto row : rows)
            for (uint32_t c = 0; c < copiedValueCount && c < row.GetCount(); ++c)
                if (IsStringLike(row[c].Type)) heapBytes += row[c].Length;
        Heap.resize(heapBytes ? heapBytes : 1);
        size_t off = 0;
        for (size_t r = 0; r < rows.size(); ++r) {
            RowValueCounts[r] = std::min<uint32_t>(copiedValueCount, rows[r].GetCount());
            for (uint32_t c = 0; c < valueCount; ++c) {
                ytgpu_value& dst = Values[r * (size_t)valueCount + c];
                if (c >= copiedValueCount || c >= rows[r].GetCount()) {
                    dst = ytgpu_value{0xffff, YTGPU_TYPE_NULL, 0, 0, 0};
                    continue;
                }
                const TUnversionedValue& v = rows[r][c];
                dst.id = v.Id;
                dst.type = (uint8_t)v.Type;
                dst.flags = v.Flags;
                dst.length = v.Length;
                if (IsStringLike(v.Type)) {
                    std::memcpy(Heap.data() + off, v.Data.String, v.Length);
                    dst.data = off;
                    off += v.Length;
                } else if (v.Type == EValueType::Boolean) {
                    dst.data = v.Data.Boolean ? 1 : 0;
                } else {
                    dst.data = v.Data.Uint64;
                }
            }
        }
        View.values = Values.data();
        View.row_count = rows.size();
        View.value_count = valueCount;
        View.string_heap = Heap.data();
        View.string_heap_bytes = Heap.size();
        View.mem = YTGPU_MEM_HOST;
    }
};

inline std::vector<ytgpu_key_column> KeyColumnsOf(const TComparator& comparator) {
    std::vector<ytgpu_key_column> cols(comparator.GetLength());
    for (int i = 0; i < comparator.GetLength(); ++i) {
        cols[i] = ytgpu_key_column{};
        cols[i].index = (uint32_t)i;
        cols[i].type = 0;   // schemaless key column: any scalar type (type order first, unversioned_row.cpp:440-442)
        cols[i].width = 0;  // measured on the device
        cols[i].descending = comparator.SortOrders()[i] == ESortOrder::Descending;
    }
    return cols;
}

// ---- exact size of a row inside a horizontal block (the block writers account capacity with it) ----
inline uint32_t VarUintSize(uint64_t v) {
    uint32_t s = 1;
    while (v >= 0x80) {
        v >>= 7;
        ++s;
    }
    return s;
}

inline uint64_t ZigZagEncode64(int64_t v) { return ((uint64_t)v << 1) ^ (uint64_t)(v >> 63); }

//! Bytes WriteRowValue emits for one value (unversioned_row.cpp:159-206).
inline uint32_t EncodedValueSize(const TUnversionedValue& v) {
    auto type = v.Type == EValueType::Composite ? EValueType::Any : v.Type;
    uint32_t s = VarUintSize(v.Id) + VarUintSize((uint16_t)type);
    switch (type) {
        case EValueType::Int64: s += VarUintSize(ZigZagEncode64(v.Data.Int64)); break;
        case EValueType::Uint64: s += VarUintSize(v.Data.Uint64); break;
        case EValueType::Double: s += 8; break;
        case EValueType::Boolean: s += 1; break;
        case EValueType::String:
        case EValueType::Any: s += VarUintSize(v.Length) + v.Length; break;
        default: break;
    }
    return s;
}

//! ui32 offset + varuint32 value count + values (schemaless_block_writer.cpp:40-64).
inline int64_t EncodedRowSize(TUnversionedRow row) {
    int64_t s = 4 + VarUintSize(row.GetCount());
    for (const auto* v = row.Begin(); v != row.End(); ++v) s += EncodedValueSize(*v);
    return s;
}

inline int64_t GetDataWeight(TUnversionedRow row) {  // unversioned_row.cpp:601-611
    int64_t w = 1;
    for (const auto* v = row.Begin(); v != row.End(); ++v) w += IsStringLike(v->Type) ? v->Length : (v->Type == EValueType::Null ? 0 : 8);
    return w;
}

}  // namespace NYT::NTableClient::NDetail

namespace NYql::NMiniKQL::NDetail {

//! A fixed-width Arrow column (host memory) as the column view of the C ABI: its offset as start_index, its validity
//! bitmap (if any) as an Arrow validity bitmap.
inline ytgpu_column_view ArrowColumnView(const TArrowColumn& a) {
    ytgpu_column_view v{};
    v.start_index = a.Offset;
    v.value_count = a.Length;
    v.value_type = a.ValueType;
    v.has_values = 1;
    v.bit_width = 64;
    v.values = a.Values;
    v.values_count = (uint64_t)(a.Offset + a.Length);
    v.null_bitmap = a.Validity;
    v.reserved = a.Validity ? YTGPU_COLUMN_ARROW_VALIDITY : 0;
    v.mem = YTGPU_MEM_HOST;
    return v;
}

// Element i of an Arrow binary / utf8 array is [Offsets[Offset + i], Offsets[Offset + i + 1]): the offsets of the window
// must not decrease (nor start below 0).
inline void CheckOffsets(const TArrowColumn& a, const char* side) {
    using NYT::NTableClient::TErrorException;
    const int32_t* o = a.Offsets + a.Offset;
    if (o[0] < 0) throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, std::string(side) + " string key: a negative offset");
    for (int64_t i = 0; i < a.Length; ++i)
        if (o[i + 1] < o[i]) throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, std::string(side) + " string key: decreasing offsets");
}

inline bool IsValid(const TArrowColumn& a, int64_t i) {
    const int64_t bit = a.Offset + i;
    return !a.Validity || ((a.Validity[bit >> 3] >> (bit & 7)) & 1);
}

}  // namespace NYql::NMiniKQL::NDetail
