// gpu_map_join.cpp — the YQL block map join (IBlockMapJoin, yt_query_client.h) over the GPU join table of the C ABI
// (ytgpu_join_table_build_strings / ytgpu_join_table_probe_strings).  No CPU fallback: errors of the C ABI surface as TErrorException.
#include <cstring>

#include "gpu_internal.h"
#include "yt_query_client.h"

namespace NYql::NMiniKQL {

namespace {

using NYT::NTableClient::TErrorException;
using NYT::NTableClient::NDetail::GetGpuContext;
using NYT::NTableClient::NDetail::ThrowFrom;

int KindOf(EBlockJoinKind kind) {
    switch (kind) {
        case EBlockJoinKind::Inner: return YTGPU_JOIN_INNER;
        case EBlockJoinKind::Left: return YTGPU_JOIN_LEFT;
        case EBlockJoinKind::LeftSemi: return YTGPU_JOIN_SEMI;
        case EBlockJoinKind::LeftOnly: return YTGPU_JOIN_ANTI;
    }
    throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "unknown block join kind");
}

bool IsString(const TArrowColumn& a) { return a.ValueType == YTGPU_TYPE_STRING; }

//! A left block's string key as the C ABI takes it: starts and lengths from the Arrow offsets, the heap from
//! Offsets[Offset], so no byte before the window is passed.  Column's starts, lengths and null bytemap are set from the
//! vectors where they end up.
struct TLeftStrings {
    std::vector<uint64_t> Starts;
    std::vector<uint32_t> Lengths;
    std::vector<uint8_t> Nulls;  // empty without NULLs
    ytgpu_string_column Column{};
};

using NDetail::CheckOffsets;
using NDetail::IsValid;

class TGpuBlockMapJoin : public IBlockMapJoin {
public:
    TGpuBlockMapJoin(EBlockJoinKind kind, uint32_t keyCount) : Kind_(KindOf(kind)), KeyCount_(keyCount) {
        if (keyCount == 0 || keyCount > YTGPU_JOIN_MAX_KEYS)
            throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "a map join has 1.." + std::to_string(YTGPU_JOIN_MAX_KEYS) + " key columns");
        Right_.resize(keyCount);
    }

    ~TGpuBlockMapJoin() override {
        ytgpu_error err{};
        ytgpu_join_table_destroy(Table_, &err);  // before the process-wide context, which is never destroyed
    }

    void AddRightBlock(const std::vector<TArrowColumn>& keys) override {
        if (Table_) throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "AddRightBlock after the first ProbeBlock");
        CheckKeys(keys, "right");
        for (uint32_t k = 0; k < KeyCount_; ++k)
            if (HaveRight_ && Right_[k].Type != keys[k].ValueType)
                throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "right key " + std::to_string(k) + " changes its type between blocks");
        for (uint32_t k = 0; k < KeyCount_; ++k) Right_[k].Type = keys[k].ValueType;
        HaveRight_ = true;
        // the right side is copied into one column per key: numeric keys with an Arrow validity bitmap over all its rows,
        // string keys as one heap with starts, lengths and a null bytemap
        const int64_t n = keys[0].Length;
        for (uint32_t k = 0; k < KeyCount_; ++k) {
            const TArrowColumn& a = keys[k];
            TRightColumn& c = Right_[k];
            if (IsString(a)) {
                const uint8_t* bytes = static_cast<const uint8_t*>(a.Values);
                for (int64_t i = 0; i < n; ++i) {
                    const bool valid = IsValid(a, i);
                    const int32_t from = a.Offsets[a.Offset + i], to = a.Offsets[a.Offset + i + 1];
                    c.Starts.push_back(c.Heap.size());
                    c.Lengths.push_back(valid ? (uint32_t)(to - from) : 0);
                    c.Nulls.push_back(valid ? 0 : 1);
                    if (valid) c.Heap.insert(c.Heap.end(), bytes + from, bytes + to);
                }
                continue;
            }
            const uint64_t* src = static_cast<const uint64_t*>(a.Values);
            c.Values.insert(c.Values.end(), src + a.Offset, src + a.Offset + n);
            c.Validity.resize((RightRows_ + n + 7) / 8, 0);
            for (int64_t i = 0; i < n; ++i) {
                const uint64_t at = RightRows_ + (uint64_t)i;
                if (IsValid(a, i)) c.Validity[at >> 3] |= (uint8_t)(1u << (at & 7));
            }
        }
        RightRows_ += (uint64_t)n;
    }

    TResult ProbeBlock(const std::vector<TArrowColumn>& leftKeys) override {
        CheckKeys(leftKeys, "left");
        ytgpu_context* ctx = GetGpuContext();
        ytgpu_error err{};
        if (!Table_) Build(ctx, leftKeys);
        std::vector<ytgpu_column_view> views;
        std::vector<TLeftStrings> strings;
        for (const TArrowColumn& a : leftKeys)
            if (IsString(a)) strings.push_back(LeftStrings(a));
            else views.push_back(NDetail::ArrowColumnView(a));
        std::vector<ytgpu_string_column> columns;
        for (const TLeftStrings& s : strings) {
            ytgpu_string_column c = s.Column;
            c.starts = s.Starts.data();
            c.lengths = s.Lengths.data();
            c.null_bytemap = s.Nulls.empty() ? nullptr : s.Nulls.data();
            columns.push_back(c);
        }
        const uint32_t numeric = (uint32_t)views.size(), stringCount = (uint32_t)columns.size();
        TResult r;
        uint64_t count = 0;
        const bool rowsOnly = Kind_ == YTGPU_JOIN_SEMI || Kind_ == YTGPU_JOIN_ANTI;
        uint64_t capacity = (uint64_t)leftKeys[0].Length;  // a SEMI / ANTI list has at most one entry per left row
        if (!rowsOnly) {
            if (ytgpu_join_table_probe_strings(ctx, Table_, views.data(), numeric, columns.data(), stringCount, Kind_, nullptr, nullptr, 0, &count,
                                               YTGPU_MEM_HOST, &err) != YTGPU_OK)
                ThrowFrom(err);
            capacity = count;
            r.RightRows.resize(capacity);
        }
        r.LeftRows.resize(capacity);
        if (capacity && ytgpu_join_table_probe_strings(ctx, Table_, views.data(), numeric, columns.data(), stringCount, Kind_, r.LeftRows.data(),
                                                       rowsOnly ? nullptr : r.RightRows.data(), capacity, &count, YTGPU_MEM_HOST, &err) != YTGPU_OK)
            ThrowFrom(err);
        r.LeftRows.resize(capacity ? count : 0);
        if (!rowsOnly) r.RightRows.resize(r.LeftRows.size());
        return r;
    }

private:
    struct TRightColumn {
        std::vector<uint64_t> Values;
        std::vector<uint8_t> Validity;
        std::vector<uint8_t> Heap;  // a string key's bytes, starts, lengths and NULLs
        std::vector<uint64_t> Starts;
        std::vector<uint32_t> Lengths;
        std::vector<uint8_t> Nulls;
        uint8_t Type = 0;
    };

    // Key types: INT64, UINT64, DOUBLE, and STRING as an Arrow binary / utf8 array (Offsets given).  Whether a position is a
    // string key is fixed by the first block, right or left.
    void CheckKeys(const std::vector<TArrowColumn>& keys, const char* side) {
        if (keys.size() != KeyCount_)
            throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, std::string(side) + " block: " + std::to_string(keys.size()) + " key columns, the join has " +
                                                                  std::to_string(KeyCount_));
        for (size_t k = 0; k < keys.size(); ++k) {
            const uint8_t t = keys[k].ValueType;
            if (t != YTGPU_TYPE_INT64 && t != YTGPU_TYPE_UINT64 && t != YTGPU_TYPE_DOUBLE && !(t == YTGPU_TYPE_STRING && keys[k].Offsets))
                throw TErrorException(YTGPU_ERR_UNSUPPORTED, std::string(side) + " key " + std::to_string(k) +
                                                                 ": the map join takes INT64, UINT64, DOUBLE and STRING keys with 32-bit offsets");
            if (keys[k].Length != keys[0].Length)
                throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, std::string(side) + " block: key columns differ in length");
        }
        if (StringKey_.empty())
            for (const TArrowColumn& a : keys) StringKey_.push_back(IsString(a));
        for (size_t k = 0; k < keys.size(); ++k) {
            if (IsString(keys[k]) != StringKey_[k])
                throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, std::string(side) + " key " + std::to_string(k) +
                                                                      ": a string key in one block and a numeric key in another");
            if (IsString(keys[k])) CheckOffsets(keys[k], side);
        }
    }

    static TLeftStrings LeftStrings(const TArrowColumn& a) {
        TLeftStrings s;
        const int32_t* o = a.Offsets + a.Offset;
        s.Starts.resize(a.Length);
        s.Lengths.resize(a.Length);
        bool anyNull = false;
        for (int64_t i = 0; i < a.Length; ++i) {
            s.Starts[i] = (uint64_t)(o[i] - o[0]);
            s.Lengths[i] = (uint32_t)(o[i + 1] - o[i]);
            anyNull = anyNull || !IsValid(a, i);
        }
        if (anyNull) {
            s.Nulls.resize(a.Length);
            for (int64_t i = 0; i < a.Length; ++i) s.Nulls[i] = IsValid(a, i) ? 0 : 1;
        }
        s.Column.heap = static_cast<const uint8_t*>(a.Values) + o[0];
        s.Column.heap_bytes = (uint64_t)(o[a.Length] - o[0]);
        s.Column.row_count = (uint64_t)a.Length;
        s.Column.mem = YTGPU_MEM_HOST;
        return s;
    }

    // The right side as one table; without any right block its key types are the first left block's.
    void Build(ytgpu_context* ctx, const std::vector<TArrowColumn>& leftKeys) {
        std::vector<ytgpu_column_view> views;
        std::vector<ytgpu_string_column> strings;
        for (uint32_t k = 0; k < KeyCount_; ++k) {
            const TRightColumn& c = Right_[k];
            if (StringKey_[k]) {
                ytgpu_string_column s{};
                s.heap = c.Heap.data();
                s.heap_bytes = c.Heap.size();
                s.starts = c.Starts.data();
                s.lengths = c.Lengths.data();
                s.null_bytemap = c.Nulls.data();
                s.row_count = RightRows_;
                s.mem = YTGPU_MEM_HOST;
                strings.push_back(s);
                continue;
            }
            ytgpu_column_view v{};
            v.value_count = (int64_t)RightRows_;
            v.value_type = HaveRight_ ? c.Type : leftKeys[k].ValueType;
            v.has_values = 1;
            v.bit_width = 64;
            v.values = c.Values.data();
            v.values_count = RightRows_;
            v.null_bitmap = c.Validity.data();
            v.reserved = YTGPU_COLUMN_ARROW_VALIDITY;
            v.mem = YTGPU_MEM_HOST;
            views.push_back(v);
        }
        ytgpu_error err{};
        if (ytgpu_join_table_build_strings(ctx, views.data(), (uint32_t)views.size(), strings.data(), (uint32_t)strings.size(),
                                           YTGPU_JOIN_NULLS_NEVER_MATCH, &Table_, &err) != YTGPU_OK)
            ThrowFrom(err);
        Right_ = std::vector<TRightColumn>(KeyCount_);  // the table owns its copy
    }

    const int Kind_;
    const uint32_t KeyCount_;
    std::vector<TRightColumn> Right_;
    std::vector<bool> StringKey_;
    uint64_t RightRows_ = 0;
    bool HaveRight_ = false;
    ytgpu_join_table* Table_ = nullptr;
};

}  // namespace

std::unique_ptr<IBlockMapJoin> CreateGpuBlockMapJoin(EBlockJoinKind kind, uint32_t keyCount) {
    return std::make_unique<TGpuBlockMapJoin>(kind, keyCount);
}

}  // namespace NYql::NMiniKQL
