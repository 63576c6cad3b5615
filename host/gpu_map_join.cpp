// gpu_map_join.cpp — the YQL block map join (IBlockMapJoin, yt_query_client.h) over the GPU join table of the C ABI
// (ytgpu_join_table_build / ytgpu_join_table_probe).  No CPU fallback: errors of the C ABI surface as TErrorException.
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
        // the right side is copied into one column per key, with an Arrow validity bitmap over all its rows
        const int64_t n = keys[0].Length;
        for (uint32_t k = 0; k < KeyCount_; ++k) {
            const TArrowColumn& a = keys[k];
            TRightColumn& c = Right_[k];
            const uint64_t* src = static_cast<const uint64_t*>(a.Values);
            c.Values.insert(c.Values.end(), src + a.Offset, src + a.Offset + n);
            c.Validity.resize((RightRows_ + n + 7) / 8, 0);
            for (int64_t i = 0; i < n; ++i) {
                const int64_t bit = a.Offset + i;
                const bool valid = !a.Validity || ((a.Validity[bit >> 3] >> (bit & 7)) & 1);
                const uint64_t at = RightRows_ + (uint64_t)i;
                if (valid) c.Validity[at >> 3] |= (uint8_t)(1u << (at & 7));
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
        for (const TArrowColumn& a : leftKeys) views.push_back(NDetail::ArrowColumnView(a));
        TResult r;
        uint64_t count = 0;
        const bool rowsOnly = Kind_ == YTGPU_JOIN_SEMI || Kind_ == YTGPU_JOIN_ANTI;
        uint64_t capacity = (uint64_t)leftKeys[0].Length;  // a SEMI / ANTI list has at most one entry per left row
        if (!rowsOnly) {
            if (ytgpu_join_table_probe(ctx, Table_, views.data(), KeyCount_, Kind_, nullptr, nullptr, 0, &count, YTGPU_MEM_HOST, &err) != YTGPU_OK)
                ThrowFrom(err);
            capacity = count;
            r.RightRows.resize(capacity);
        }
        r.LeftRows.resize(capacity);
        if (capacity && ytgpu_join_table_probe(ctx, Table_, views.data(), KeyCount_, Kind_, r.LeftRows.data(),
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
        uint8_t Type = 0;
    };

    void CheckKeys(const std::vector<TArrowColumn>& keys, const char* side) const {
        if (keys.size() != KeyCount_)
            throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, std::string(side) + " block: " + std::to_string(keys.size()) + " key columns, the join has " +
                                                                  std::to_string(KeyCount_));
        for (size_t k = 0; k < keys.size(); ++k) {
            const uint8_t t = keys[k].ValueType;
            if (t != YTGPU_TYPE_INT64 && t != YTGPU_TYPE_UINT64 && t != YTGPU_TYPE_DOUBLE)
                throw TErrorException(YTGPU_ERR_UNSUPPORTED, std::string(side) + " key " + std::to_string(k) + ": the map join takes INT64, UINT64 and DOUBLE keys");
            if (keys[k].Length != keys[0].Length)
                throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, std::string(side) + " block: key columns differ in length");
        }
    }

    // The right side as one table; without any right block its key types are the first left block's.
    void Build(ytgpu_context* ctx, const std::vector<TArrowColumn>& leftKeys) {
        std::vector<ytgpu_column_view> views(KeyCount_);
        for (uint32_t k = 0; k < KeyCount_; ++k) {
            ytgpu_column_view& v = views[k];
            const TRightColumn& c = Right_[k];
            v.value_count = (int64_t)RightRows_;
            v.value_type = HaveRight_ ? c.Type : leftKeys[k].ValueType;
            v.has_values = 1;
            v.bit_width = 64;
            v.values = c.Values.data();
            v.values_count = RightRows_;
            v.null_bitmap = c.Validity.data();
            v.reserved = YTGPU_COLUMN_ARROW_VALIDITY;
            v.mem = YTGPU_MEM_HOST;
        }
        ytgpu_error err{};
        if (ytgpu_join_table_build(ctx, views.data(), KeyCount_, YTGPU_JOIN_NULLS_NEVER_MATCH, &Table_, &err) != YTGPU_OK) ThrowFrom(err);
        for (TRightColumn& c : Right_) {  // the table owns its copy
            c.Values = {};
            c.Validity = {};
        }
    }

    const int Kind_;
    const uint32_t KeyCount_;
    std::vector<TRightColumn> Right_;
    uint64_t RightRows_ = 0;
    bool HaveRight_ = false;
    ytgpu_join_table* Table_ = nullptr;
};

}  // namespace

std::unique_ptr<IBlockMapJoin> CreateGpuBlockMapJoin(EBlockJoinKind kind, uint32_t keyCount) {
    return std::make_unique<TGpuBlockMapJoin>(kind, keyCount);
}

}  // namespace NYql::NMiniKQL
