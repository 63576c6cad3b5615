// gpu_block_combine_keys.cpp — YQL BlockCombineHashed over key tuples with aggregate lists (IBlockCombineHashedKeys,
// yt_query_client.h) over one GPU GROUP BY table of the C ABI (ytgpu_groupby_table_*).  Blocks are staged in pinned host
// memory and folded into the table BlockCombineHashedKeysStageRows rows at a time.  No CPU fallback: errors of the C ABI
// surface as TErrorException.
#include <algorithm>
#include <cstring>

#include "gpu_internal.h"
#include "yt_query_client.h"

namespace NYql::NMiniKQL {

namespace {

using NDetail::CheckOffsets;
using NDetail::IsValid;
using NYT::NQueryClient::TAggregateItem;
using NYT::NTableClient::TErrorException;
using NYT::NTableClient::NDetail::GetGpuContext;
using NYT::NTableClient::NDetail::ThrowFrom;

//! A pinned host array (ytgpu_host_alloc) that grows by doubling and keeps its contents.
template <class T>
class TPinned {
public:
    TPinned() = default;
    TPinned(const TPinned&) = delete;
    TPinned& operator=(const TPinned&) = delete;
    ~TPinned() { ytgpu_host_free(Data_); }
    T* Data() { return Data_; }
    void Reserve(size_t n) {
        if (n <= Capacity_) return;
        size_t cap = Capacity_ ? Capacity_ : 1024;
        while (cap < n) cap <<= 1;
        T* p = static_cast<T*>(ytgpu_host_alloc(cap * sizeof(T)));
        if (!p) throw TErrorException(YTGPU_ERR_OUT_OF_MEMORY, "pinned host allocation failed");
        if (Data_) std::memcpy(p, Data_, Capacity_ * sizeof(T));
        ytgpu_host_free(Data_);
        Data_ = p;
        Capacity_ = cap;
    }

private:
    T* Data_ = nullptr;
    size_t Capacity_ = 0;
};

//! One staged column: numeric values with a null bytemap turned into Arrow validity bits, or a string column's heap,
//! starts, lengths and null bytemap.
struct TStaged {
    TPinned<uint64_t> Values;
    TPinned<uint8_t> Validity;  // Arrow bits, 1 = valid
    TPinned<uint8_t> Heap;
    TPinned<uint64_t> Starts;
    TPinned<uint32_t> Lengths;
    TPinned<uint8_t> Nulls;
    uint64_t HeapBytes = 0;
};

bool IsString(const TArrowColumn& a) { return a.ValueType == YTGPU_TYPE_STRING; }
bool IsNumber(uint8_t t) { return t == YTGPU_TYPE_INT64 || t == YTGPU_TYPE_UINT64 || t == YTGPU_TYPE_DOUBLE; }

class TGpuBlockCombineHashedKeys : public IBlockCombineHashedKeys {
public:
    TGpuBlockCombineHashedKeys(std::vector<TAggregateItem> aggregates, uint64_t hint) : Aggregates_(std::move(aggregates)), Hint_(hint) {}

    ~TGpuBlockCombineHashedKeys() override {
        ytgpu_error err{};
        ytgpu_groupby_table_destroy(Table_, &err);  // before the process-wide context, which is never destroyed
    }

    void AddBlock(const std::vector<TArrowColumn>& keys, const std::vector<TArrowColumn>& values) override {
        Check(keys, values);
        if (!Table_) Create(keys, values);
        const int64_t n = keys[0].Length;
        for (int64_t done = 0; done < n;) {
            const int64_t take = std::min<int64_t>(n - done, (int64_t)(BlockCombineHashedKeysStageRows - Staged_));
            Stage(keys, values, done, take);
            done += take;
            if (Staged_ == BlockCombineHashedKeysStageRows) Flush();
        }
    }

    TResult Finish() override {
        TResult r;
        if (!Table_) return r;
        Flush();
        ytgpu_context* ctx = GetGpuContext();
        ytgpu_error err{};
        const uint32_t strings = (uint32_t)StringKeys_.size(), numeric = (uint32_t)NumericKeys_.size(), aggs = (uint32_t)Aggregates_.size();
        const uint32_t valueStrings = StringValued_, outputs = strings + valueStrings;
        std::vector<ytgpu_groupby_string_keys> sout(outputs);  // the string keys, then the string-valued aggregates
        uint64_t* none[1] = {nullptr};
        uint8_t* noneb[1] = {nullptr};
        ytgpu_groupby_multi_result q{};
        q.keys = none;
        q.key_null = noneb;
        q.values = none;
        q.value_null = noneb;
        const int code = ytgpu_groupby_table_result_strings(ctx, Table_, &q, sout.data(), strings, sout.data() + strings, valueStrings,
                                                            YTGPU_MEM_HOST, &err);
        if (code != YTGPU_OK && !(code == YTGPU_ERR_INVALID_ARGUMENT && q.group_count > 0)) ThrowFrom(err);  // capacity 0: the count
        const uint64_t g = q.group_count;
        r.Keys.assign(numeric, std::vector<uint64_t>(g));
        r.KeyValid.assign(numeric, std::vector<uint8_t>(g));
        r.Values.assign(aggs, std::vector<uint64_t>(g));
        r.ValueValid.assign(aggs, std::vector<uint8_t>(g));
        if (g == 0) {
            r.StringKeyBytes.assign(strings, std::string());
            r.StringKeyOffsets.assign(strings, std::vector<int32_t>(1, 0));
            r.StringKeyValid.assign(strings, std::vector<uint8_t>());
            r.StringValueBytes.assign(valueStrings, std::string());
            r.StringValueOffsets.assign(valueStrings, std::vector<int32_t>(1, 0));
            r.StringValueValid.assign(valueStrings, std::vector<uint8_t>());
            return r;
        }
        std::vector<uint64_t*> keys(numeric + 1), values(aggs + 1);
        std::vector<uint8_t*> keyNull(numeric + 1), valueNull(aggs + 1);
        for (uint32_t k = 0; k < numeric; ++k) {
            keys[k] = r.Keys[k].data();
            keyNull[k] = r.KeyValid[k].data();
        }
        for (uint32_t a = 0; a < aggs; ++a) {
            values[a] = r.Values[a].data();
            valueNull[a] = r.ValueValid[a].data();
        }
        std::vector<std::vector<uint8_t>> heaps(outputs), nulls(outputs);
        std::vector<std::vector<uint64_t>> starts(outputs);
        std::vector<std::vector<uint32_t>> lengths(outputs);
        for (uint32_t s = 0; s < outputs; ++s) {
            heaps[s].resize(std::max<uint64_t>(sout[s].heap_bytes, 1));
            starts[s].resize(g);
            lengths[s].resize(g);
            nulls[s].resize(g);
            sout[s].heap = heaps[s].data();
            sout[s].heap_capacity = sout[s].heap_bytes;
            sout[s].starts = starts[s].data();
            sout[s].lengths = lengths[s].data();
            sout[s].null_bytemap = nulls[s].data();
        }
        ytgpu_groupby_multi_result out{};
        out.capacity = g;
        out.keys = keys.data();
        out.key_null = keyNull.data();
        out.values = values.data();
        out.value_null = valueNull.data();
        if (ytgpu_groupby_table_result_strings(ctx, Table_, &out, sout.data(), strings, sout.data() + strings, valueStrings, YTGPU_MEM_HOST,
                                               &err) != YTGPU_OK)
            ThrowFrom(err);
        for (auto& v : r.KeyValid)
            for (uint8_t& b : v) b = !b;  // null bytemap -> validity
        for (auto& v : r.ValueValid)
            for (uint8_t& b : v) b = !b;
        for (uint32_t s = 0; s < outputs; ++s) {
            const bool key = s < strings;
            if (sout[s].heap_bytes > (uint64_t)INT32_MAX)
                throw TErrorException(YTGPU_ERR_UNSUPPORTED, std::string(key ? "string key " : "string value ") + std::to_string(key ? s : s - strings) +
                                                                 ": more than 2^31 - 1 bytes in 32-bit Arrow offsets");
            (key ? r.StringKeyBytes : r.StringValueBytes).emplace_back(reinterpret_cast<const char*>(heaps[s].data()), sout[s].heap_bytes);
            std::vector<int32_t> offsets(g + 1, 0);
            for (uint64_t o = 0; o < g; ++o) offsets[o + 1] = offsets[o] + (int32_t)lengths[s][o];  // starts are in output order
            (key ? r.StringKeyOffsets : r.StringValueOffsets).push_back(std::move(offsets));
            std::vector<uint8_t> valid(g);
            for (uint64_t o = 0; o < g; ++o) valid[o] = !nulls[s][o];
            (key ? r.StringKeyValid : r.StringValueValid).push_back(std::move(valid));
        }
        return r;
    }

private:
    // Every check of a block, before anything is staged.
    void Check(const std::vector<TArrowColumn>& keys, const std::vector<TArrowColumn>& values) {
        if (keys.empty() || keys.size() > 8)
            throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "a block has 1..8 key columns");
        for (size_t k = 0; k < keys.size(); ++k) {
            const TArrowColumn& a = keys[k];
            if (!IsNumber(a.ValueType) && !(IsString(a) && a.Offsets))
                throw TErrorException(YTGPU_ERR_UNSUPPORTED, "key " + std::to_string(k) + ": INT64, UINT64, DOUBLE and STRING keys with 32-bit offsets");
            if (a.Length != keys[0].Length || a.Offset < 0 || a.Length < 0)
                throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "key columns differ in length or have a negative window");
            if (IsString(a)) CheckOffsets(a, "block");
        }
        for (size_t v = 0; v < values.size(); ++v) {
            const TArrowColumn& a = values[v];
            if (!IsNumber(a.ValueType) && !(IsString(a) && a.Offsets))
                throw TErrorException(YTGPU_ERR_UNSUPPORTED, "value " + std::to_string(v) + ": INT64, UINT64, DOUBLE and STRING values with 32-bit offsets");
            if (a.Length != keys[0].Length || a.Offset < 0)
                throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "value column " + std::to_string(v) + " differs in length from the keys");
            if (IsString(a)) CheckOffsets(a, "block");
        }
        if (!Table_) return;
        if (keys.size() != KeyTypes_.size() || values.size() != ValueTypes_.size())
            throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "a block's key or value count differs from the first block's");
        for (size_t k = 0; k < keys.size(); ++k)
            if (keys[k].ValueType != KeyTypes_[k])
                throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "key " + std::to_string(k) + " changes its type between blocks");
        for (size_t v = 0; v < values.size(); ++v)
            if (values[v].ValueType != ValueTypes_[v])
                throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "value " + std::to_string(v) + " changes its type between blocks");
    }

    void Create(const std::vector<TArrowColumn>& keys, const std::vector<TArrowColumn>& values) {
        std::vector<uint8_t> numericTypes;
        for (size_t k = 0; k < keys.size(); ++k) {
            KeyTypes_.push_back(keys[k].ValueType);
            if (IsString(keys[k])) StringKeys_.push_back(k);
            else {
                NumericKeys_.push_back(k);
                numericTypes.push_back(keys[k].ValueType);
            }
        }
        // the table's value columns are the numeric values in their order, then the string values in theirs
        std::vector<uint8_t> numericValueTypes;
        for (size_t v = 0; v < values.size(); ++v) {
            ValueTypes_.push_back(values[v].ValueType);
            if (IsString(values[v])) StringValues_.push_back(v);
            else {
                NumericValues_.push_back(v);
                numericValueTypes.push_back(values[v].ValueType);
            }
        }
        std::vector<int32_t> index(values.size());
        for (size_t i = 0; i < NumericValues_.size(); ++i) index[NumericValues_[i]] = (int32_t)i;
        for (size_t i = 0; i < StringValues_.size(); ++i) index[StringValues_[i]] = (int32_t)(NumericValues_.size() + i);
        auto remap = [&](int32_t c) { return c >= 0 && (size_t)c < values.size() ? index[c] : c; };
        std::vector<ytgpu_aggregate> aggs;
        StringValued_ = 0;
        for (const TAggregateItem& a : Aggregates_) {
            aggs.push_back(ytgpu_aggregate{(int32_t)a.Function, remap(a.Column), remap(a.ByColumn), 0});  // EAggregateFunction follows ytgpu_agg_op
            if (a.Column >= 0 && (size_t)a.Column < values.size() && IsString(values[a.Column]) && aggs.back().op != YTGPU_AGG_COUNT) ++StringValued_;
        }
        ytgpu_error err{};
        ytgpu_groupby_table* t = nullptr;
        if (ytgpu_groupby_table_create_strings(GetGpuContext(), numericTypes.data(), (uint32_t)numericTypes.size(), (uint32_t)StringKeys_.size(),
                                               numericValueTypes.data(), (uint32_t)numericValueTypes.size(), (uint32_t)StringValues_.size(),
                                               aggs.data(), (uint32_t)aggs.size(), Hint_, &t, &err) != YTGPU_OK) {
            KeyTypes_.clear();
            StringKeys_.clear();
            NumericKeys_.clear();
            ValueTypes_.clear();
            NumericValues_.clear();
            StringValues_.clear();
            ThrowFrom(err);
        }
        Table_ = t;
        Keys_ = std::vector<TStaged>(keys.size());
        Values_ = std::vector<TStaged>(values.size());
        for (TStaged& s : Keys_) Reserve(s);
        for (TStaged& s : Values_) Reserve(s);
    }

    static void Reserve(TStaged& s) {
        s.Values.Reserve(BlockCombineHashedKeysStageRows);
        s.Validity.Reserve(BlockCombineHashedKeysStageRows / 8);
    }

    // Rows [from, from + count) of the block after the staged rows.
    void Stage(const std::vector<TArrowColumn>& keys, const std::vector<TArrowColumn>& values, int64_t from, int64_t count) {
        auto numeric = [&](const TArrowColumn& a, TStaged& s) {
            const uint64_t* src = static_cast<const uint64_t*>(a.Values) + a.Offset + from;
            std::memcpy(s.Values.Data() + Staged_, src, (size_t)count * 8);
            uint8_t* bits = s.Validity.Data();
            for (int64_t i = 0; i < count; ++i) {
                const uint64_t at = Staged_ + (uint64_t)i;
                if (at % 8 == 0) bits[at >> 3] = 0;
                if (IsValid(a, from + i)) bits[at >> 3] |= (uint8_t)(1u << (at & 7));
            }
        };
        auto strings = [&](const TArrowColumn& a, TStaged& s) {
            s.Starts.Reserve(BlockCombineHashedKeysStageRows);
            s.Lengths.Reserve(BlockCombineHashedKeysStageRows);
            s.Nulls.Reserve(BlockCombineHashedKeysStageRows);
            const int32_t* o = a.Offsets + a.Offset + from;
            const uint64_t bytes = (uint64_t)(o[count] - o[0]);
            s.Heap.Reserve(s.HeapBytes + bytes + 1);
            std::memcpy(s.Heap.Data() + s.HeapBytes, static_cast<const uint8_t*>(a.Values) + o[0], bytes);
            for (int64_t i = 0; i < count; ++i) {
                const uint64_t at = Staged_ + (uint64_t)i;
                s.Starts.Data()[at] = s.HeapBytes + (uint64_t)(o[i] - o[0]);
                s.Lengths.Data()[at] = (uint32_t)(o[i + 1] - o[i]);
                s.Nulls.Data()[at] = IsValid(a, from + i) ? 0 : 1;
            }
            s.HeapBytes += bytes;
        };
        auto stage = [&](const TArrowColumn& a, TStaged& s) {
            if (IsString(a)) strings(a, s);
            else numeric(a, s);
        };
        for (size_t k = 0; k < keys.size(); ++k) stage(keys[k], Keys_[k]);
        for (size_t v = 0; v < values.size(); ++v) stage(values[v], Values_[v]);
        Staged_ += (uint64_t)count;
    }

    // One update over the staged rows.
    void Flush() {
        if (Staged_ == 0) return;
        auto view = [&](TStaged& s, uint8_t type) {
            ytgpu_column_view v{};
            v.value_count = (int64_t)Staged_;
            v.value_type = type;
            v.has_values = 1;
            v.bit_width = 64;
            v.values = s.Values.Data();
            v.values_count = Staged_;
            v.null_bitmap = s.Validity.Data();
            v.reserved = YTGPU_COLUMN_ARROW_VALIDITY;
            v.mem = YTGPU_MEM_HOST;
            return v;
        };
        auto stringView = [&](TStaged& s) {
            ytgpu_string_column c{};
            c.heap = s.Heap.Data();
            c.heap_bytes = s.HeapBytes;
            c.starts = s.Starts.Data();
            c.lengths = s.Lengths.Data();
            c.null_bytemap = s.Nulls.Data();
            c.row_count = Staged_;
            c.mem = YTGPU_MEM_HOST;
            return c;
        };
        std::vector<ytgpu_column_view> keys, values;
        std::vector<ytgpu_string_column> strings, stringValues;
        for (size_t k : NumericKeys_) keys.push_back(view(Keys_[k], KeyTypes_[k]));
        for (size_t k : StringKeys_) strings.push_back(stringView(Keys_[k]));
        for (size_t v : NumericValues_) values.push_back(view(Values_[v], ValueTypes_[v]));
        for (size_t v : StringValues_) stringValues.push_back(stringView(Values_[v]));
        ytgpu_error err{};
        const int code = ytgpu_groupby_table_update_strings(GetGpuContext(), Table_, keys.data(), (uint32_t)keys.size(), strings.data(),
                                                            (uint32_t)strings.size(), values.data(), (uint32_t)values.size(),
                                                            stringValues.data(), (uint32_t)stringValues.size(), nullptr, -1, &err);
        Staged_ = 0;
        for (TStaged& s : Keys_) s.HeapBytes = 0;
        for (TStaged& s : Values_) s.HeapBytes = 0;
        if (code != YTGPU_OK) ThrowFrom(err);
    }

    const std::vector<TAggregateItem> Aggregates_;
    const uint64_t Hint_;
    ytgpu_groupby_table* Table_ = nullptr;
    std::vector<uint8_t> KeyTypes_, ValueTypes_;
    std::vector<size_t> NumericKeys_, StringKeys_, NumericValues_, StringValues_;
    uint32_t StringValued_ = 0;  // aggregates whose result is a string
    std::vector<TStaged> Keys_, Values_;
    uint64_t Staged_ = 0;
};

}  // namespace

std::unique_ptr<IBlockCombineHashedKeys> CreateGpuBlockCombineHashedKeys(std::vector<NYT::NQueryClient::TAggregateItem> aggregates, uint64_t groupCountHint) {
    return std::make_unique<TGpuBlockCombineHashedKeys>(std::move(aggregates), groupCountHint);
}

}  // namespace NYql::NMiniKQL
