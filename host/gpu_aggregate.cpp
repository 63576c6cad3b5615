// gpu_aggregate.cpp — aggregate-side adapters: the reference's scan -> filter -> GROUP BY entry points
// (yt_query_client.h) whose compute is ytgpu_scan_filter_groupby (include/ytgpu.h).  Host code stays C++; no CPU
// fallback: errors of the C ABI surface as TErrorException.
#include <algorithm>
#include <cstring>
#include <map>
#include <numeric>
#include <unordered_map>

#include "gpu_internal.h"
#include "yt_query_client.h"

namespace NYT {

namespace {

using namespace NTableClient;
using namespace NTableClient::NDetail;

ytgpu_column_view ViewOf(const TColumnarColumn& c) {
    ytgpu_column_view v{};
    v.start_index = c.StartIndex;
    v.value_count = c.ValueCount;
    v.value_type = (uint8_t)c.Type;
    v.has_values = c.Values != nullptr;
    v.zigzag = c.ZigZagEncoded;
    v.bit_width = (uint8_t)c.BitWidth;
    v.base_value = c.BaseValue;
    v.values = c.Values;
    v.values_count = c.ValuesCount;
    v.null_bitmap = c.NullBitmap;
    v.dictionary_indexes = c.DictionaryIndexes;
    v.dictionary_index_count = c.DictionaryIndexCount;
    v.rle_indexes = c.RleIndexes;
    v.rle_count = c.RleCount;
    v.mem = YTGPU_MEM_HOST;
    return v;
}

int CmpOf(NQueryClient::EBinaryOp op) {
    using E = NQueryClient::EBinaryOp;
    switch (op) {
        case E::None: return YTGPU_CMP_NONE;
        case E::Less: return YTGPU_CMP_LT;
        case E::LessOrEqual: return YTGPU_CMP_LE;
        case E::Greater: return YTGPU_CMP_GT;
        case E::GreaterOrEqual: return YTGPU_CMP_GE;
        case E::Equal: return YTGPU_CMP_EQ;
        default: return YTGPU_CMP_NE;
    }
}

//! Partial aggregation states of the batches seen so far (Aggregator::executeOnBlock per batch) and their merge
//! (Aggregator::mergeBlocks; QL: the Intermediate -> Aggregated stream tags, cg_routines/registry.cpp:1783-1834).
class TPartialStates {
public:
    explicit TPartialStates(uint64_t hint, bool withMinMax = false) : Hint_(hint), WithMinMax_(withMinMax) {}

    //! One batch: decode + filter + GROUP BY on the GPU.  firstRowBase = rows of earlier batches (first-seen order).
    void AddBatch(const ytgpu_column_view& key, const ytgpu_column_view& value, int cmpOp, uint64_t constant, uint64_t firstRowBase) {
        const uint64_t n = (uint64_t)key.value_count;
        if (n == 0) return;
        ValueType_ = value.value_type;
        uint64_t cap = std::min<uint64_t>(n, Hint_ ? 2 * Hint_ : n) + 2;
        for (;;) {
            std::vector<uint64_t> k(cap), s(cap), c(cap), f(cap), mn(WithMinMax_ ? cap : 0), mx(WithMinMax_ ? cap : 0);
            std::vector<uint8_t> kn(cap), sn(cap);
            ytgpu_groupby_result res{0, k.data(), kn.data(), s.data(), sn.data(), c.data(), cap, f.data(),
                                     WithMinMax_ ? mn.data() : nullptr, WithMinMax_ ? mx.data() : nullptr};
            ytgpu_predicate pred{cmpOp, 0, constant};
            ytgpu_error err{};
            int code = ytgpu_scan_filter_groupby(GetGpuContext(), &key, &value, cmpOp == YTGPU_CMP_NONE ? nullptr : &pred, Hint_, &res,
                                                 YTGPU_MEM_HOST, &err);
            if (code == YTGPU_ERR_INVALID_ARGUMENT && res.group_count > cap) {  // more groups than the hint promised
                cap = res.group_count + 2;
                continue;
            }
            if (code != YTGPU_OK) ThrowFrom(err);
            ++Batches_;
            for (uint64_t i = 0; i < res.group_count; ++i) {
                Keys_.push_back(k[i]);
                KeyNulls_.push_back(kn[i]);
                Sums_.push_back(s[i]);
                SumNulls_.push_back(sn[i]);
                Counts_.push_back(c[i]);
                Firsts_.push_back(f[i] + firstRowBase);
                if (WithMinMax_) {
                    Mins_.push_back(mn[i]);
                    Maxs_.push_back(mx[i]);
                }
            }
            return;
        }
    }

    struct TMerged {
        std::vector<uint64_t> Keys, Sums, Counts, Firsts, Mins, Maxs;  // Mins / Maxs: NULL where SumNulls is set
        std::vector<uint8_t> KeyNulls, SumNulls;
    };

    //! Groups ordered by (key_null, key), with the first row index of every group.
    TMerged Merge() {
        TMerged m;
        const uint64_t p = Keys_.size();
        if (p == 0) return m;
        if (Batches_ <= 1) {
            m.Keys = Keys_; m.Sums = Sums_; m.Counts = Counts_; m.Firsts = Firsts_; m.KeyNulls = KeyNulls_; m.SumNulls = SumNulls_;
            m.Mins = Mins_; m.Maxs = Maxs_;
            return m;
        }
        // SUM of the partial sums and SUM of the partial counts per key: the same kernel, the partial states as its input
        auto bitmap = [](const std::vector<uint8_t>& flags) {
            std::vector<uint8_t> bm((flags.size() + 7) / 8, 0);
            for (size_t i = 0; i < flags.size(); ++i)
                if (flags[i]) bm[i >> 3] |= (uint8_t)(1u << (i & 7));
            return bm;
        };
        const auto knBitmap = bitmap(KeyNulls_), snBitmap = bitmap(SumNulls_);
        const bool anyKeyNull = std::any_of(KeyNulls_.begin(), KeyNulls_.end(), [](uint8_t x) { return x; });
        const bool anySumNull = std::any_of(SumNulls_.begin(), SumNulls_.end(), [](uint8_t x) { return x; });
        auto column = [&](const std::vector<uint64_t>& vals, uint8_t type, const std::vector<uint8_t>* bm) {
            ytgpu_column_view v{};
            v.value_count = (int64_t)p;
            v.value_type = type;
            v.has_values = 1;
            v.bit_width = 64;
            v.values = vals.data();
            v.values_count = p;
            v.null_bitmap = bm ? bm->data() : nullptr;
            v.mem = YTGPU_MEM_HOST;
            return v;
        };
        const auto kcol = column(Keys_, YTGPU_TYPE_UINT64, anyKeyNull ? &knBitmap : nullptr);
        const auto scol = column(Sums_, ValueType_, anySumNull ? &snBitmap : nullptr);
        const auto ccol = column(Counts_, YTGPU_TYPE_UINT64, nullptr);
        const uint64_t cap = p + 2;
        std::vector<uint64_t> k2(cap), c2(cap), unused(cap);
        std::vector<uint8_t> kn2(cap), un2(cap);
        m.Keys.resize(cap); m.Sums.resize(cap); m.KeyNulls.resize(cap); m.SumNulls.resize(cap);
        ytgpu_error err{};
        ytgpu_groupby_result r1{0, m.Keys.data(), m.KeyNulls.data(), m.Sums.data(), m.SumNulls.data(), unused.data(), cap, nullptr};
        if (ytgpu_scan_filter_groupby(GetGpuContext(), &kcol, &scol, nullptr, p, &r1, YTGPU_MEM_HOST, &err) != YTGPU_OK) ThrowFrom(err);
        ytgpu_groupby_result r2{0, k2.data(), kn2.data(), c2.data(), un2.data(), unused.data(), cap, nullptr};
        if (ytgpu_scan_filter_groupby(GetGpuContext(), &kcol, &ccol, nullptr, p, &r2, YTGPU_MEM_HOST, &err) != YTGPU_OK) ThrowFrom(err);
        const uint64_t g = r1.group_count;
        if (WithMinMax_) {
            // MIN of the partial minima, MAX of the partial maxima (a partial state without values is NULL like its sum)
            const auto mncol = column(Mins_, ValueType_, anySumNull ? &snBitmap : nullptr);
            const auto mxcol = column(Maxs_, ValueType_, anySumNull ? &snBitmap : nullptr);
            m.Mins.resize(cap); m.Maxs.resize(cap);
            std::vector<uint64_t> s3(cap);
            ytgpu_groupby_result r3{0, k2.data(), kn2.data(), s3.data(), un2.data(), unused.data(), cap, nullptr, m.Mins.data(), nullptr};
            if (ytgpu_scan_filter_groupby(GetGpuContext(), &kcol, &mncol, nullptr, p, &r3, YTGPU_MEM_HOST, &err) != YTGPU_OK) ThrowFrom(err);
            ytgpu_groupby_result r4{0, k2.data(), kn2.data(), s3.data(), un2.data(), unused.data(), cap, nullptr, nullptr, m.Maxs.data()};
            if (ytgpu_scan_filter_groupby(GetGpuContext(), &kcol, &mxcol, nullptr, p, &r4, YTGPU_MEM_HOST, &err) != YTGPU_OK) ThrowFrom(err);
            m.Mins.resize(g); m.Maxs.resize(g);
        }
        m.Keys.resize(g); m.Sums.resize(g); m.KeyNulls.resize(g); m.SumNulls.resize(g);
        m.Counts.assign(c2.begin(), c2.begin() + g);
        // first row of a merged group = the smallest first row of its partial states (ordering metadata, host side)
        std::unordered_map<uint64_t, uint64_t> firstOf;
        uint64_t firstNull = UINT64_MAX;
        for (uint64_t i = 0; i < p; ++i) {
            if (KeyNulls_[i]) { firstNull = std::min(firstNull, Firsts_[i]); continue; }
            auto [it, inserted] = firstOf.emplace(Keys_[i], Firsts_[i]);
            if (!inserted) it->second = std::min(it->second, Firsts_[i]);
        }
        m.Firsts.resize(g);
        for (uint64_t i = 0; i < g; ++i) m.Firsts[i] = m.KeyNulls[i] ? firstNull : firstOf[m.Keys[i]];
        return m;
    }

private:
    uint64_t Hint_;
    bool WithMinMax_;
    uint8_t ValueType_ = YTGPU_TYPE_INT64;
    int Batches_ = 0;
    std::vector<uint64_t> Keys_, Sums_, Counts_, Firsts_, Mins_, Maxs_;
    std::vector<uint8_t> KeyNulls_, SumNulls_;
};

const TColumnarColumn& FindColumn(const std::vector<TColumnarColumn>& columns, int id) {
    for (const auto& c : columns)
        if (c.Id == id) return c;
    throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "No such column in the columnar batch");
}

}  // namespace

namespace NTableClient {

void PipeReaderToWriter(const ISchemalessMultiChunkReaderPtr& reader, const IUnversionedRowsetWriterPtr& writer,
                        const TPipeReaderToWriterOptions& options) {
    TRowBatchReadOptions readOptions;
    readOptions.MaxRowsPerRead = options.BufferRowCount;
    readOptions.MaxDataWeightPerRead = options.BufferDataWeight;
    while (auto batch = reader->Read(readOptions)) {
        if (batch->IsEmpty()) continue;  // the reference waits on reader->GetReadyEvent() here
        (void)writer->Write(batch->MaterializeRows());  // false = "wait for the writer's ready event"
    }
    writer->Close();
}

}  // namespace NTableClient

// ---- CHYT ----
namespace NClickHouseServer {

namespace {

class TGpuAggregatingSource : public IAggregatingSource {
public:
    TGpuAggregatingSource(IColumnarReaderPtr reader, int keyId, int valueId, NQueryClient::EBinaryOp op, uint64_t constant, uint64_t hint,
                          bool withMinMax)
        : Reader_(std::move(reader)), KeyId_(keyId), ValueId_(valueId), Op_(CmpOf(op)), Constant_(constant), States_(hint, withMinMax) {}

    TAggregatedChunk generate() override {
        TAggregatedChunk chunk;
        if (Finished_) return chunk;  // an empty chunk ends the stream, as in ISource
        uint64_t rowsSeen = 0;
        while (auto batch = Reader_->Read()) {
            if (batch->GetRowCount() == 0) continue;  // the reference waits on GetReadyEvent() here
            const auto& columns = batch->MaterializeColumns();
            States_.AddBatch(ViewOf(FindColumn(columns, KeyId_)), ViewOf(FindColumn(columns, ValueId_)), Op_, Constant_, rowsSeen);
            rowsSeen += (uint64_t)batch->GetRowCount();
        }
        Finished_ = true;
        auto m = States_.Merge();
        chunk.Keys = std::move(m.Keys);
        chunk.KeyNulls = std::move(m.KeyNulls);
        chunk.Sums = std::move(m.Sums);
        chunk.SumNulls = std::move(m.SumNulls);
        chunk.Counts = std::move(m.Counts);
        chunk.Mins = std::move(m.Mins);
        chunk.Maxs = std::move(m.Maxs);
        return chunk;
    }

private:
    IColumnarReaderPtr Reader_;
    int KeyId_, ValueId_, Op_;
    uint64_t Constant_;
    TPartialStates States_;
    bool Finished_ = false;
};

}  // namespace

std::unique_ptr<IAggregatingSource> CreateGpuAggregatingSource(IColumnarReaderPtr reader, int keyColumnId, int valueColumnId,
                                                               NQueryClient::EBinaryOp prewhereOp, uint64_t prewhereConstant,
                                                               uint64_t groupCountHint, bool withMinMax) {
    return std::make_unique<TGpuAggregatingSource>(std::move(reader), keyColumnId, valueColumnId, prewhereOp, prewhereConstant, groupCountHint,
                                                   withMinMax);
}

}  // namespace NClickHouseServer

// ---- YT QL ----
namespace NQueryClient {

namespace {

bool IsPredicate(EExpressionOp op) { return op >= EExpressionOp::In && op <= EExpressionOp::Like; }

// The library node of an expression node.  A String constant, and the list, prefix, needle or pattern of a predicate, are
// appended to `constants` (the call's string_constants); an In list's entries go at an 8-byte boundary, each its bit
// pattern or, for a string, (offset << 32) | length of its bytes appended before them.  *listType: the entries' one type
// (Null for an empty list); entries of several types, or a NULL one, throw.
ytgpu_expr_node LibraryNode(const TExpressionNode& node, std::string* constants, EValueType* listType) {
    ytgpu_expr_node x{};
    x.op = (int32_t)node.Op;
    x.column = node.Column;
    x.type = (uint8_t)node.Type;
    x.constant = node.Bits;
    *listType = EValueType::Null;
    auto append = [&](const std::string& bytes) {
        const uint64_t c = ((uint64_t)constants->size() << 32) | bytes.size();
        *constants += bytes;
        return c;
    };
    if ((node.Op == EExpressionOp::Constant && node.Type == EValueType::String) ||
        (IsPredicate(node.Op) && node.Op != EExpressionOp::In) || node.Op == EExpressionOp::FormatTimestamp)
        x.constant = append(node.Bytes);
    if (node.Op != EExpressionOp::In) return x;
    std::vector<uint64_t> entries;
    for (size_t e = 0; e < node.List.size(); ++e) {
        const TExpressionLiteral& v = node.List[e];
        if (v.Type == EValueType::Null) throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "in: the list holds a NULL");
        if (*listType != EValueType::Null && v.Type != *listType)
            throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "in: list entries of different types");
        *listType = v.Type;
        entries.push_back(v.Type == EValueType::String ? append(v.Bytes) : v.Bits);
    }
    constants->append((8 - constants->size() % 8) % 8, '\0');
    x.constant = ((uint64_t)constants->size() << 32) | entries.size();
    constants->append(reinterpret_cast<const char*>(entries.data()), entries.size() * 8);
    return x;
}

// Throws INVALID_ARGUMENT when the In node k of `program` has a list of another type than its operand: the operand,
// compared with a constant of the list's type, must type-check.  `typeQuery` checks a program without evaluating it (a
// BOOLEAN result: no launch) and returns its ytgpu_error code.  A malformed program is left to the call that evaluates it.
template <class F>
void CheckInList(const std::vector<ytgpu_expr_node>& program, size_t k, EValueType listType, F&& typeQuery) {
    if (listType == EValueType::Null) return;
    int need = 1;
    size_t s = k;
    while (need > 0) {
        if (s == 0) return;
        const int op = program[--s].op;
        const int arity = op == YTGPU_EXPR_COLUMN || op == YTGPU_EXPR_CONSTANT ? 0
                        : op == YTGPU_EXPR_IF ? 3
                        : op == YTGPU_EXPR_FARM_HASH ? program[s].column
                        : (op == YTGPU_EXPR_NEG || op == YTGPU_EXPR_BIT_NOT || op == YTGPU_EXPR_CAST || op == YTGPU_EXPR_LOWER ||
                           op == YTGPU_EXPR_UPPER || (op >= YTGPU_EXPR_NOT && op <= YTGPU_EXPR_IS_NOT_NULL) || op >= YTGPU_EXPR_IN) ? 1 : 2;
        need += arity - 1;
    }
    std::vector<ytgpu_expr_node> check(program.begin() + (std::ptrdiff_t)s, program.begin() + (std::ptrdiff_t)k);
    ytgpu_expr_node c{};
    c.op = YTGPU_EXPR_CONSTANT;
    c.type = (uint8_t)listType;  // a STRING constant of 0 bytes at offset 0
    check.push_back(c);
    ytgpu_expr_node cmp{};
    cmp.op = YTGPU_EXPR_COMPARE;
    cmp.column = YTGPU_CMP_EQ;
    check.push_back(cmp);
    if (typeQuery(check) != YTGPU_OK)
        throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "in: list entries of type " + std::to_string((int)listType) +
                                                              " against an operand of another type");
}

// A column the query touches, flattened once: 64-bit payloads + a null bitmap, or (strings) one heap with starts, lengths
// and a null bytemap
struct TFlatColumn {
    int Position;
    EValueType Type = EValueType::Null;
    std::vector<uint64_t> Values;
    std::vector<uint8_t> Nulls;  // bitmap
    bool AnyNull = false;
    std::string Heap;
    std::vector<uint64_t> Starts;
    std::vector<uint32_t> Lengths;
    std::vector<uint8_t> NullBytes;
    std::string_view StringAt(uint64_t row) const { return std::string_view(Heap.data() + Starts[row], Lengths[row]); }
};

// The column's first `rows` rows as a value column (an all-NULL column as INT64) or a string column.  Over zero rows the
// views carry no buffers.
ytgpu_column_view FlatView(const TFlatColumn& c, uint64_t rows) {
    ytgpu_column_view v{};
    v.value_count = (int64_t)rows;
    v.value_type = (uint8_t)(c.Type == EValueType::Null ? EValueType::Int64 : c.Type);
    v.has_values = rows > 0;
    v.bit_width = 64;
    v.values = rows > 0 ? c.Values.data() : nullptr;
    v.values_count = rows;
    v.null_bitmap = rows > 0 && c.AnyNull ? c.Nulls.data() : nullptr;
    v.mem = YTGPU_MEM_HOST;
    return v;
}

ytgpu_string_column FlatStringView(const TFlatColumn& c, uint64_t rows) {
    return ytgpu_string_column{reinterpret_cast<const uint8_t*>(c.Heap.data()), c.Heap.size(), rows > 0 ? c.Starts.data() : nullptr,
                               rows > 0 ? c.Lengths.data() : nullptr, rows > 0 ? c.NullBytes.data() : nullptr, rows, YTGPU_MEM_HOST, 0};
}

class TGpuEvaluator : public IEvaluator {
public:
    TQueryStatistics Run(const TGroupQuery& query, const ISchemalessMultiChunkReaderPtr& reader, const IUnversionedRowsetWriterPtr& writer) override {
        TQueryStatistics stats;
        TPartialStates states(0, query.WithMinMax);
        // ScanOpHelper (cg_routines/registry.cpp:315-438): read row batches; the key / value columns of a batch become two
        // 64-bit vectors + null bitmaps (what MaterializeColumns() would hand over for a columnar chunk)
        while (auto batch = reader->Read()) {
            if (batch->IsEmpty()) continue;
            const auto& rows = batch->MaterializeRows();
            const size_t n = rows.size();
            std::vector<uint64_t> keys(n), vals(n);
            std::vector<uint8_t> keyNull((n + 7) / 8, 0), valNull((n + 7) / 8, 0);
            bool anyKeyNull = false, anyValNull = false;
            for (size_t i = 0; i < n; ++i) {
                const auto& k = rows[i][query.KeyColumn];
                const auto& v = rows[i][query.ValueColumn];
                if (k.Type == EValueType::Null) { keyNull[i >> 3] |= (uint8_t)(1u << (i & 7)); anyKeyNull = true; }
                else if (k.Type == EValueType::Int64 || k.Type == EValueType::Uint64 || k.Type == EValueType::Boolean) keys[i] = k.Type == EValueType::Boolean ? (k.Data.Boolean ? 1 : 0) : k.Data.Uint64;
                else throw TErrorException(YTGPU_ERR_UNSUPPORTED, "GROUP BY key must be an integer or boolean column on the GPU path");
                if (v.Type == EValueType::Null) { valNull[i >> 3] |= (uint8_t)(1u << (i & 7)); anyValNull = true; }
                else if (v.Type == query.ValueType) vals[i] = v.Data.Uint64;
                else throw TErrorException(YTGPU_ERR_SCHEMA_VIOLATION, "Aggregated column has an unexpected value type");
            }
            auto column = [&](const std::vector<uint64_t>& data, uint8_t type, const std::vector<uint8_t>& bm, bool any) {
                ytgpu_column_view c{};
                c.value_count = (int64_t)n;
                c.value_type = type;
                c.has_values = 1;
                c.bit_width = 64;
                c.values = data.data();
                c.values_count = n;
                c.null_bitmap = any ? bm.data() : nullptr;
                c.mem = YTGPU_MEM_HOST;
                return c;
            };
            states.AddBatch(column(keys, YTGPU_TYPE_UINT64, keyNull, anyKeyNull), column(vals, (uint8_t)query.ValueType, valNull, anyValNull),
                            CmpOf(query.WhereOp), query.WhereConstant.Data.Uint64, (uint64_t)stats.RowsRead);
            stats.RowsRead += (int64_t)n;
        }
        auto m = states.Merge();
        // groups in first-seen order; ids 0..n-1, flags cleared (registry.cpp:283-291); sum(1) counts the rows of the group
        std::vector<size_t> order(m.Keys.size());
        std::iota(order.begin(), order.end(), 0);
        std::sort(order.begin(), order.end(), [&](size_t a, size_t b) { return m.Firsts[a] < m.Firsts[b]; });
        std::vector<TUnversionedOwningRow> owned;
        owned.reserve(order.size());
        for (size_t g : order) {
            TUnversionedOwningRowBuilder b;
            b.AddValue(m.KeyNulls[g] ? MakeUnversionedNullValue(0) : MakeUnversionedUint64Value(m.Keys[g], 0));
            if (m.SumNulls[g]) b.AddValue(MakeUnversionedNullValue(1));
            else if (query.ValueType == EValueType::Int64) b.AddValue(MakeUnversionedInt64Value((int64_t)m.Sums[g], 1));
            else if (query.ValueType == EValueType::Uint64) b.AddValue(MakeUnversionedUint64Value(m.Sums[g], 1));
            else { double d; std::memcpy(&d, &m.Sums[g], 8); b.AddValue(MakeUnversionedDoubleValue(d, 1)); }
            int id = 2;
            if (query.WithCount) b.AddValue(MakeUnversionedInt64Value((int64_t)m.Counts[g], id++));
            if (query.WithMinMax) {
                // min(value), max(value): Null for a group without values (udf/min.c:21-26)
                for (uint64_t bits : {m.Mins[g], m.Maxs[g]}) {
                    if (m.SumNulls[g]) b.AddValue(MakeUnversionedNullValue(id++));
                    else if (query.ValueType == EValueType::Int64) b.AddValue(MakeUnversionedInt64Value((int64_t)bits, id++));
                    else if (query.ValueType == EValueType::Uint64) b.AddValue(MakeUnversionedUint64Value(bits, id++));
                    else { double d; std::memcpy(&d, &bits, 8); b.AddValue(MakeUnversionedDoubleValue(d, id++)); }
                }
            }
            owned.push_back(b.FinishRow());
        }
        std::vector<TUnversionedRow> out(owned.begin(), owned.end());
        // WriteOpHelper hands rows over in batches (registry.cpp:2035+: RowsetProcessingBatchSize)
        constexpr size_t kBatch = 1024;
        for (size_t i = 0; i < out.size(); i += kBatch) {
            std::vector<TUnversionedRow> part(out.begin() + i, out.begin() + std::min(out.size(), i + kBatch));
            (void)writer->Write(part);  // false = "wait for GetReadyEvent()": the adapters are synchronous
        }
        writer->Close();
        stats.RowsWritten = (int64_t)out.size();
        return stats;
    }

    TQueryStatistics Run(const TMultiGroupQuery& query, const ISchemalessMultiChunkReaderPtr& reader,
                         const IUnversionedRowsetWriterPtr& writer) override {
        TQueryStatistics stats;
        const bool project = !query.Project.empty();
        if (project) {
            if (!query.GroupColumns.empty() || !query.AggregateItems.empty())
                throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "Project is the output row of a query without GROUP BY: no group or aggregate items");
            if (query.Having) throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "Having without GROUP BY");
        } else if (query.GroupColumns.empty() || query.GroupColumns.size() > 8) {
            throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "1..8 group items");
        }
        if (!query.OrderBy.empty() && !query.Limit) throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "ORDER BY used without LIMIT");
        if (query.Offset != 0 && query.OrderBy.empty()) throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "OFFSET used without ORDER BY");
        if (query.Offset < 0 || (query.Limit && *query.Limit < 0)) throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "negative OFFSET or LIMIT");
        if (query.OrderBy.size() > 32) throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "at most 32 ORDER BY items");
        // the columns the query touches, each flattened once (TFlatColumn)
        std::vector<TFlatColumn> columns;
        auto columnIndex = [&](int position) {
            for (size_t i = 0; i < columns.size(); ++i)
                if (columns[i].Position == position) return (int)i;
            columns.push_back(TFlatColumn{position});
            return (int)columns.size() - 1;
        };
        std::vector<int> keyIndex, aggIndex, byIndex;
        for (int position : query.GroupColumns) keyIndex.push_back(columnIndex(position));
        std::vector<int> projectIndex;
        for (int position : query.Project) projectIndex.push_back(columnIndex(position));
        for (const auto& item : query.AggregateItems) {
            aggIndex.push_back(columnIndex(item.Column));
            const bool arg = item.Function == EAggregateFunction::ArgMin || item.Function == EAggregateFunction::ArgMax;
            if (arg && item.ByColumn < 0) throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "argmin / argmax need two arguments");
            byIndex.push_back(arg ? columnIndex(item.ByColumn) : -1);
        }
        const int whereIndex = query.WhereOp != EBinaryOp::None ? columnIndex(query.WhereColumn) : -1;
        if (query.Where && query.WhereOp != EBinaryOp::None)
            throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "a query has either Where or WhereColumn / WhereOp");
        // with computed columns, or without GROUP BY, the WhereOp form runs as a one-node COMPARE program: the WHERE is then
        // one filter pass that comes before the computed columns it does not read (its constant gets the column's type once
        // that is known)
        std::optional<TFilterExpression> where = query.Where;
        const bool whereOpAsProgram = query.WhereOp != EBinaryOp::None &&
            (project || std::any_of(columns.begin(), columns.end(), [](const TFlatColumn& c) { return TMultiGroupQuery::IsComputedColumn(c.Position); }));
        if (whereOpAsProgram) {
            where = TFilterExpression().Compare(query.WhereColumn, query.WhereOp, query.WhereConstant);
            where->Nodes[0].Constant.Bits = query.WhereConstant.Data.Uint64;  // the built-in predicate's bits
        }
        std::vector<int> filterIndex, filterIndex2;  // flattened columns of the expression's leaves
        if (where) {
            for (const auto& node : where->Nodes) {
                const bool leaf = node.Op != EFilterOp::And && node.Op != EFilterOp::Or && node.Op != EFilterOp::Not;
                filterIndex.push_back(leaf ? columnIndex(node.Column) : -1);
                filterIndex2.push_back(node.Op == EFilterOp::CompareColumns ? columnIndex(node.Column2) : -1);
            }
        }
        // the input columns of every computed column that is named (leafIndex[j][k]: flattened column of node k, -1 for an op)
        std::vector<std::vector<int>> leafIndex(query.Computed.size());
        auto isComputed = [&](int i) { return i >= 0 && TMultiGroupQuery::IsComputedColumn(columns[i].Position); };
        for (size_t i = 0; i < columns.size(); ++i) {
            if (!isComputed((int)i)) continue;
            const size_t j = (size_t)(-2 - columns[i].Position);
            if (j >= query.Computed.size())
                throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "no computed column " + std::to_string(j));
            for (const auto& node : query.Computed[j].Nodes) {
                if (node.Op == EExpressionOp::Column && TMultiGroupQuery::IsComputedColumn(node.Column))
                    throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "a computed column reads input positions only");
                leafIndex[j].push_back(node.Op == EExpressionOp::Column ? columnIndex(node.Column) : -1);
            }
        }
        // JOIN clauses, applied left to right: Join, then NextJoins
        using TJoinClause = TMultiGroupQuery::TJoinClause;
        if (!query.Join && !query.NextJoins.empty()) throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "NextJoins without Join");
        std::vector<const TJoinClause*> joins;
        if (query.Join) joins.push_back(&*query.Join);
        for (const auto& clause : query.NextJoins) joins.push_back(&clause);
        if (joins.size() > (size_t)TMultiGroupQuery::kMaxJoinClauses)
            throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "at most " + std::to_string(TMultiGroupQuery::kMaxJoinClauses) + " join clauses");
        for (const auto& c : columns) {
            if (!TMultiGroupQuery::IsForeignColumn(c.Position)) continue;
            if (joins.empty()) throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "a foreign column without Join");
            if ((size_t)TMultiGroupQuery::ForeignClause(c.Position) >= joins.size())
                throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "a foreign column of join clause " +
                                                                      std::to_string(TMultiGroupQuery::ForeignClause(c.Position)) + ", which does not exist");
        }
        // With joins every side is a table of its own (source 0: the primary rows, source c + 1: clause c's foreign rows)
        // holding the columns something names, at their positions in that side's rows: keys, key expression leaves and the
        // columns above.  A key reference is (source, column of its table), or (-1, e) for expression e of its side's list.
        std::vector<std::vector<TFlatColumn>> tables(joins.empty() ? 0 : joins.size() + 1);
        auto tableIndex = [&](size_t s, int position) {
            for (size_t i = 0; i < tables[s].size(); ++i)
                if (tables[s][i].Position == position) return (int)i;
            tables[s].push_back(TFlatColumn{position});
            return (int)tables[s].size() - 1;
        };
        struct TKeyRef {
            int Source;
            int Index;
        };
        struct TClausePlan {
            std::vector<TKeyRef> Self, Foreign;                           // per key
            std::vector<std::vector<TKeyRef>> SelfLeaves, ForeignLeaves;  // per expression and node ({-1, -1}: an op)
        };
        std::vector<TClausePlan> plans(joins.size());
        for (size_t c = 0; c < joins.size(); ++c) {
            const TJoinClause& join = *joins[c];
            const std::string what = "join clause " + std::to_string(c);
            if (!join.Foreign) throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, what + ": no foreign reader");
            if (join.SelfColumns.empty() || join.SelfColumns.size() > YTGPU_JOIN_MAX_KEYS || join.SelfColumns.size() != join.ForeignColumns.size())
                throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, what + ": 1..8 key columns on each side, as many on both");
            auto notComputed = [&](int position) {
                if (TMultiGroupQuery::IsComputedColumn(position))
                    throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, what + ": a join key reads computed column " + std::to_string(-2 - position) +
                                                                          ", which is evaluated after WHERE");
                if (position < 0) throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, what + ": no position " + std::to_string(position));
            };
            // a self key reads a primary position or a foreign position of an earlier clause
            auto selfInput = [&](int position) {
                notComputed(position);
                if (!TMultiGroupQuery::IsForeignColumn(position)) return TKeyRef{0, tableIndex(0, position)};
                const int clause = TMultiGroupQuery::ForeignClause(position);
                if ((size_t)clause >= c)
                    throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, what + ": a self key reads the foreign columns of clause " + std::to_string(clause) +
                                                                          ", which is not joined before it");
                return TKeyRef{clause + 1, tableIndex(clause + 1, TMultiGroupQuery::ForeignIndex(position))};
            };
            // a foreign key reads a position of this clause's foreign rows
            auto foreignInput = [&](int position) {
                notComputed(position);
                if (TMultiGroupQuery::IsForeignColumn(position))
                    throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, what + ": a foreign key names a position j of the clause's foreign rows");
                return TKeyRef{(int)c + 1, tableIndex(c + 1, position)};
            };
            auto plan = [&](const std::vector<int>& positions, const std::vector<TExpression>& expressions, auto&& input, std::vector<TKeyRef>* keys,
                            std::vector<std::vector<TKeyRef>>* leaves, const char* side) {
                leaves->resize(expressions.size());
                for (int position : positions) {
                    if (!TMultiGroupQuery::IsComputedColumn(position)) {
                        keys->push_back(input(position));
                        continue;
                    }
                    const size_t e = (size_t)(-2 - position);
                    if (e >= expressions.size())
                        throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, what + ": no " + side + " key expression " + std::to_string(e));
                    keys->push_back({-1, (int)e});
                    if (!(*leaves)[e].empty()) continue;
                    for (const auto& node : expressions[e].Nodes)
                        (*leaves)[e].push_back(node.Op == EExpressionOp::Column ? input(node.Column) : TKeyRef{-1, -1});
                }
            };
            plan(join.SelfColumns, join.SelfExpressions, selfInput, &plans[c].Self, &plans[c].SelfLeaves, "self");
            plan(join.ForeignColumns, join.ForeignExpressions, foreignInput, &plans[c].Foreign, &plans[c].ForeignLeaves, "foreign");
        }
        std::vector<TKeyRef> sourceOf(columns.size(), TKeyRef{-1, -1});  // a column above: where it comes from
        for (size_t i = 0; i < columns.size() && !joins.empty(); ++i) {
            const int position = columns[i].Position;
            if (TMultiGroupQuery::IsComputedColumn(position)) continue;
            if (!TMultiGroupQuery::IsForeignColumn(position)) {
                sourceOf[i] = {0, tableIndex(0, position)};
                continue;
            }
            const int s = TMultiGroupQuery::ForeignClause(position) + 1;
            sourceOf[i] = {s, tableIndex(s, TMultiGroupQuery::ForeignIndex(position))};
        }
        // ScanOpHelper (cg_routines/registry.cpp:315-438): the columns of one side's table, row batch by row batch -> its row
        // count
        auto flatten = [&](const ISchemalessMultiChunkReaderPtr& source, std::vector<TFlatColumn>& table) {
            uint64_t sideRows = 0;
            while (auto batch = source->Read()) {
                if (batch->IsEmpty()) continue;
                const auto& rows = batch->MaterializeRows();
                for (auto& c : table) {
                    if (TMultiGroupQuery::IsComputedColumn(c.Position)) continue;
                    const int position = c.Position;
                    const size_t base = c.Values.size();
                    c.Values.resize(base + rows.size());
                    c.Nulls.resize((base + rows.size() + 7) / 8, 0);
                    c.NullBytes.resize(base + rows.size(), 0);
                    for (size_t i = 0; i < rows.size(); ++i) {
                        const auto& v = rows[i][position];
                        if (v.Type == EValueType::Null) {
                            c.Nulls[(base + i) >> 3] |= (uint8_t)(1u << ((base + i) & 7));
                            c.NullBytes[base + i] = 1;
                            c.AnyNull = true;
                            continue;
                        }
                        if (v.Type != EValueType::Int64 && v.Type != EValueType::Uint64 && v.Type != EValueType::Double && v.Type != EValueType::Boolean &&
                            v.Type != EValueType::String)
                            throw TErrorException(YTGPU_ERR_UNSUPPORTED, "GROUP BY columns must be fixed-width scalars or strings on the GPU path");
                        if (c.Type == EValueType::Null) c.Type = v.Type;
                        else if (c.Type != v.Type) throw TErrorException(YTGPU_ERR_SCHEMA_VIOLATION, "Column changes its value type");
                        if (v.Type == EValueType::String) {
                            if (c.Starts.size() < base + rows.size()) {
                                c.Starts.resize(base + rows.size(), 0);
                                c.Lengths.resize(base + rows.size(), 0);
                            }
                            c.Starts[base + i] = c.Heap.size();
                            c.Lengths[base + i] = v.Length;
                            c.Heap.append(v.Data.String, v.Length);
                            continue;
                        }
                        c.Values[base + i] = v.Type == EValueType::Boolean ? (v.Data.Boolean ? 1 : 0) : v.Data.Uint64;
                    }
                }
                sideRows += rows.size();
            }
            return sideRows;
        };
        // The result type of an expression (query.Computed[j], or a join key expression) from its program and its inputs'
        // types (leaves[k]: the column node k reads, nullptr for an op), by the typing rules of check_expression
        // (csrc/expression.cu): the value / string split below needs it before the column is evaluated.
        // An input column without a non-NULL value has no type: it is a STRING where the program reads it as one (an
        // operand of CONCAT, LOWER, UPPER, of IF_NULL or COMPARE with a STRING, or an IF branch beside one; it is passed as
        // an all-NULL string column), a BOOLEAN under AND / OR / NOT or as IF's condition, the other operand's type in a
        // COMPARE or beside an IF branch, the list's type under IN, a STRING under IsPrefix / IsSubstr / Like, INT64 everywhere
        // else, as view() passes it.  (*leafTypes)[column] records the type
        // it is read as (absent: INT64).  A malformed program types as INT64 and is refused by the call.
        using TLeafTypes = std::unordered_map<const TFlatColumn*, EValueType>;
        auto typeExpression = [&](const TExpression& expression, const std::vector<TFlatColumn*>& leaves, TLeafTypes* leafTypes) {
            struct TEntry {
                EValueType Type;
                std::vector<const TFlatColumn*> NullLeaves;  // untyped input columns the entry may be
            };
            auto asType = [&](TEntry& e, EValueType type) {
                if (e.Type != EValueType::Null || type == EValueType::Null) return;
                for (const TFlatColumn* leaf : e.NullLeaves) (*leafTypes)[leaf] = type;
                e = {type, {}};
            };
            auto asString = [&](TEntry& e) { asType(e, EValueType::String); };
            auto asNumber = [](TEntry& e) {
                if (e.Type == EValueType::Null) e.Type = EValueType::Int64;
                e.NullLeaves.clear();
            };
            std::vector<TEntry> st;
            for (size_t k = 0; k < expression.Nodes.size(); ++k) {
                const TExpressionNode& node = expression.Nodes[k];
                const size_t need = node.Op == EExpressionOp::Column || node.Op == EExpressionOp::Constant ? 0
                                  : node.Op == EExpressionOp::FarmHash ? (size_t)std::max(node.Column, 1)
                                  : node.Op == EExpressionOp::If ? 3
                                  : (node.Op == EExpressionOp::Neg || node.Op == EExpressionOp::BitNot || node.Op == EExpressionOp::Cast ||
                                     node.Op == EExpressionOp::Lower || node.Op == EExpressionOp::Upper || node.Op == EExpressionOp::Not ||
                                     node.Op == EExpressionOp::IsNull || node.Op == EExpressionOp::IsNotNull || IsPredicate(node.Op) ||
                                     node.Op == EExpressionOp::TimestampFloor || node.Op == EExpressionOp::FormatTimestamp) ? 1 : 2;
                if (st.size() < need) return EValueType::Int64;
                switch (node.Op) {
                    case EExpressionOp::Column: {
                        const TFlatColumn* leaf = leaves[k];
                        const EValueType t = leaf->Type;
                        st.push_back(t == EValueType::Null ? TEntry{EValueType::Null, {leaf}} : TEntry{t, {}});
                        break;
                    }
                    case EExpressionOp::Constant: st.push_back({node.Type, {}}); break;
                    case EExpressionOp::Lower: case EExpressionOp::Upper:
                        if (st.back().Type == EValueType::Null) asString(st.back());
                        break;
                    case EExpressionOp::Neg: case EExpressionOp::BitNot:
                        asNumber(st.back());
                        break;
                    case EExpressionOp::Cast:
                        asNumber(st.back());
                        st.back().Type = node.Type;
                        break;
                    case EExpressionOp::TimestampFloor:  // an untyped operand is an Int64
                        asNumber(st.back());
                        break;
                    case EExpressionOp::FormatTimestamp:
                        asNumber(st.back());
                        st.back().Type = EValueType::String;
                        break;
                    case EExpressionOp::FarmHash:  // a NULL hashes alike whichever type it is read as
                        st.resize(st.size() - need);
                        st.push_back({EValueType::Uint64, {}});
                        break;
                    case EExpressionOp::Not:
                        asType(st.back(), EValueType::Boolean);
                        break;
                    case EExpressionOp::IsNull: case EExpressionOp::IsNotNull:  // NULL whichever type it is read as
                        st.back() = {EValueType::Boolean, {}};
                        break;
                    case EExpressionOp::In:  // an untyped operand takes the list's type
                        for (const auto& e : node.List)
                            if (e.Type != EValueType::Null) asType(st.back(), e.Type);
                        st.back() = {EValueType::Boolean, {}};
                        break;
                    case EExpressionOp::IsPrefix: case EExpressionOp::IsSubstr: case EExpressionOp::Like:
                        asString(st.back());
                        st.back() = {EValueType::Boolean, {}};
                        break;
                    case EExpressionOp::Compare: case EExpressionOp::And: case EExpressionOp::Or: {
                        TEntry b = std::move(st.back());
                        st.pop_back();
                        TEntry& a = st.back();
                        if (node.Op != EExpressionOp::Compare) {
                            asType(a, EValueType::Boolean);
                            asType(b, EValueType::Boolean);
                        } else {
                            asType(a, b.Type);
                            asType(b, a.Type);
                        }
                        a = {EValueType::Boolean, {}};
                        break;
                    }
                    case EExpressionOp::If: {
                        TEntry b = std::move(st.back());
                        st.pop_back();
                        TEntry a = std::move(st.back());
                        st.pop_back();
                        asType(st.back(), EValueType::Boolean);
                        asType(a, b.Type);
                        asType(b, a.Type);
                        a.NullLeaves.insert(a.NullLeaves.end(), b.NullLeaves.begin(), b.NullLeaves.end());  // both untyped
                        st.back() = std::move(a);
                        break;
                    }
                    default: {  // binary ops, IfNull, Concat: operands of one type
                        TEntry b = std::move(st.back());
                        st.pop_back();
                        TEntry& a = st.back();
                        const bool str = node.Op == EExpressionOp::Concat ||
                                         (node.Op == EExpressionOp::IfNull && (a.Type == EValueType::String || b.Type == EValueType::String));
                        if (str) {
                            if (a.Type == EValueType::Null) asString(a);
                            if (b.Type == EValueType::Null) asString(b);
                        } else if (node.Op == EExpressionOp::IfNull && a.Type == EValueType::Null && b.Type == EValueType::Null) {
                            a.NullLeaves.insert(a.NullLeaves.end(), b.NullLeaves.begin(), b.NullLeaves.end());
                        } else {
                            if (a.Type == EValueType::Null) a.Type = b.Type;
                            asNumber(a);
                        }
                        break;
                    }
                }
            }
            if (st.size() != 1) return EValueType::Int64;
            return st[0].Type == EValueType::Null ? EValueType::Int64 : st[0].Type;
        };
        // An expression over `rows` rows of its input columns (leaves as typeExpression's) into `c`: one
        // ytgpu_evaluate_expression_strings call (string inputs as string columns), rows outside `selection` NULL; a string
        // result takes a second call once its heap is sized
        auto evaluateExpression = [&](const TExpression& expression, const std::vector<TFlatColumn*>& leaves, uint64_t rows,
                                      const uint8_t* selection, TFlatColumn& c) {
            std::vector<ytgpu_column_view> inputs;
            std::vector<ytgpu_string_column> stringInputs;
            std::string constants;
            std::unordered_map<const TFlatColumn*, int> slot;  // scalar: slot; string: -2 - string slot
            std::vector<ytgpu_expr_node> program;
            TLeafTypes leafTypes;  // the types untyped input columns are read as
            typeExpression(expression, leaves, &leafTypes);
            std::vector<std::pair<size_t, EValueType>> inLists;  // In nodes and their lists' types
            for (size_t k = 0; k < expression.Nodes.size(); ++k) {
                const TExpressionNode& node = expression.Nodes[k];
                EValueType listType;
                ytgpu_expr_node x = LibraryNode(node, &constants, &listType);
                if (node.Op == EExpressionOp::In) inLists.push_back({k, listType});
                TFlatColumn* leaf = leaves[k];
                if (leaf && !slot.count(leaf)) {
                    const auto readAs = leafTypes.find(leaf);
                    const EValueType leafType = readAs == leafTypes.end() ? EValueType::Null : readAs->second;
                    if (leaf->Type == EValueType::String || leafType == EValueType::String) {  // all-NULL: an empty heap
                        leaf->Starts.resize(rows, 0);
                        leaf->Lengths.resize(rows, 0);
                        slot[leaf] = -2 - (int)stringInputs.size();
                        stringInputs.push_back(FlatStringView(*leaf, rows));
                    } else {
                        slot[leaf] = (int)inputs.size();
                        inputs.push_back(FlatView(*leaf, rows));
                        if (leaf->Type == EValueType::Null && leafType != EValueType::Null)
                            inputs.back().value_type = (uint8_t)leafType;  // all-NULL, read as the program reads it
                    }
                }
                program.push_back(x);
            }
            for (size_t k = 0; k < program.size(); ++k)  // string inputs follow the scalar ones
                if (const TFlatColumn* leaf = leaves[k]) {
                    const int s = slot[leaf];
                    program[k].column = s >= 0 ? s : (int)inputs.size() + (-2 - s);
                }
            if (inputs.empty() && stringInputs.empty()) {  // constants only: a column without values gives the row count
                ytgpu_column_view count{};
                count.value_count = (int64_t)rows;
                count.value_type = YTGPU_TYPE_INT64;
                count.bit_width = 64;
                count.mem = YTGPU_MEM_HOST;
                inputs.push_back(count);
            }
            for (const auto& [k, listType] : inLists)
                CheckInList(program, k, listType, [&](const std::vector<ytgpu_expr_node>& check) {
                    ytgpu_error qerr{};
                    uint64_t heapBytes = 0;
                    return ytgpu_evaluate_expression_strings(
                        GetGpuContext(), inputs.data(), (uint32_t)inputs.size(), stringInputs.data(), (uint32_t)stringInputs.size(),
                        reinterpret_cast<const uint8_t*>(constants.data()), constants.size(), check.data(), (uint32_t)check.size(),
                        nullptr, nullptr, nullptr, nullptr, 0, nullptr, nullptr, nullptr, &heapBytes, nullptr, nullptr, YTGPU_MEM_HOST, &qerr);
                });
            c.Values.assign(rows, 0);
            c.Nulls.assign((rows + 63) / 64 * 8, 0);
            uint8_t type = 0;
            uint64_t nullCount = 0, heapBytes = 0;
            ytgpu_error err{};
            auto call = [&](bool fill) {
                if (ytgpu_evaluate_expression_strings(
                        GetGpuContext(), inputs.data(), (uint32_t)inputs.size(), stringInputs.data(), (uint32_t)stringInputs.size(),
                        reinterpret_cast<const uint8_t*>(constants.data()), constants.size(), program.data(), (uint32_t)program.size(),
                        selection, c.Values.data(), c.Nulls.data(), fill ? reinterpret_cast<uint8_t*>(c.Heap.data()) : nullptr,
                        c.Heap.size(), c.Starts.data(), c.Lengths.data(), c.NullBytes.data(), &heapBytes, &type, &nullCount,
                        YTGPU_MEM_HOST, &err) != YTGPU_OK)
                    ThrowFrom(err);
            };
            call(false);  // a numeric result is complete; a string result has its heap size
            c.Type = (EValueType)type;
            c.AnyNull = nullCount != 0;
            if (c.Type == EValueType::String) {
                c.Heap.assign(heapBytes, '\0');
                c.Starts.assign(rows, 0);
                c.Lengths.assign(rows, 0);
                c.NullBytes.assign(rows, 0);
                call(true);
                for (uint64_t r = 0; r < rows; ++r)  // a string GROUP BY key's NULLs are the ids' null bitmap (view())
                    if (c.NullBytes[r]) c.Nulls[r >> 3] |= (uint8_t)(1u << (r & 7));
            }
        };
        auto computedLeaves = [&](size_t j) {
            std::vector<TFlatColumn*> leaves;
            for (int leaf : leafIndex[j]) leaves.push_back(leaf >= 0 ? &columns[leaf] : nullptr);
            return leaves;
        };
        uint64_t n = 0;
        if (joins.empty()) {
            stats.RowsRead = (int64_t)flatten(reader, columns);
            n = (uint64_t)stats.RowsRead;
        } else {
            // The joined rows, clause by clause.  maps[s] holds source s's row at every joined row (YTGPU_JOIN_NO_ROW where a
            // LEFT clause found no match); only the key inputs of each clause are gathered at the current joined rows, and
            // every column above once, after the last clause.
            auto keyView = [](const TFlatColumn& c, const uint64_t* values, uint64_t rows, EValueType type) {
                ytgpu_column_view v{};
                v.value_count = (int64_t)rows;
                v.value_type = (uint8_t)type;
                v.has_values = 1;
                v.bit_width = 64;
                v.values = values;
                v.values_count = rows;
                v.null_bitmap = c.AnyNull ? c.Nulls.data() : nullptr;
                v.mem = YTGPU_MEM_HOST;
                return v;
            };
            // column `c` of a side's table at `rows` of that side (NO_ROW: NULL); a string column's gather takes `heap`, the
            // column's heap or a copy of it
            auto gatherFlat = [&](TFlatColumn& c, const std::vector<uint32_t>& rows, std::string heap) {
                const uint64_t sideRows = c.Values.size(), count = rows.size();
                TFlatColumn g{c.Position, c.Type};
                ytgpu_error err{};
                if (c.Type == EValueType::String) {
                    c.Starts.resize(sideRows, 0);
                    c.Lengths.resize(sideRows, 0);
                    const ytgpu_string_column source{reinterpret_cast<const uint8_t*>(heap.data()), heap.size(), c.Starts.data(),
                                                     c.Lengths.data(), c.NullBytes.data(), sideRows, YTGPU_MEM_HOST, 0};
                    g.Starts.resize(count);
                    g.Lengths.resize(count);
                    g.NullBytes.resize(count);
                    if (ytgpu_gather_string_column(GetGpuContext(), &source, rows.data(), count, g.Starts.data(), g.Lengths.data(),
                                                   g.NullBytes.data(), YTGPU_MEM_HOST, &err) != YTGPU_OK)
                        ThrowFrom(err);
                    g.Nulls.assign((count + 63) / 64 * 8, 0);
                    for (uint64_t r = 0; r < count; ++r)
                        if (g.NullBytes[r]) {
                            g.Nulls[r >> 3] |= (uint8_t)(1u << (r & 7));
                            g.AnyNull = true;
                        }
                    g.Values.assign(count, 0);
                    g.Heap = std::move(heap);
                    return g;
                }
                const ytgpu_column_view source = keyView(c, c.Values.data(), sideRows, c.Type == EValueType::Null ? EValueType::Int64 : c.Type);
                g.Values.resize(count);
                g.Nulls.resize((count + 63) / 64 * 8);
                uint64_t nullCount = 0;
                if (ytgpu_gather_column(GetGpuContext(), &source, rows.data(), count, g.Values.data(), g.Nulls.data(), &nullCount, YTGPU_MEM_HOST,
                                        &err) != YTGPU_OK)
                    ThrowFrom(err);
                g.AnyNull = nullCount != 0;
                g.NullBytes.assign(count, 0);
                for (uint64_t r = 0; r < count; ++r) g.NullBytes[r] = (g.Nulls[r >> 3] >> (r & 7)) & 1;
                return g;
            };
            stats.RowsRead = (int64_t)flatten(reader, tables[0]);
            n = (uint64_t)stats.RowsRead;
            std::vector<std::vector<uint32_t>> maps(joins.size() + 1);
            for (size_t c = 0; c < joins.size(); ++c) {
                const TJoinClause& join = *joins[c];
                const TClausePlan& plan = plans[c];
                const std::string what = "join clause " + std::to_string(c);
                const uint64_t np = n, nf = flatten(join.Foreign, tables[c + 1]);
                // the self key inputs at the current joined rows: clause 0 reads the primary columns themselves
                std::map<std::pair<int, int>, TFlatColumn> gathered;
                auto input = [&](TKeyRef r) {
                    TFlatColumn& source = tables[r.Source][r.Index];
                    if (c == 0 || r.Source == (int)c + 1) return &source;
                    auto [it, inserted] = gathered.try_emplace({r.Source, r.Index}, TFlatColumn{source.Position});
                    if (inserted) it->second = gatherFlat(source, maps[r.Source], source.Heap);
                    return &it->second;
                };
                // each key expression named, evaluated once over its side's rows
                std::map<std::pair<bool, int>, TFlatColumn> evaluated;
                auto keyColumn = [&](TKeyRef r, bool self) {
                    if (r.Source >= 0) return input(r);
                    auto [it, inserted] = evaluated.try_emplace({self, r.Index}, TFlatColumn{-1});
                    if (inserted) {
                        std::vector<TFlatColumn*> leaves;
                        for (TKeyRef leaf : (self ? plan.SelfLeaves : plan.ForeignLeaves)[r.Index]) leaves.push_back(leaf.Source >= 0 ? input(leaf) : nullptr);
                        evaluateExpression((self ? join.SelfExpressions : join.ForeignExpressions)[r.Index], leaves, self ? np : nf, nullptr, it->second);
                    }
                    return &it->second;
                };
                const size_t keyCount = plan.Self.size();
                std::vector<ytgpu_column_view> primaryKeys, foreignKeys;
                std::vector<std::vector<uint64_t>> stringIds(keyCount);
                for (size_t k = 0; k < keyCount; ++k) {
                    const TFlatColumn& p = *keyColumn(plan.Self[k], true);
                    const TFlatColumn& f = *keyColumn(plan.Foreign[k], false);
                    if (p.Type != EValueType::Null && f.Type != EValueType::Null && p.Type != f.Type)
                        throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, what + ", key " + std::to_string(k) +
                                                                              ": the primary and foreign keys differ in type (cast first)");
                    const EValueType type = p.Type != EValueType::Null ? p.Type : f.Type != EValueType::Null ? f.Type : EValueType::Int64;
                    if (type != EValueType::String) {
                        primaryKeys.push_back(keyView(p, p.Values.data(), np, type));
                        foreignKeys.push_back(keyView(f, f.Values.data(), nf, type));
                        continue;
                    }
                    // one ytgpu_string_value_ids call over the foreign values followed by the primary ones: equal strings on
                    // either side get the same id
                    std::string heap = f.Heap + p.Heap;
                    std::vector<uint64_t> starts(nf + np, 0);
                    std::vector<uint32_t> lengths(nf + np, 0);
                    std::vector<uint8_t> nulls(f.NullBytes.begin(), f.NullBytes.end());
                    nulls.insert(nulls.end(), p.NullBytes.begin(), p.NullBytes.end());
                    for (uint64_t r = 0; r < f.Starts.size(); ++r) { starts[r] = f.Starts[r]; lengths[r] = f.Lengths[r]; }
                    for (uint64_t r = 0; r < p.Starts.size(); ++r) { starts[nf + r] = f.Heap.size() + p.Starts[r]; lengths[nf + r] = p.Lengths[r]; }
                    stringIds[k].assign(nf + np, 0);
                    ytgpu_error err{};
                    if (ytgpu_string_value_ids(GetGpuContext(), reinterpret_cast<const uint8_t*>(heap.data()), heap.size(), starts.data(), lengths.data(),
                                               nulls.data(), nf + np, stringIds[k].data(), nullptr, YTGPU_MEM_HOST, &err) != YTGPU_OK)
                        ThrowFrom(err);
                    primaryKeys.push_back(keyView(p, stringIds[k].data() + nf, np, EValueType::Uint64));
                    foreignKeys.push_back(keyView(f, stringIds[k].data(), nf, EValueType::Uint64));
                }
                const int kind = join.IsLeft ? YTGPU_JOIN_LEFT : YTGPU_JOIN_INNER;
                uint64_t pairs = 0;
                ytgpu_error err{};
                if (ytgpu_hash_join(GetGpuContext(), primaryKeys.data(), foreignKeys.data(), (uint32_t)keyCount, kind, nullptr, nullptr, 0, &pairs,
                                    YTGPU_MEM_HOST, &err) != YTGPU_OK)
                    ThrowFrom(err);
                // the joined rows are the next clause's primary side and the input of GROUP BY / ORDER BY: fewer than 2^30
                if (pairs >= (1ull << 30))
                    throw TErrorException(YTGPU_ERR_UNSUPPORTED, what + ": " + std::to_string(pairs) + " joined rows, at most 2^30 - 1 on the GPU path");
                std::vector<uint32_t> primaryRows(pairs), foreignRows(pairs);
                if (ytgpu_hash_join(GetGpuContext(), primaryKeys.data(), foreignKeys.data(), (uint32_t)keyCount, kind, primaryRows.data(),
                                    foreignRows.data(), pairs, &pairs, YTGPU_MEM_HOST, &err) != YTGPU_OK)
                    ThrowFrom(err);
                // compose: map_s <- map_s[primaryRows], a gather of the map as a UINT64 column (primaryRows never holds
                // NO_ROW, so a NO_ROW in the map carries through as a value)
                for (size_t s = 0; c > 0 && s <= c; ++s) {
                    const std::vector<uint64_t> wide(maps[s].begin(), maps[s].end());
                    ytgpu_column_view source{};
                    source.value_count = (int64_t)wide.size();
                    source.value_type = YTGPU_TYPE_UINT64;
                    source.has_values = 1;
                    source.bit_width = 64;
                    source.values = wide.data();
                    source.values_count = wide.size();
                    source.mem = YTGPU_MEM_HOST;
                    std::vector<uint64_t> composed(pairs);
                    std::vector<uint8_t> nulls((pairs + 63) / 64 * 8);
                    if (ytgpu_gather_column(GetGpuContext(), &source, primaryRows.data(), pairs, composed.data(), nulls.data(), nullptr,
                                            YTGPU_MEM_HOST, &err) != YTGPU_OK)
                        ThrowFrom(err);
                    maps[s].assign(composed.begin(), composed.end());
                }
                if (c == 0) maps[0] = std::move(primaryRows);
                maps[c + 1] = std::move(foreignRows);
                n = pairs;
            }
            // every column above, once, from its side's table through that side's map
            for (size_t i = 0; i < columns.size(); ++i) {
                if (sourceOf[i].Source < 0) continue;
                TFlatColumn& source = tables[sourceOf[i].Source][sourceOf[i].Index];
                const int position = columns[i].Position;
                columns[i] = gatherFlat(source, maps[sourceOf[i].Source], std::move(source.Heap));
                columns[i].Position = position;
            }
        }
        for (size_t i = 0; i < columns.size(); ++i) {
            if (!isComputed((int)i)) continue;
            TLeafTypes leafTypes;
            const size_t j = (size_t)(-2 - columns[i].Position);
            columns[i].Type = typeExpression(query.Computed[j], computedLeaves(j), &leafTypes);
        }
        if (whereIndex >= 0 && columns[whereIndex].Type == EValueType::String)
            throw TErrorException(YTGPU_ERR_UNSUPPORTED, "the WHERE column (position " + std::to_string(query.WhereColumn) +
                                                             ") holds strings: string predicates are not on the GPU path");
        for (size_t a = 0; a < query.AggregateItems.size(); ++a) {
            const auto f = query.AggregateItems[a].Function;
            if ((f == EAggregateFunction::Sum || f == EAggregateFunction::Avg) && columns[aggIndex[a]].Type == EValueType::String)
                throw TErrorException(YTGPU_ERR_UNSUPPORTED, "sum / avg of a string column");
        }
        std::vector<TUnversionedOwningRow> owned;
        // a program over output positions; the string functions and string predicates are not taken there
        struct TOutputProgram {
            std::vector<ytgpu_expr_node> Nodes;
            std::string Constants;  // In lists
            std::vector<std::pair<size_t, EValueType>> InLists;
        };
        auto outputProgram = [&](const TExpression& e, const std::string& what) {
            TOutputProgram program;
            for (const auto& node : e.Nodes) {
                if (node.Op == EExpressionOp::Concat || node.Op == EExpressionOp::Lower || node.Op == EExpressionOp::Upper ||
                    node.Op == EExpressionOp::FarmHash || node.Op == EExpressionOp::IsPrefix || node.Op == EExpressionOp::IsSubstr ||
                    node.Op == EExpressionOp::Like || node.Op == EExpressionOp::FormatTimestamp)
                    throw TErrorException(YTGPU_ERR_UNSUPPORTED, what + ": string functions over the output row");
                EValueType listType;
                if (node.Op == EExpressionOp::In) {
                    for (const auto& v : node.List)
                        if (v.Type == EValueType::String)
                            throw TErrorException(YTGPU_ERR_UNSUPPORTED, what + ": string functions over the output row");
                }
                program.Nodes.push_back(LibraryNode(node, &program.Constants, &listType));
                if (node.Op == EExpressionOp::In) program.InLists.push_back({program.Nodes.size() - 1, listType});
            }
            return program;
        };
        // One call over the output row's views: ytgpu_evaluate_expression, or with In the string entry point without string
        // columns (it takes the lists in string_constants).
        auto evaluateOutput = [&](const TOutputProgram& program, const std::vector<ytgpu_column_view>& views, const uint8_t* selection,
                                  uint64_t* values, uint64_t* nulls, uint8_t* type) {
            ytgpu_error oerr{};
            int code;
            if (program.InLists.empty()) {
                code = ytgpu_evaluate_expression(GetGpuContext(), views.data(), (uint32_t)views.size(), program.Nodes.data(),
                                                 (uint32_t)program.Nodes.size(), selection, values, reinterpret_cast<uint8_t*>(nulls), type,
                                                 nullptr, YTGPU_MEM_HOST, &oerr);
            } else {
                auto call = [&](const std::vector<ytgpu_expr_node>& nodes, uint64_t* v, uint64_t* nb, uint8_t* t, ytgpu_error* e) {
                    uint64_t heapBytes = 0;
                    return ytgpu_evaluate_expression_strings(
                        GetGpuContext(), views.data(), (uint32_t)views.size(), nullptr, 0,
                        reinterpret_cast<const uint8_t*>(program.Constants.data()), program.Constants.size(), nodes.data(),
                        (uint32_t)nodes.size(), selection, v, reinterpret_cast<uint8_t*>(nb), nullptr, 0, nullptr, nullptr, nullptr,
                        &heapBytes, t, nullptr, YTGPU_MEM_HOST, e);
                };
                for (const auto& [k, listType] : program.InLists)
                    CheckInList(program.Nodes, k, listType, [&](const std::vector<ytgpu_expr_node>& check) {
                        ytgpu_error qerr{};
                        return call(check, nullptr, nullptr, nullptr, &qerr);
                    });
                const bool empty = views.empty() || views[0].value_count == 0;
                code = call(program.Nodes, empty ? nullptr : values, empty ? nullptr : nulls, type, &oerr);
            }
            if (code != YTGPU_OK) ThrowFrom(oerr);
        };
        // Having over the output row's views (`groups` rows each) -> its TRUE rows as a selection bitmap in the layout of
        // ytgpu_evaluate_filter's out_bitmap (ceil(groups / 64) words).  With no groups the call only checks the program:
        // a Having that is not a Boolean, or reads a string position, is refused whatever the data.
        auto evaluateHaving = [&](const std::vector<ytgpu_column_view>& views, uint64_t groups) {
            const auto program = outputProgram(*query.Having, "having");
            std::vector<uint64_t> values(groups), nulls((groups + 63) / 64), kept((groups + 63) / 64, 0);
            uint8_t type = 0;
            evaluateOutput(program, views, nullptr, values.data(), nulls.data(), &type);
            if (type != (uint8_t)EValueType::Boolean)
                throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "having: the expression is not a Boolean");
            for (uint64_t g = 0; g < groups; ++g)
                if (values[g] == 1 && !((nulls[g >> 6] >> (g & 63)) & 1)) kept[g >> 6] |= 1ull << (g & 63);
            return kept;
        };
        // ORDER BY, OFFSET and LIMIT over the output row -> the rows written, in order.  `views` are the output row's positions
        // (rowCount rows each; a string position's view has value_type STRING), strings[p] position p as a flat string column
        // when it holds strings, `selection` the rows WHERE / HAVING keep and `kept` their list (nullptr: every row).  The items
        // are evaluated over the kept rows only; one ytgpu_order_rows call orders the kept rows and cuts the window.  Without
        // ORDER BY the window is the first Limit kept rows.  With an empty window the items are checked over zero rows, so a
        // malformed item is refused whatever the data.
        auto orderWindow = [&](const std::vector<ytgpu_column_view>& views, const std::vector<std::optional<ytgpu_string_column>>& strings,
                               const uint8_t* selection, const std::vector<uint32_t>* kept, uint64_t rowCount) {
            const uint64_t candidates = kept ? kept->size() : rowCount;
            const uint64_t offset = (uint64_t)query.Offset, limit = query.Limit ? (uint64_t)*query.Limit : candidates;
            const uint64_t count = std::min(limit, candidates - std::min(offset, candidates));
            std::vector<uint32_t> window(count);
            if (query.OrderBy.empty()) {
                for (uint64_t i = 0; i < count; ++i) window[i] = kept ? (*kept)[i] : (uint32_t)i;
                return window;
            }
            std::vector<ytgpu_column_view> none;  // the views over zero rows
            if (count == 0) {
                none = views;
                for (auto& v : none) {
                    v.value_count = 0;
                    v.values_count = 0;
                    v.has_values = 0;
                    v.values = nullptr;
                    v.null_bitmap = nullptr;
                }
                rowCount = 0;
                selection = nullptr;
            }
            const auto& itemViews = count == 0 ? none : views;
            std::vector<ytgpu_column_view> orderColumns;
            std::vector<ytgpu_string_column> orderStrings;
            std::vector<ytgpu_order_item> items;
            std::vector<std::vector<uint64_t>> values, nulls;  // the evaluated items
            values.reserve(query.OrderBy.size());
            nulls.reserve(query.OrderBy.size());
            for (size_t i = 0; i < query.OrderBy.size(); ++i) {
                const auto& item = query.OrderBy[i];
                const uint8_t descending = item.Descending ? 1 : 0;
                const auto& nodes = item.Expression.Nodes;
                if (nodes.size() == 1 && nodes[0].Op == EExpressionOp::Column) {
                    const int p = nodes[0].Column;
                    if (p < 0 || (size_t)p >= views.size())
                        throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "order by item " + std::to_string(i) + ": no output position " + std::to_string(p));
                    if (strings[p]) {
                        items.push_back({(uint32_t)orderStrings.size(), 1, descending, 0});
                        orderStrings.push_back(*strings[p]);
                    } else {
                        items.push_back({(uint32_t)orderColumns.size(), 0, descending, 0});
                        orderColumns.push_back(itemViews[p]);
                    }
                    continue;
                }
                const auto program = outputProgram(item.Expression, "order by item " + std::to_string(i));
                values.emplace_back(rowCount);
                nulls.emplace_back((rowCount + 63) / 64);
                uint8_t type = 0;
                evaluateOutput(program, itemViews, selection, values.back().data(), nulls.back().data(), &type);
                ytgpu_column_view v{};
                v.value_count = (int64_t)rowCount;
                v.value_type = type;
                v.has_values = 1;
                v.bit_width = 64;
                v.values = values.back().data();
                v.values_count = rowCount;
                v.null_bitmap = reinterpret_cast<const uint8_t*>(nulls.back().data());
                v.mem = YTGPU_MEM_HOST;
                items.push_back({(uint32_t)orderColumns.size(), 0, descending, 0});
                orderColumns.push_back(v);
            }
            if (count == 0) return window;
            uint64_t got = 0;
            ytgpu_error err{};
            if (ytgpu_order_rows(GetGpuContext(), orderColumns.data(), (uint32_t)orderColumns.size(), orderStrings.data(), (uint32_t)orderStrings.size(),
                                 items.data(), (uint32_t)items.size(), kept ? kept->data() : nullptr, candidates, offset, limit, window.data(), &got,
                                 YTGPU_MEM_HOST, &err) != YTGPU_OK)
                ThrowFrom(err);
            return window;
        };
        // a string result (and a string key) is the index of a row that holds it
        auto make = [&](const TFlatColumn* strings, EValueType type, uint64_t bits, bool null, int id) {
            if (null) return MakeUnversionedNullValue(id);
            if (strings) return MakeUnversionedStringValue(strings->StringAt(bits), id);
            switch (type) {
                case EValueType::Uint64: return MakeUnversionedUint64Value(bits, id);
                case EValueType::Double: { double d; std::memcpy(&d, &bits, 8); return MakeUnversionedDoubleValue(d, id); }
                case EValueType::Boolean: return MakeUnversionedBooleanValue(bits != 0, id);
                default: return MakeUnversionedInt64Value((int64_t)bits, id);
            }
        };
        // the output row's positions
        struct TOutput {
            EValueType Type;
            const TFlatColumn* Strings;
            const uint64_t* Values;
            const uint8_t* Null;  // bytemap
        };
        // Select over the output row's positions (`rows` rows each) -> the written row's positions.  A bare Column passes its
        // position through; every other item is one ytgpu_evaluate_expression call over the views (a string position is
        // refused by the call as UNSUPPORTED), over `selection` only.  selectValues / selectNulls hold the results.
        std::vector<std::vector<uint64_t>> selectValues, selectNulls;  // selectNulls: null bitmaps
        auto evaluateSelect = [&](const std::vector<TOutput>& outputs, const std::vector<ytgpu_column_view>& outViews, const uint8_t* selection,
                                  uint64_t rows) {
            std::vector<TOutput> selected;
            selectValues.assign(query.Select->size(), {});
            selectNulls.assign(query.Select->size(), {});
            for (size_t s = 0; s < query.Select->size(); ++s) {
                const auto& nodes = (*query.Select)[s].Nodes;
                if (nodes.size() == 1 && nodes[0].Op == EExpressionOp::Column) {
                    if (nodes[0].Column < 0 || (size_t)nodes[0].Column >= outputs.size())
                        throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "select item " + std::to_string(s) + ": no output position " +
                                                                              std::to_string(nodes[0].Column));
                    selected.push_back(outputs[nodes[0].Column]);
                    continue;
                }
                const auto program = outputProgram((*query.Select)[s], "select item " + std::to_string(s));
                selectValues[s].assign(rows, 0);
                selectNulls[s].assign((rows + 63) / 64, 0);
                uint8_t type = 0;
                evaluateOutput(program, outViews, selection, selectValues[s].data(), selectNulls[s].data(), &type);
                selected.push_back({(EValueType)type, nullptr, selectValues[s].data(), nullptr});
            }
            return selected;
        };
        auto writeRow = [&](const std::vector<TOutput>& selected, uint64_t g) {
            TUnversionedOwningRowBuilder b;
            for (size_t s = 0; s < selected.size(); ++s) {
                const TOutput& o = selected[s];
                const bool null = o.Null ? o.Null[g] != 0 : ((selectNulls[s][g >> 6] >> (g & 63)) & 1) != 0;
                b.AddValue(make(o.Strings, o.Type, o.Values[g], null, (int)s));
            }
            owned.push_back(b.FinishRow());
        };
        if (n == 0 && query.Having) {  // no rows, no groups: the output row's types from the columns' (NULL: INT64)
            std::vector<ytgpu_column_view> views;
            auto add = [&](EValueType type) {
                ytgpu_column_view v{};
                v.value_type = (uint8_t)(type == EValueType::Null ? EValueType::Int64 : type);
                v.bit_width = 64;
                v.mem = YTGPU_MEM_HOST;
                views.push_back(v);
            };
            for (int k : keyIndex) add(columns[k].Type);
            for (size_t a = 0; a < query.AggregateItems.size(); ++a) {
                const auto f = query.AggregateItems[a].Function;
                add(f == EAggregateFunction::Count ? EValueType::Int64 : f == EAggregateFunction::Avg ? EValueType::Double : columns[aggIndex[a]].Type);
            }
            evaluateHaving(views, 0);
        }
        if (n == 0 && project) {  // no rows: ORDER BY and Select are still checked, over zero-row views of the output row
            std::vector<ytgpu_column_view> views;
            std::vector<std::optional<ytgpu_string_column>> strings;
            std::vector<TOutput> outputs;
            for (int i : projectIndex) {
                const TFlatColumn& c = columns[i];
                const bool str = c.Type == EValueType::String;
                ytgpu_column_view v{};
                v.value_type = (uint8_t)(str ? EValueType::String : c.Type == EValueType::Null ? EValueType::Int64 : c.Type);
                v.bit_width = 64;
                v.mem = YTGPU_MEM_HOST;
                views.push_back(v);
                strings.push_back(str ? std::optional(ytgpu_string_column{nullptr, 0, nullptr, nullptr, nullptr, 0, YTGPU_MEM_HOST, 0}) : std::nullopt);
                outputs.push_back({c.Type, str ? &c : nullptr, nullptr, nullptr});
            }
            orderWindow(views, strings, nullptr, nullptr, 0);
            if (query.Select) evaluateSelect(outputs, views, nullptr, 0);
        }
        if (n > 0) {
            auto view = [&](const TFlatColumn& c) { return FlatView(c, n); };
            auto stringView = [&](const TFlatColumn& c) { return FlatStringView(c, n); };
            // a computed column over every row, those outside `selection` NULL
            auto evaluateComputed = [&](int i, const uint8_t* selection) {
                const size_t j = (size_t)(-2 - columns[i].Position);
                evaluateExpression(query.Computed[j], computedLeaves(j), n, selection, columns[i]);
            };
            // the computed columns the WHERE reads, over all rows
            std::vector<uint8_t> evaluated(columns.size(), 0);
            for (const auto* leaves : {&filterIndex, &filterIndex2})
                for (int i : *leaves)
                    if (isComputed(i) && !evaluated[i]) {
                        evaluateComputed(i, nullptr);
                        evaluated[i] = 1;
                    }
            if (whereOpAsProgram) where->Nodes[0].Constant.Type = columns[filterIndex[0]].Type;
            // scalar columns are value columns, string columns follow them as string columns of the call
            std::vector<int> argIndex(columns.size());
            std::vector<ytgpu_column_view> keyViews, valueViews;
            std::vector<ytgpu_string_column> stringViews;
            for (auto& c : columns) {
                if (c.Type != EValueType::String) continue;
                c.Starts.resize(n, 0);
                c.Lengths.resize(n, 0);
                stringViews.push_back(ytgpu_string_column{reinterpret_cast<const uint8_t*>(c.Heap.data()), c.Heap.size(), c.Starts.data(),
                                                          c.Lengths.data(), c.NullBytes.data(), n, YTGPU_MEM_HOST, 0});
            }
            for (size_t i = 0, s = 0; i < columns.size(); ++i) {
                if (columns[i].Type == EValueType::String) {
                    argIndex[i] = -1 - (int)s++;
                } else {
                    argIndex[i] = (int)valueViews.size();
                    valueViews.push_back(view(columns[i]));
                }
            }
            int predicateColumn = whereIndex;
            std::vector<uint8_t> selection;  // the WHERE expression's bitmap: one more BOOLEAN value column
            if (where) {
                const int scalarCount = (int)valueViews.size();
                auto callIndex = [&](int i) { return argIndex[i] >= 0 ? argIndex[i] : scalarCount + (-1 - argIndex[i]); };
                std::vector<ytgpu_filter_node> program;
                std::vector<uint64_t> lists;
                std::string constants;
                auto addString = [&](const std::string& b) {
                    const uint64_t off = constants.size();
                    constants += b;
                    return off;
                };
                for (size_t k = 0; k < where->Nodes.size(); ++k) {
                    const TFilterNode& node = where->Nodes[k];
                    ytgpu_filter_node f{(int32_t)node.Op, 0, -1, -1, 0, 0, 0};
                    if (filterIndex[k] < 0) {
                        program.push_back(f);
                        continue;
                    }
                    const TFlatColumn& c = columns[filterIndex[k]];
                    f.column = callIndex(filterIndex[k]);
                    const bool noValues = c.Type == EValueType::Null ||
                                          (node.Op == EFilterOp::CompareColumns && columns[filterIndex2[k]].Type == EValueType::Null);
                    auto typed = [&](const TFilterConstant& v) {
                        if (v.Type != c.Type)
                            throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "WHERE node " + std::to_string(k) + ": the constant's type differs from column " +
                                                                                  std::to_string(node.Column) + "'s");
                    };
                    if (noValues && node.Op != EFilterOp::IsNull && node.Op != EFilterOp::IsNotNull) {
                        // a column without a value: every comparison, IN and prefix test is NULL, as COMPARE over it is
                        f.op = YTGPU_FILTER_COMPARE;
                        f.cmp = YTGPU_CMP_EQ;
                        f.column = callIndex(c.Type == EValueType::Null ? filterIndex[k] : filterIndex2[k]);
                        program.push_back(f);
                        continue;
                    }
                    switch (node.Op) {
                        case EFilterOp::Compare:
                            typed(node.Constant);
                            f.cmp = CmpOf(node.Cmp);
                            if (c.Type == EValueType::String) {
                                f.constant = addString(node.Constant.Bytes);
                                f.length = (uint32_t)node.Constant.Bytes.size();
                            } else {
                                f.constant = node.Constant.Bits;
                            }
                            break;
                        case EFilterOp::CompareColumns:
                            f.cmp = CmpOf(node.Cmp);
                            f.column2 = callIndex(filterIndex2[k]);
                            break;
                        case EFilterOp::StartsWith:
                        case EFilterOp::Contains:
                        case EFilterOp::Like:
                            typed(node.Constant);
                            f.constant = addString(node.Constant.Bytes);
                            f.length = (uint32_t)node.Constant.Bytes.size();
                            if (node.Op == EFilterOp::Like) f.column2 = node.Escape;
                            break;
                        case EFilterOp::In:
                            f.constant = lists.size();
                            f.length = (uint32_t)node.List.size();
                            for (const auto& v : node.List) {
                                typed(v);
                                lists.push_back(c.Type == EValueType::String ? (addString(v.Bytes) << 32) | v.Bytes.size() : v.Bits);
                            }
                            break;
                        default:
                            break;
                    }
                    program.push_back(f);
                }
                selection.assign((n + 63) / 64 * 8, 0);
                uint64_t selected = 0;
                ytgpu_error err{};
                if (ytgpu_evaluate_filter(GetGpuContext(), valueViews.data(), (uint32_t)valueViews.size(), stringViews.data(),
                                          (uint32_t)stringViews.size(), program.data(), (uint32_t)program.size(), lists.data(), lists.size(),
                                          reinterpret_cast<const uint8_t*>(constants.data()), constants.size(), selection.data(), nullptr,
                                          nullptr, 0, &selected, YTGPU_MEM_HOST, &err) != YTGPU_OK)
                    ThrowFrom(err);
                ytgpu_column_view v{};
                v.value_count = (int64_t)n;
                v.value_type = (uint8_t)EValueType::Boolean;
                v.has_values = 1;
                v.bit_width = 1;
                v.values = selection.data();
                v.values_count = n;
                v.mem = YTGPU_MEM_HOST;
                predicateColumn = (int)valueViews.size();
                valueViews.push_back(v);
            }
            // the other computed columns, over the rows the WHERE selects
            for (size_t i = 0; i < columns.size(); ++i)
                if (isComputed((int)i) && !evaluated[i]) {
                    const EValueType planned = columns[i].Type;
                    evaluateComputed((int)i, where ? selection.data() : nullptr);
                    if ((columns[i].Type == EValueType::String) != (planned == EValueType::String))
                        throw TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "computed column " + std::to_string(-2 - columns[i].Position) +
                                                                              ": result type differs from its inputs' typing");
                    if (argIndex[i] >= 0) valueViews[argIndex[i]] = view(columns[i]);
                    else stringViews[-1 - argIndex[i]] = stringView(columns[i]);
                }
            for (auto& a : argIndex)
                if (a < 0) a = (int)valueViews.size() + (-1 - a);
            for (int k : keyIndex) {
                auto& c = columns[k];
                if (c.Type == EValueType::String) {  // a string group item: canonical row ids (the first row of every value)
                    ytgpu_error err{};
                    if (ytgpu_string_value_ids(GetGpuContext(), reinterpret_cast<const uint8_t*>(c.Heap.data()), c.Heap.size(), c.Starts.data(),
                                               c.Lengths.data(), c.NullBytes.data(), n, c.Values.data(), nullptr, YTGPU_MEM_HOST, &err) != YTGPU_OK)
                        ThrowFrom(err);
                    auto ids = view(c);
                    ids.value_type = (uint8_t)EValueType::Uint64;
                    keyViews.push_back(ids);
                } else {
                    keyViews.push_back(view(c));
                }
            }
            std::vector<ytgpu_aggregate> aggregates;
            for (size_t a = 0; a < query.AggregateItems.size(); ++a) {
                static const int ops[] = {YTGPU_AGG_SUM, YTGPU_AGG_MIN, YTGPU_AGG_MAX, YTGPU_AGG_COUNT, YTGPU_AGG_AVG, YTGPU_AGG_ARGMIN, YTGPU_AGG_ARGMAX, YTGPU_AGG_FIRST};
                aggregates.push_back(ytgpu_aggregate{ops[(int)query.AggregateItems[a].Function], argIndex[aggIndex[a]],
                                                     byIndex[a] >= 0 ? argIndex[byIndex[a]] : -1, 0});
            }
            if (project) {
                // the output row: the projected columns over all rows; the WHERE's rows are the ones ordered
                std::vector<ytgpu_column_view> projected;
                std::vector<std::optional<ytgpu_string_column>> strings;
                for (int i : projectIndex) {
                    const TFlatColumn& c = columns[i];
                    projected.push_back(view(c));
                    strings.push_back(std::nullopt);
                    if (c.Type == EValueType::String) {
                        projected.back().value_type = (uint8_t)EValueType::String;
                        strings.back() = stringView(c);
                    }
                }
                std::vector<uint32_t> kept;
                if (where)
                    for (uint64_t r = 0; r < n; ++r)
                        if ((selection[r >> 3] >> (r & 7)) & 1) kept.push_back((uint32_t)r);
                const std::vector<uint32_t> rows = orderWindow(projected, strings, where ? selection.data() : nullptr, where ? &kept : nullptr, n);
                // the output columns gathered at the window's rows: Select sees those rows only.  A string position keeps the
                // row index into its flat column.
                const uint64_t m = rows.size();
                const size_t np = projectIndex.size();
                std::vector<uint64_t> rowIds(rows.begin(), rows.end());
                std::vector<std::vector<uint64_t>> gathered(np);
                std::vector<std::vector<uint8_t>> bitmaps(np), nullBytes(np);
                std::vector<TOutput> outputs;
                std::vector<ytgpu_column_view> outViews;
                for (size_t p = 0; p < np; ++p) {
                    const TFlatColumn& c = columns[projectIndex[p]];
                    bitmaps[p].assign((m + 63) / 64 * 8, 0);
                    nullBytes[p].assign(m, 0);
                    if (c.Type == EValueType::String) {
                        for (uint64_t i = 0; i < m; ++i) nullBytes[p][i] = c.NullBytes[rows[i]];
                    } else if (m > 0) {
                        gathered[p].assign(m, 0);
                        const ytgpu_column_view source = view(c);
                        uint64_t nullCount = 0;
                        ytgpu_error err{};
                        if (ytgpu_gather_column(GetGpuContext(), &source, rows.data(), m, gathered[p].data(), bitmaps[p].data(), &nullCount,
                                                YTGPU_MEM_HOST, &err) != YTGPU_OK)
                            ThrowFrom(err);
                    }
                    for (uint64_t i = 0; i < m; ++i) {
                        if (c.Type != EValueType::String) nullBytes[p][i] = (bitmaps[p][i >> 3] >> (i & 7)) & 1;
                        else if (nullBytes[p][i]) bitmaps[p][i >> 3] |= (uint8_t)(1u << (i & 7));
                    }
                    const bool str = c.Type == EValueType::String;
                    outputs.push_back({c.Type, str ? &c : nullptr, str ? rowIds.data() : gathered[p].data(), nullBytes[p].data()});
                    ytgpu_column_view v{};
                    v.value_count = (int64_t)m;
                    v.value_type = (uint8_t)(str ? EValueType::String : c.Type == EValueType::Null ? EValueType::Int64 : c.Type);
                    v.has_values = m > 0;
                    v.bit_width = 64;
                    v.values = m == 0 ? nullptr : str ? rowIds.data() : gathered[p].data();
                    v.values_count = m;
                    v.null_bitmap = bitmaps[p].data();
                    v.mem = YTGPU_MEM_HOST;
                    outViews.push_back(v);
                }
                const std::vector<TOutput> selected = query.Select ? evaluateSelect(outputs, outViews, nullptr, m) : outputs;
                owned.reserve(m);
                for (uint64_t i = 0; i < m; ++i) writeRow(selected, i);
            }
            const size_t nk = keyViews.size(), na = aggregates.size();
            uint64_t cap = std::min<uint64_t>(n, 1 << 16);
            while (!project) {  // the GROUP BY call, again with the capacity it reports when its first guess was too small
                std::vector<std::vector<uint64_t>> keys(nk, std::vector<uint64_t>(cap)), values(na, std::vector<uint64_t>(cap));
                std::vector<std::vector<uint8_t>> keyNull(nk, std::vector<uint8_t>(cap)), valueNull(na, std::vector<uint8_t>(cap));
                std::vector<uint64_t*> pk, pv;
                std::vector<uint8_t*> pkn, pvn;
                for (size_t k = 0; k < nk; ++k) { pk.push_back(keys[k].data()); pkn.push_back(keyNull[k].data()); }
                for (size_t a = 0; a < na; ++a) { pv.push_back(values[a].data()); pvn.push_back(valueNull[a].data()); }
                ytgpu_groupby_multi_result res{0, cap, pk.data(), pkn.data(), pv.data(), pvn.data(), nullptr, nullptr};
                ytgpu_predicate pred{CmpOf(query.WhereOp), 0, query.WhereConstant.Data.Uint64};
                if (where) pred = ytgpu_predicate{YTGPU_CMP_EQ, 0, 1};
                const int predArg = where ? predicateColumn : (whereIndex >= 0 ? argIndex[whereIndex] : -1);
                ytgpu_error err{};
                const int code = ytgpu_scan_filter_groupby_multi_strings(
                    GetGpuContext(), keyViews.data(), (uint32_t)nk, valueViews.data(), (uint32_t)valueViews.size(), aggregates.data(),
                    (uint32_t)na, predArg >= 0 ? &pred : nullptr, predArg, 0, &res, YTGPU_MEM_HOST,
                    stringViews.data(), (uint32_t)stringViews.size(), &err);
                if (code == YTGPU_ERR_INVALID_ARGUMENT && res.group_count > cap) {  // more groups than the first guess
                    cap = res.group_count;
                    continue;
                }
                if (code != YTGPU_OK) ThrowFrom(err);
                auto stringsOf = [&](int index) { return columns[index].Type == EValueType::String ? &columns[index] : nullptr; };
                // the output row's positions: group items, then aggregates
                std::vector<TOutput> outputs;
                for (size_t k = 0; k < nk; ++k)
                    outputs.push_back({columns[keyIndex[k]].Type, stringsOf(keyIndex[k]), keys[k].data(), keyNull[k].data()});
                for (size_t a = 0; a < na; ++a) {
                    const auto f = query.AggregateItems[a].Function;
                    const EValueType type = f == EAggregateFunction::Count ? EValueType::Int64
                        : f == EAggregateFunction::Avg ? EValueType::Double : columns[aggIndex[a]].Type;
                    outputs.push_back({type, f == EAggregateFunction::Count ? nullptr : stringsOf(aggIndex[a]), values[a].data(), valueNull[a].data()});
                }
                const uint64_t groups = res.group_count;
                // Select, Having and the ORDER BY items are evaluated over the result arrays (evaluateSelect)
                std::vector<TOutput> selected;
                std::vector<uint64_t> having;  // Having: bit g set where group g is written
                std::vector<std::vector<uint8_t>> bitmaps(outputs.size());
                std::vector<ytgpu_column_view> outViews;
                if (query.Select || query.Having || !query.OrderBy.empty()) {
                    for (size_t p = 0; p < outputs.size(); ++p) {
                        bitmaps[p].assign((groups + 63) / 64 * 8, 0);
                        for (uint64_t g = 0; g < groups; ++g)
                            if (outputs[p].Null[g]) bitmaps[p][g >> 3] |= (uint8_t)(1u << (g & 7));
                        ytgpu_column_view v{};
                        v.value_count = (int64_t)groups;
                        v.value_type = (uint8_t)(outputs[p].Strings ? EValueType::String
                                                 : outputs[p].Type == EValueType::Null ? EValueType::Int64 : outputs[p].Type);
                        v.has_values = 1;
                        v.bit_width = 64;
                        v.values = outputs[p].Values;
                        v.values_count = groups;
                        v.null_bitmap = bitmaps[p].data();
                        v.mem = YTGPU_MEM_HOST;
                        outViews.push_back(v);
                    }
                }
                if (query.Having) having = evaluateHaving(outViews, groups);
                // ORDER BY, OFFSET and LIMIT over the groups Having keeps: the window's groups, in order
                const bool windowed = !query.OrderBy.empty() || query.Limit;
                std::vector<uint32_t> window;
                std::vector<uint64_t> windowBits;
                if (windowed) {
                    std::vector<uint32_t> kept;
                    for (uint64_t g = 0; query.Having && g < groups; ++g)
                        if ((having[g >> 6] >> (g & 63)) & 1) kept.push_back((uint32_t)g);
                    // a string position as a flat column over the groups: its rows' starts and lengths
                    std::vector<std::optional<ytgpu_string_column>> strings(outputs.size());
                    std::vector<std::vector<uint64_t>> starts(outputs.size());
                    std::vector<std::vector<uint32_t>> lengths(outputs.size());
                    for (size_t p = 0; p < outputs.size() && !query.OrderBy.empty(); ++p) {
                        const TFlatColumn* S = outputs[p].Strings;
                        if (!S) continue;
                        starts[p].assign(groups, 0);
                        lengths[p].assign(groups, 0);
                        for (uint64_t g = 0; g < groups; ++g)
                            if (!outputs[p].Null[g]) {
                                starts[p][g] = S->Starts[outputs[p].Values[g]];
                                lengths[p][g] = S->Lengths[outputs[p].Values[g]];
                            }
                        strings[p] = ytgpu_string_column{reinterpret_cast<const uint8_t*>(S->Heap.data()), S->Heap.size(), starts[p].data(),
                                                         lengths[p].data(), outputs[p].Null, groups, YTGPU_MEM_HOST, 0};
                    }
                    window = orderWindow(outViews, strings, query.Having ? reinterpret_cast<const uint8_t*>(having.data()) : nullptr,
                                         query.Having ? &kept : nullptr, groups);
                    windowBits.assign((groups + 63) / 64, 0);
                    for (uint32_t g : window) windowBits[g >> 6] |= 1ull << (g & 63);
                }
                // Select is evaluated over the groups written only, as QL projects after HAVING and LIMIT: a division by zero
                // in a dropped group does not throw
                const uint8_t* selectSelection = windowed ? reinterpret_cast<const uint8_t*>(windowBits.data())
                                               : query.Having ? reinterpret_cast<const uint8_t*>(having.data()) : nullptr;
                selected = query.Select ? evaluateSelect(outputs, outViews, selectSelection, groups) : outputs;
                if (windowed) {
                    owned.reserve(window.size());
                    for (uint32_t g : window) writeRow(selected, g);
                    break;
                }
                owned.reserve(groups);
                for (uint64_t g = 0; g < groups; ++g) {  // already in first-seen order
                    if (query.Having && !((having[g >> 6] >> (g & 63)) & 1)) continue;
                    writeRow(selected, g);
                }
                break;
            }
        }
        std::vector<TUnversionedRow> out(owned.begin(), owned.end());
        constexpr size_t kBatch = 1024;
        for (size_t i = 0; i < out.size(); i += kBatch) {
            std::vector<TUnversionedRow> part(out.begin() + i, out.begin() + std::min(out.size(), i + kBatch));
            (void)writer->Write(part);
        }
        writer->Close();
        stats.RowsWritten = (int64_t)out.size();
        return stats;
    }
};

}  // namespace

IEvaluatorPtr CreateGpuEvaluator() { return std::make_shared<TGpuEvaluator>(); }

// ---- ORDER BY ... LIMIT k ----
TTopCollector::TTopCollector(int64_t limit, TComparator comparator)
    : Limit_(limit), Comparator_(std::move(comparator)), CompactAt_(std::max<size_t>(65536, 4 * (size_t)std::max<int64_t>(limit, 0))) {}

void TTopCollector::AddRow(TUnversionedRow row) {
    if (Limit_ <= 0) return;
    Rows_.emplace_back(row.Begin(), row.End());
    if (Rows_.size() >= CompactAt_) Compact();
}

void TTopCollector::Compact() {
    if (Rows_.empty()) return;
    std::vector<TUnversionedRow> rows(Rows_.begin(), Rows_.end());
    TFlatRowset flat(rows, (uint32_t)Comparator_.GetLength());
    auto cols = KeyColumnsOf(Comparator_);
    ytgpu_sort_spec spec{cols.data(), (uint32_t)cols.size()};
    std::vector<uint32_t> perm(rows.size());
    ytgpu_error err{};
    if (ytgpu_sort_rowset(GetGpuContext(), &flat.View, &spec, perm.data(), nullptr, YTGPU_MEM_HOST, &err) != YTGPU_OK) ThrowFrom(err);
    std::vector<TUnversionedOwningRow> kept;
    const size_t keep = std::min<size_t>((size_t)Limit_, rows.size());
    kept.reserve(keep);
    for (size_t i = 0; i < keep; ++i) kept.push_back(std::move(Rows_[perm[i]]));
    Rows_ = std::move(kept);
}

std::vector<TUnversionedOwningRow> TTopCollector::GetRows() {
    Compact();
    return Rows_;
}

}  // namespace NQueryClient

}  // namespace NYT

// ---- YQL ----
namespace NYql::NMiniKQL {

namespace {

class TGpuBlockCombineHashed : public IBlockCombineHashed {
public:
    TGpuBlockCombineHashed(uint64_t hint, bool withMinMax) : States_(hint, withMinMax) {}

    void AddBlock(const TArrowColumn& keys, const TArrowColumn& values) override {
        if (keys.Length != values.Length) throw NYT::NTableClient::TErrorException(YTGPU_ERR_INVALID_ARGUMENT, "Block columns differ in length");
        States_.AddBatch(NDetail::ArrowColumnView(keys), NDetail::ArrowColumnView(values), YTGPU_CMP_NONE, 0, Rows_);
        Rows_ += (uint64_t)keys.Length;
    }

    TResult Finish() override {
        auto m = States_.Merge();
        TResult r;
        r.Keys = std::move(m.Keys);
        r.Sums = std::move(m.Sums);
        r.Counts = std::move(m.Counts);
        r.Mins = std::move(m.Mins);
        r.Maxs = std::move(m.Maxs);
        r.KeyValid.resize(r.Keys.size());
        r.SumValid.resize(r.Keys.size());
        for (size_t i = 0; i < r.Keys.size(); ++i) {
            r.KeyValid[i] = !m.KeyNulls[i];
            r.SumValid[i] = !m.SumNulls[i];
        }
        return r;
    }

private:
    NYT::TPartialStates States_;
    uint64_t Rows_ = 0;
};

}  // namespace

std::unique_ptr<IBlockCombineHashed> CreateGpuBlockCombineHashed(uint64_t groupCountHint, bool withMinMax) {
    return std::make_unique<TGpuBlockCombineHashed>(groupCountHint, withMinMax);
}

}  // namespace NYql::NMiniKQL
