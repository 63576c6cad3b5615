// conditional_expression_ut.cpp — the QL evaluator adapter (TGpuEvaluator::Run(TMultiGroupQuery)) with conditional computed
// columns, against row-at-a-time restatements:
//   * sum(if(status = 200, 1, 0)) and the guarded division sum(if(b = 0, 0, a / b)) over zero divisors;
//   * GROUP BY if(a > 0, s, 'other'), a string IF key, and GROUP BY if(flag, 1, 2) with a NULL condition;
//   * Select with a comparison (sum(a) > 100) and Having over the output row; Select evaluated over the kept groups only
//     (sum(a) / sum(b) with a group whose sum(b) is 0, dropped by Having); Having checked on an empty input;
//   * an input column that is NULL in every row compared with a string, as an IF branch beside a string, under AND / NOT
//     and as IF's condition.
// Runs on the GPU box (tests/test_conditional_expressions.py drives it); exit code = number of failed expectations.
#include <cstdio>
#include <cstring>
#include <map>
#include <optional>
#include <random>
#include <string>
#include <vector>

#include "../../include/ytgpu.h"
#include "../yt_query_client.h"

using namespace NYT::NTableClient;
using namespace NYT::NQueryClient;

static int Failures = 0;
#define EXPECT_EQ(a, b) do { auto _a = (a); auto _b = (b); if (!(_a == _b)) { ++Failures; std::fprintf(stderr, "%s:%d: EXPECT_EQ(%s, %s) failed\n", __FILE__, __LINE__, #a, #b); } } while (0)
#define EXPECT_TRUE(a) do { if (!(a)) { ++Failures; std::fprintf(stderr, "%s:%d: EXPECT_TRUE(%s) failed\n", __FILE__, __LINE__, #a); } } while (0)

namespace {

struct TCollectingWriter : IUnversionedRowsetWriter {
    std::vector<TUnversionedOwningRow> Rows;
    bool Write(const std::vector<TUnversionedRow>& rows) override {
        for (auto r : rows) {
            TUnversionedOwningRowBuilder b;
            for (const auto* v = r.Begin(); v != r.End(); ++v) b.AddValue(*v);
            Rows.push_back(b.FinishRow());
        }
        return true;
    }
    void Close() override {}
};

std::vector<TUnversionedOwningRow> Run(const TMultiGroupQuery& q, const std::vector<TUnversionedOwningRow>& rows,
                                       TQueryStatistics* stats = nullptr) {
    auto writer = std::make_shared<TCollectingWriter>();
    const auto s = CreateGpuEvaluator()->Run(q, CreateInMemoryReader(rows), writer);
    if (stats) *stats = s;
    return writer->Rows;
}

int Code(const TMultiGroupQuery& q, const std::vector<TUnversionedOwningRow>& rows) {
    try {
        Run(q, rows);
    } catch (const TErrorException& e) {
        return e.GetCode();
    }
    return 0;
}

using TOptStr = std::optional<std::string>;
// input positions: 0 k, 1 status (nullable), 2 a, 3 b (zeros among them), 4 s (nullable string), 5 flag (nullable
// boolean), 6 n (NULL in every row)
struct TRow { int64_t K; std::optional<int64_t> Status; int64_t A, B; TOptStr S; std::optional<bool> Flag; };

std::vector<TUnversionedOwningRow> Owned(const std::vector<TRow>& rows) {
    std::vector<TUnversionedOwningRow> owned;
    for (const auto& r : rows) {
        TUnversionedOwningRowBuilder b;
        b.AddValue(MakeUnversionedInt64Value(r.K, 0));
        b.AddValue(r.Status ? MakeUnversionedInt64Value(*r.Status, 1) : MakeUnversionedNullValue(1));
        b.AddValue(MakeUnversionedInt64Value(r.A, 2));
        b.AddValue(MakeUnversionedInt64Value(r.B, 3));
        b.AddValue(r.S ? MakeUnversionedStringValue(*r.S, 4) : MakeUnversionedNullValue(4));
        b.AddValue(r.Flag ? MakeUnversionedBooleanValue(*r.Flag, 5) : MakeUnversionedNullValue(5));
        b.AddValue(MakeUnversionedNullValue(6));
        owned.push_back(b.FinishRow());
    }
    return owned;
}

std::vector<TRow> RandomRows(size_t count, uint64_t seed) {
    static const char* hosts[] = {"example.com", "yt.tech", "", "a-b.c"};
    static const int64_t statuses[] = {200, 404, 500, 200};
    std::mt19937_64 rng(seed);
    std::vector<TRow> rows;
    for (size_t i = 0; i < count; ++i) {
        TRow r{(int64_t)(rng() % 5), std::nullopt, (int64_t)(rng() % 2001) - 1000, (int64_t)(rng() % 5) - 2, std::nullopt, std::nullopt};
        if (rng() % 9) r.Status = statuses[rng() % 4];
        if (rng() % 6) r.S = hosts[rng() % 4];
        if (rng() % 4) r.Flag = (rng() & 1) != 0;
        rows.push_back(r);
    }
    return rows;
}

// SELECT k, sum(if(status = 200, 1, 0)), sum(if(b = 0, 0, a / b)) GROUP BY k
void TestConditionalSums() {
    const auto rows = RandomRows(20000, 3);
    TMultiGroupQuery q;
    q.Computed = {
        TExpression().Column(1).Constant(MakeUnversionedInt64Value(200)).Compare(EBinaryOp::Equal)
            .Constant(MakeUnversionedInt64Value(1)).Constant(MakeUnversionedInt64Value(0)).If(),
        TExpression().Column(3).Constant(MakeUnversionedInt64Value(0)).Compare(EBinaryOp::Equal)
            .Constant(MakeUnversionedInt64Value(0)).Column(2).Column(3).Div().If(),
    };
    q.GroupColumns = {0};
    q.AggregateItems = {{EAggregateFunction::Sum, TMultiGroupQuery::ComputedColumn(0)}, {EAggregateFunction::Sum, TMultiGroupQuery::ComputedColumn(1)}};
    const auto got = Run(q, Owned(rows));
    std::vector<int64_t> order;
    std::map<int64_t, std::pair<int64_t, int64_t>> want;
    for (const auto& r : rows) {
        if (!want.count(r.K)) order.push_back(r.K);
        auto& w = want[r.K];
        // a NULL status makes the comparison NULL, so if() takes neither branch: NULL, which sum skips
        w.first += r.Status && *r.Status == 200 ? 1 : 0;
        w.second += r.B == 0 ? 0 : r.A / r.B;
    }
    EXPECT_EQ(got.size(), order.size());
    for (size_t g = 0; g < std::min(got.size(), order.size()); ++g) {
        EXPECT_EQ(got[g][0].Data.Int64, order[g]);
        EXPECT_TRUE(got[g][1].Type == EValueType::Int64 && got[g][1].Data.Int64 == want[order[g]].first);
        EXPECT_TRUE(got[g][2].Type == EValueType::Int64 && got[g][2].Data.Int64 == want[order[g]].second);
    }
    // the unguarded division throws "Division by zero"; guarded the other way round it throws too
    q.Computed[1] = TExpression().Column(2).Column(3).Div();
    EXPECT_EQ(Code(q, Owned(rows)), (int)YTGPU_ERR_INVALID_ARGUMENT);
    q.Computed[1] = TExpression().Column(3).Constant(MakeUnversionedInt64Value(0)).Compare(EBinaryOp::Equal)
                        .Column(2).Column(3).Div().Constant(MakeUnversionedInt64Value(0)).If();
    EXPECT_EQ(Code(q, Owned(rows)), (int)YTGPU_ERR_INVALID_ARGUMENT);
}

// SELECT key, count(a) GROUP BY if(a > 0, s, 'other') AS key; and GROUP BY if(flag, 1, 2)
void TestStringIfKeyAndNullCondition() {
    const auto rows = RandomRows(5000, 5);
    TMultiGroupQuery q;
    q.Computed = {TExpression().Column(2).Constant(MakeUnversionedInt64Value(0)).Compare(EBinaryOp::Greater)
                      .Column(4).Constant(MakeUnversionedStringValue("other")).If()};
    q.GroupColumns = {TMultiGroupQuery::ComputedColumn(0)};
    q.AggregateItems = {{EAggregateFunction::Count, 2}};
    auto got = Run(q, Owned(rows));
    std::vector<TOptStr> order;
    std::map<TOptStr, int64_t> want;
    for (const auto& r : rows) {
        const TOptStr k = r.A > 0 ? r.S : TOptStr("other");
        if (!want.count(k)) order.push_back(k);
        ++want[k];
    }
    EXPECT_EQ(got.size(), order.size());
    for (size_t g = 0; g < std::min(got.size(), order.size()); ++g) {
        EXPECT_TRUE(order[g] ? got[g][0].Type == EValueType::String && got[g][0].AsStringBuf() == *order[g] : got[g][0].Type == EValueType::Null);
        EXPECT_EQ(got[g][1].Data.Int64, want[order[g]]);
    }
    q.Computed = {TExpression().Column(5).Constant(MakeUnversionedInt64Value(1)).Constant(MakeUnversionedInt64Value(2)).If()};
    got = Run(q, Owned(rows));
    std::vector<std::optional<int64_t>> korder;
    std::map<std::optional<int64_t>, int64_t> kwant;
    for (const auto& r : rows) {
        const std::optional<int64_t> k = r.Flag ? std::optional<int64_t>(*r.Flag ? 1 : 2) : std::nullopt;
        if (!kwant.count(k)) korder.push_back(k);
        ++kwant[k];
    }
    EXPECT_EQ(got.size(), korder.size());
    for (size_t g = 0; g < std::min(got.size(), korder.size()); ++g) {
        EXPECT_TRUE(korder[g] ? got[g][0].Type == EValueType::Int64 && got[g][0].Data.Int64 == *korder[g] : got[g][0].Type == EValueType::Null);
        EXPECT_EQ(got[g][1].Data.Int64, kwant[korder[g]]);
    }
}

// SELECT k, sum(a), sum(a) > 100 GROUP BY k HAVING sum(a) > 100 [AND k != 3]
void TestSelectAndHaving() {
    const auto rows = RandomRows(3000, 9);
    TMultiGroupQuery q;
    q.GroupColumns = {0};
    q.AggregateItems = {{EAggregateFunction::Sum, 2}};
    q.Select = std::vector<TExpression>{TExpression().Column(0), TExpression().Column(1),
                                        TExpression().Column(1).Constant(MakeUnversionedInt64Value(100)).Compare(EBinaryOp::Greater)};
    std::vector<int64_t> order;
    std::map<int64_t, int64_t> sums;
    for (const auto& r : rows) {
        if (!sums.count(r.K)) order.push_back(r.K);
        sums[r.K] += r.A;
    }
    TQueryStatistics stats;
    auto got = Run(q, Owned(rows), &stats);
    EXPECT_EQ(got.size(), order.size());
    EXPECT_EQ(stats.RowsWritten, (int64_t)order.size());
    for (size_t g = 0; g < std::min(got.size(), order.size()); ++g) {
        EXPECT_TRUE(got[g][2].Type == EValueType::Boolean && got[g][2].Data.Boolean == (sums[order[g]] > 100));
        EXPECT_EQ(got[g][1].Data.Int64, sums[order[g]]);
    }
    for (int64_t bound : {-100000, 100, 100000}) {
        q.Having = TExpression().Column(1).Constant(MakeUnversionedInt64Value(bound)).Compare(EBinaryOp::Greater)
                       .Column(0).Constant(MakeUnversionedInt64Value(3)).Compare(EBinaryOp::NotEqual).And();
        got = Run(q, Owned(rows), &stats);
        std::vector<int64_t> kept;
        for (int64_t k : order)
            if (sums[k] > bound && k != 3) kept.push_back(k);
        EXPECT_EQ(got.size(), kept.size());
        EXPECT_EQ(stats.RowsWritten, (int64_t)kept.size());
        for (size_t g = 0; g < std::min(got.size(), kept.size()); ++g) {
            EXPECT_EQ(got[g][0].Data.Int64, kept[g]);
            EXPECT_EQ(got[g][1].Data.Int64, sums[kept[g]]);
        }
    }
    // Having without Select; a non-Boolean Having is INVALID_ARGUMENT; a string position UNSUPPORTED
    q.Select.reset();
    q.Having = TExpression().Column(0).Constant(MakeUnversionedInt64Value(2)).Compare(EBinaryOp::LessOrEqual);
    got = Run(q, Owned(rows));
    size_t small = 0;
    for (int64_t k : order) small += k <= 2;
    EXPECT_EQ(got.size(), small);
    for (const auto& r : got) EXPECT_TRUE(r[0].Data.Int64 <= 2 && r.GetCount() == 2);
    q.Having = TExpression().Column(1);
    EXPECT_EQ(Code(q, Owned(rows)), (int)YTGPU_ERR_INVALID_ARGUMENT);
    q.GroupColumns = {4};
    q.Having = TExpression().Column(0).IsNull();
    EXPECT_EQ(Code(q, Owned(rows)), (int)YTGPU_ERR_UNSUPPORTED);
}

// SELECT k, sum(a) / sum(b) GROUP BY k HAVING sum(b) != 0: Select runs over the kept groups only, so the group whose
// sum(b) is 0 does not throw "Division by zero"; without Having it does
void TestSelectAfterHaving() {
    std::vector<TRow> rows;
    for (int64_t k = 0; k < 4; ++k)
        for (int64_t i = 0; i < 100; ++i)  // group 2: b sums to 0
            rows.push_back(TRow{k, 200, 10 * (k + 1) + i, k == 2 ? (i % 2 ? 1 : -1) : k + 1, std::nullopt, std::nullopt});
    std::map<int64_t, std::pair<int64_t, int64_t>> sums;
    for (const auto& r : rows) {
        sums[r.K].first += r.A;
        sums[r.K].second += r.B;
    }
    TMultiGroupQuery q;
    q.GroupColumns = {0};
    q.AggregateItems = {{EAggregateFunction::Sum, 2}, {EAggregateFunction::Sum, 3}};
    q.Select = std::vector<TExpression>{TExpression().Column(0), TExpression().Column(1).Column(2).Div()};
    EXPECT_EQ(Code(q, Owned(rows)), (int)YTGPU_ERR_INVALID_ARGUMENT);
    q.Having = TExpression().Column(2).Constant(MakeUnversionedInt64Value(0)).Compare(EBinaryOp::NotEqual);
    TQueryStatistics stats;
    const auto got = Run(q, Owned(rows), &stats);
    EXPECT_EQ(got.size(), (size_t)3);
    EXPECT_EQ(stats.RowsWritten, (int64_t)3);
    const int64_t keys[] = {0, 1, 3};
    for (size_t g = 0; g < std::min<size_t>(got.size(), 3); ++g) {
        EXPECT_EQ(got[g][0].Data.Int64, keys[g]);
        EXPECT_TRUE(got[g][1].Type == EValueType::Int64 && got[g][1].Data.Int64 == sums[keys[g]].first / sums[keys[g]].second);
    }
}

// Having's shape is checked whatever the data: on an empty input and when the WHERE leaves no group
void TestHavingCheckedWithoutGroups() {
    TMultiGroupQuery q;
    q.GroupColumns = {0};
    q.AggregateItems = {{EAggregateFunction::Sum, 2}};
    q.Having = TExpression().Column(1);  // an Int64, not a Boolean
    EXPECT_EQ(Code(q, {}), (int)YTGPU_ERR_INVALID_ARGUMENT);
    const auto rows = RandomRows(500, 13);
    q.Where = TFilterExpression().Compare(2, EBinaryOp::Less, MakeUnversionedInt64Value(-100000));
    EXPECT_EQ(Code(q, Owned(rows)), (int)YTGPU_ERR_INVALID_ARGUMENT);
    q.Having = TExpression().Column(1).Constant(MakeUnversionedInt64Value(0)).Compare(EBinaryOp::Greater);
    EXPECT_EQ(Code(q, {}), 0);
    TQueryStatistics stats;
    EXPECT_TRUE(Run(q, Owned(rows), &stats).empty() && stats.RowsWritten == 0);
    q.Having = TExpression().Column(1).Lower();  // a string function over the output row
    EXPECT_EQ(Code(q, {}), (int)YTGPU_ERR_UNSUPPORTED);
}

// n (position 6) is NULL in every row
void TestAllNullInputColumn() {
    const auto rows = RandomRows(2000, 11);
    auto groups = [&](TExpression e) {
        TMultiGroupQuery q;
        q.Computed = {std::move(e)};
        q.GroupColumns = {TMultiGroupQuery::ComputedColumn(0)};
        q.AggregateItems = {{EAggregateFunction::Count, 2}};
        return Run(q, Owned(rows));
    };
    // compared with a string: NULL
    auto got = groups(TExpression().Column(6).Constant(MakeUnversionedStringValue("x")).Compare(EBinaryOp::Equal));
    EXPECT_EQ(got.size(), (size_t)1);
    if (!got.empty()) EXPECT_TRUE(got[0][0].Type == EValueType::Null && got[0][1].Data.Int64 == (int64_t)rows.size());
    // an IF branch beside a string: a string key, NULL where a > 0
    got = groups(TExpression().Column(2).Constant(MakeUnversionedInt64Value(0)).Compare(EBinaryOp::Greater).Column(6)
                     .Constant(MakeUnversionedStringValue("x")).If());
    int64_t positive = 0;
    for (const auto& r : rows) positive += r.A > 0;
    EXPECT_EQ(got.size(), (size_t)2);
    for (const auto& r : got) {
        if (r[0].Type == EValueType::Null) EXPECT_EQ(r[1].Data.Int64, positive);
        else EXPECT_TRUE(r[0].Type == EValueType::String && r[0].AsStringBuf() == "x" && r[1].Data.Int64 == (int64_t)rows.size() - positive);
    }
    // under AND: FALSE where a <= 0, NULL elsewhere; under NOT: NULL
    got = groups(TExpression().Column(6).Column(2).Constant(MakeUnversionedInt64Value(0)).Compare(EBinaryOp::Greater).And());
    EXPECT_EQ(got.size(), (size_t)2);
    for (const auto& r : got) {
        if (r[0].Type == EValueType::Null) EXPECT_EQ(r[1].Data.Int64, positive);
        else EXPECT_TRUE(r[0].Type == EValueType::Boolean && !r[0].Data.Boolean && r[1].Data.Int64 == (int64_t)rows.size() - positive);
    }
    got = groups(TExpression().Column(6).Not());
    EXPECT_TRUE(got.size() == 1 && got[0][0].Type == EValueType::Null);
    // as IF's condition: NULL
    got = groups(TExpression().Column(6).Constant(MakeUnversionedInt64Value(1)).Constant(MakeUnversionedInt64Value(2)).If());
    EXPECT_TRUE(got.size() == 1 && got[0][0].Type == EValueType::Null);
    // is_null of it: TRUE everywhere
    got = groups(TExpression().Column(6).IsNull());
    EXPECT_TRUE(got.size() == 1 && got[0][0].Type == EValueType::Boolean && got[0][0].Data.Boolean);
}

}  // namespace

int main() {
    try {
        TestConditionalSums();
        TestStringIfKeyAndNullCondition();
        TestSelectAndHaving();
        TestSelectAfterHaving();
        TestHavingCheckedWithoutGroups();
        TestAllNullInputColumn();
    } catch (const std::exception& e) {
        std::fprintf(stderr, "unexpected exception: %s\n", e.what());
        return 100;
    }
    std::printf("conditional_expression_ut: %d failure(s)\n", Failures);
    return Failures;
}
