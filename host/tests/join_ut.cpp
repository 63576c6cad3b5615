// join_ut.cpp — the QL evaluator adapter (TGpuEvaluator::Run(TMultiGroupQuery)) with a JOIN clause, against rows spelled
// out below:
//   * a star join with GROUP BY a foreign attribute and sum of a primary column (one key with two foreign rows);
//   * a LEFT join whose missing foreign side feeds count (0) and first (NULL);
//   * string join keys, LEFT, with the unmatched rows in a NULL group;
//   * WHERE on a foreign column; a computed column over a primary and a foreign column;
//   * Select and Having on top;
//   * a key pair of different types (Int64 against Uint64), which throws INVALID_ARGUMENT.
// Runs on the GPU box (tests/test_hash_join.py drives it); exit code = number of failed expectations.
#include <cstdio>
#include <optional>
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

TUnversionedValue I(int64_t x) { return MakeUnversionedInt64Value(x); }
constexpr int F(int j) { return TMultiGroupQuery::ForeignColumn(j); }

// facts (primary): 0 dim_id (nullable), 1 amount, 2 dim_name (nullable string)
struct TFact { std::optional<int64_t> DimId; int64_t Amount; std::optional<std::string> DimName; };
const std::vector<TFact> Facts = {
    {1, 10, "a"}, {2, 20, "b"}, {1, 30, "a"}, {3, 40, "zz"}, {2, 50, "b"}, {std::nullopt, 60, std::nullopt},
};
// dims (foreign): 0 id, 1 region, 2 weight, 3 name; id 2 and name "b" have two rows, id 4 / "c" no fact
struct TDim { int64_t Id; std::string Region; int64_t Weight; std::string Name; };
const std::vector<TDim> Dims = {{1, "eu", 7, "a"}, {2, "us", 8, "b"}, {4, "eu", 9, "c"}, {2, "asia", 5, "b"}};

std::vector<TUnversionedOwningRow> FactRows() {
    std::vector<TUnversionedOwningRow> owned;
    for (const auto& r : Facts) {
        TUnversionedOwningRowBuilder b;
        b.AddValue(r.DimId ? MakeUnversionedInt64Value(*r.DimId, 0) : MakeUnversionedNullValue(0));
        b.AddValue(MakeUnversionedInt64Value(r.Amount, 1));
        b.AddValue(r.DimName ? MakeUnversionedStringValue(*r.DimName, 2) : MakeUnversionedNullValue(2));
        owned.push_back(b.FinishRow());
    }
    return owned;
}

std::vector<TUnversionedOwningRow> DimRows(bool unsignedIds = false) {
    std::vector<TUnversionedOwningRow> owned;
    for (const auto& r : Dims) {
        TUnversionedOwningRowBuilder b;
        b.AddValue(unsignedIds ? MakeUnversionedUint64Value((uint64_t)r.Id, 0) : MakeUnversionedInt64Value(r.Id, 0));
        b.AddValue(MakeUnversionedStringValue(r.Region, 1));
        b.AddValue(MakeUnversionedInt64Value(r.Weight, 2));
        b.AddValue(MakeUnversionedStringValue(r.Name, 3));
        owned.push_back(b.FinishRow());
    }
    return owned;
}

TMultiGroupQuery::TJoinClause Join(std::vector<int> self, std::vector<int> foreign, bool left, bool unsignedIds = false) {
    return TMultiGroupQuery::TJoinClause{CreateInMemoryReader(DimRows(unsignedIds)), std::move(self), std::move(foreign), left};
}

std::vector<TUnversionedOwningRow> Run(const TMultiGroupQuery& q, TQueryStatistics* stats = nullptr) {
    auto writer = std::make_shared<TCollectingWriter>();
    const auto s = CreateGpuEvaluator()->Run(q, CreateInMemoryReader(FactRows()), writer);
    if (stats) *stats = s;
    return writer->Rows;
}

// one output row: a string or NULL, then Int64 values (nullopt = NULL)
struct TWant { std::optional<std::string> Key; std::vector<std::optional<int64_t>> Values; };

void ExpectRows(const std::vector<TUnversionedOwningRow>& got, const std::vector<TWant>& want, int line) {
    if (got.size() != want.size()) {
        ++Failures;
        std::fprintf(stderr, "line %d: %zu rows, want %zu\n", line, got.size(), want.size());
        return;
    }
    for (size_t r = 0; r < got.size(); ++r) {
        const auto& k = got[r][0];
        const bool keyOk = want[r].Key ? (k.Type == EValueType::String && std::string(k.Data.String, k.Length) == *want[r].Key)
                                       : k.Type == EValueType::Null;
        bool valuesOk = got[r].GetCount() == 1 + (int)want[r].Values.size();
        for (size_t v = 0; valuesOk && v < want[r].Values.size(); ++v) {
            const auto& x = got[r][1 + (int)v];
            valuesOk = want[r].Values[v] ? x.Type == EValueType::Int64 && x.Data.Int64 == *want[r].Values[v] : x.Type == EValueType::Null;
        }
        if (!keyOk || !valuesOk) {
            ++Failures;
            std::fprintf(stderr, "line %d: row %zu differs\n", line, r);
        }
    }
}

// SELECT d.region, sum(f.amount) FROM facts f JOIN dims d ON f.dim_id = d.id GROUP BY d.region
// pairs in order: (0, eu) (1, us) (1, asia) (2, eu) (4, us) (4, asia); fact 3 has no dim, fact 5's NULL key matches no id
void TestStarJoinGroupByForeignAttribute() {
    TMultiGroupQuery q;
    q.Join = Join({0}, {0}, false);
    q.GroupColumns = {F(1)};
    q.AggregateItems = {{EAggregateFunction::Sum, 1}, {EAggregateFunction::Count, 1}};
    TQueryStatistics stats;
    ExpectRows(Run(q, &stats), {{"eu", {40, 2}}, {"us", {70, 2}}, {"asia", {70, 2}}}, __LINE__);
    EXPECT_EQ(stats.RowsRead, (int64_t)Facts.size());
    EXPECT_EQ(stats.RowsWritten, (int64_t)3);
}

// SELECT f.dim_name, count(d.weight), first(d.region) FROM facts f LEFT JOIN dims d ON f.dim_id = d.id GROUP BY f.dim_name
void TestLeftJoinMissingForeignSide() {
    TMultiGroupQuery q;
    q.Join = Join({0}, {0}, true);
    q.GroupColumns = {2};
    q.AggregateItems = {{EAggregateFunction::Count, F(2)}, {EAggregateFunction::First, F(1)}, {EAggregateFunction::Sum, 1}};
    const auto got = Run(q);
    // groups: "a" (facts 0, 2 -> eu), "b" (facts 1, 4 -> us, asia each), "zz" (fact 3, no dim), NULL (fact 5, no dim)
    EXPECT_EQ(got.size(), (size_t)4);
    if (got.size() != 4) return;
    const char* keys[] = {"a", "b", "zz", nullptr};
    const int64_t counts[] = {2, 4, 0, 0};
    const char* firsts[] = {"eu", "us", nullptr, nullptr};
    const int64_t sums[] = {40, 140, 40, 60};
    for (size_t g = 0; g < 4; ++g) {
        const auto& row = got[g];
        EXPECT_TRUE(keys[g] ? row[0].Type == EValueType::String && std::string(row[0].Data.String, row[0].Length) == keys[g]
                            : row[0].Type == EValueType::Null);
        EXPECT_TRUE(row[1].Type == EValueType::Int64 && row[1].Data.Int64 == counts[g]);
        EXPECT_TRUE(firsts[g] ? row[2].Type == EValueType::String && std::string(row[2].Data.String, row[2].Length) == firsts[g]
                              : row[2].Type == EValueType::Null);
        EXPECT_TRUE(row[3].Type == EValueType::Int64 && row[3].Data.Int64 == sums[g]);
    }
}

// ... LEFT JOIN dims d ON f.dim_name = d.name GROUP BY d.region: "zz" and the NULL name find no dim (no dim name is NULL)
void TestStringJoinKeys() {
    TMultiGroupQuery q;
    q.Join = Join({2}, {3}, true);
    q.GroupColumns = {F(1)};
    q.AggregateItems = {{EAggregateFunction::Sum, 1}};
    ExpectRows(Run(q), {{"eu", {40}}, {"us", {70}}, {"asia", {70}}, {std::nullopt, {100}}}, __LINE__);
    // two key columns: (dim_id, dim_name) = (id, name)
    q.Join = Join({0, 2}, {0, 3}, false);
    ExpectRows(Run(q), {{"eu", {40}}, {"us", {70}}, {"asia", {70}}}, __LINE__);
}

// ... JOIN ... WHERE d.weight > 6 GROUP BY d.region: the asia pairs (weight 5) are dropped
void TestWhereOnForeignColumn() {
    TMultiGroupQuery q;
    q.Join = Join({0}, {0}, false);
    q.Where = TFilterExpression().Compare(F(2), EBinaryOp::Greater, I(6));
    q.GroupColumns = {F(1)};
    q.AggregateItems = {{EAggregateFunction::Sum, 1}};
    ExpectRows(Run(q), {{"eu", {40}}, {"us", {70}}}, __LINE__);
}

// ... JOIN ... GROUP BY d.region with sum(f.amount * d.weight)
void TestComputedColumnOverBothSides() {
    TMultiGroupQuery q;
    q.Join = Join({0}, {0}, false);
    q.Computed = {TExpression().Column(1).Column(F(2)).Mul()};
    q.GroupColumns = {F(1)};
    q.AggregateItems = {{EAggregateFunction::Sum, TMultiGroupQuery::ComputedColumn(0)}};
    ExpectRows(Run(q), {{"eu", {280}}, {"us", {560}}, {"asia", {350}}}, __LINE__);
}

// SELECT d.region, sum(f.amount) + 1 ... GROUP BY d.region HAVING sum(f.amount) > 50
void TestSelectAndHaving() {
    TMultiGroupQuery q;
    q.Join = Join({0}, {0}, false);
    q.GroupColumns = {F(1)};
    q.AggregateItems = {{EAggregateFunction::Sum, 1}};
    q.Having = TExpression().Column(1).Constant(I(50)).Compare(EBinaryOp::Greater);
    q.Select = std::vector<TExpression>{TExpression().Column(0), TExpression().Column(1).Constant(I(1)).Add()};
    ExpectRows(Run(q), {{"us", {71}}, {"asia", {71}}}, __LINE__);
}

// f.dim_id is Int64, the dims' id Uint64: no implicit widening
void TestMistypedKeysThrow() {
    TMultiGroupQuery q;
    q.Join = Join({0}, {0}, false, true);
    q.GroupColumns = {F(1)};
    q.AggregateItems = {{EAggregateFunction::Sum, 1}};
    int code = 0;
    try {
        Run(q);
    } catch (const TErrorException& e) {
        code = e.GetCode();
    }
    EXPECT_EQ(code, (int)YTGPU_ERR_INVALID_ARGUMENT);
}

}  // namespace

int main() {
    try {
        TestStarJoinGroupByForeignAttribute();
        TestLeftJoinMissingForeignSide();
        TestStringJoinKeys();
        TestWhereOnForeignColumn();
        TestComputedColumnOverBothSides();
        TestSelectAndHaving();
        TestMistypedKeysThrow();
    } catch (const std::exception& e) {
        std::fprintf(stderr, "unexpected exception: %s\n", e.what());
        return 100;
    }
    std::printf("join_ut: %d failure(s)\n", Failures);
    return Failures;
}
