// order_ut.cpp — the QL evaluator adapter (TGpuEvaluator::Run(TMultiGroupQuery)) with ORDER BY, OFFSET and LIMIT and
// queries without GROUP BY, against rows spelled out below:
//   * a projection with WHERE and LIMIT (first rows in input order);
//   * ORDER BY two items, one DESC, over a column with NULLs; OFFSET;
//   * GROUP BY k ORDER BY sum(v) DESC LIMIT with HAVING and SELECT; ORDER BY a string group key;
//   * a projected string computed column ordered by itself; JOIN + projection ordered by a foreign column;
//   * a SELECT division by zero outside the window (no throw) and inside it (throws);
//   * every refusal;
//   * random rows over several reader batches against std::stable_sort with the comparator restated below.
// Runs on the GPU box (tests/test_order_rows.py drives it); exit code = number of failed expectations.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
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

TUnversionedValue I(int64_t x) { return MakeUnversionedInt64Value(x); }
constexpr int F(int j) { return TMultiGroupQuery::ForeignColumn(j); }
TMultiGroupQuery::TOrderItem By(TExpression e, bool descending = false) { return {std::move(e), descending}; }
TMultiGroupQuery::TOrderItem ByColumn(int position, bool descending = false) { return By(TExpression().Column(position), descending); }

// table: 0 id, 1 k (nullable), 2 v, 3 name (nullable string), 4 d (double)
struct TRow { int64_t Id; std::optional<int64_t> K; int64_t V; std::optional<std::string> Name; double D; };
const std::vector<TRow> Rows = {
    {0, 3, 10, "pear", 1.5},   {1, std::nullopt, 20, "apple", -0.0}, {2, 1, 30, std::nullopt, 2.0}, {3, 3, 40, "fig", 0.0},
    {4, 2, 0, "apple", 9.0},   {5, 1, 60, "kiwi", -3.0},             {6, std::nullopt, 70, "date", 4.0}, {7, 2, 80, "fig", 1.5},
};

std::vector<TUnversionedOwningRow> TableRows() {
    std::vector<TUnversionedOwningRow> owned;
    for (const auto& r : Rows) {
        TUnversionedOwningRowBuilder b;
        b.AddValue(MakeUnversionedInt64Value(r.Id, 0));
        b.AddValue(r.K ? MakeUnversionedInt64Value(*r.K, 1) : MakeUnversionedNullValue(1));
        b.AddValue(MakeUnversionedInt64Value(r.V, 2));
        b.AddValue(r.Name ? MakeUnversionedStringValue(*r.Name, 3) : MakeUnversionedNullValue(3));
        b.AddValue(MakeUnversionedDoubleValue(r.D, 4));
        owned.push_back(b.FinishRow());
    }
    return owned;
}

std::vector<TUnversionedOwningRow> Run(const TMultiGroupQuery& q, TQueryStatistics* stats = nullptr,
                                       std::vector<TUnversionedOwningRow> rows = TableRows()) {
    auto writer = std::make_shared<TCollectingWriter>();
    const auto s = CreateGpuEvaluator()->Run(q, CreateInMemoryReader(std::move(rows)), writer);
    if (stats) *stats = s;
    return writer->Rows;
}

int RunCode(const TMultiGroupQuery& q) {
    try {
        Run(q);
    } catch (const TErrorException& e) {
        return e.GetCode();
    }
    return 0;
}

std::vector<int64_t> Ints(const std::vector<TUnversionedOwningRow>& got, int column) {
    std::vector<int64_t> out;
    for (const auto& r : got) out.push_back(r[column].Type == EValueType::Null ? -999 : r[column].Data.Int64);
    return out;
}

std::string Str(const TUnversionedValue& v) { return v.Type == EValueType::Null ? "<null>" : std::string(v.Data.String, v.Length); }

// SELECT id, name FROM t WHERE v > 15 LIMIT 3: the first three rows WHERE keeps, in input order
void TestProjectionWhereLimit() {
    TMultiGroupQuery q;
    q.Project = {0, 3};
    q.Where = TFilterExpression().Compare(2, EBinaryOp::Greater, I(15));
    q.Limit = 3;
    TQueryStatistics stats;
    const auto got = Run(q, &stats);
    EXPECT_EQ(Ints(got, 0), (std::vector<int64_t>{1, 2, 3}));
    EXPECT_TRUE(got.size() == 3 && Str(got[0][1]) == "apple" && got[1][1].Type == EValueType::Null && Str(got[2][1]) == "fig");
    EXPECT_EQ(stats.RowsRead, (int64_t)Rows.size());
    EXPECT_EQ(stats.RowsWritten, (int64_t)3);
    // the WhereOp form, and no LIMIT: every row it keeps
    TMultiGroupQuery w;
    w.Project = {0};
    w.WhereColumn = 2;
    w.WhereOp = EBinaryOp::Less;
    w.WhereConstant = I(35);
    EXPECT_EQ(Ints(Run(w), 0), (std::vector<int64_t>{0, 1, 2, 4}));
}

// SELECT id FROM t ORDER BY k DESC, v LIMIT 100: NULLs of a DESC item come last; OFFSET 2 LIMIT 3 cuts that order
void TestOrderByTwoItemsWithNulls() {
    TMultiGroupQuery q;
    q.Project = {0, 1, 2};
    q.OrderBy = {ByColumn(1, true), ByColumn(2)};
    q.Limit = 100;
    q.Select = std::vector<TExpression>{TExpression().Column(0)};
    EXPECT_EQ(Ints(Run(q), 0), (std::vector<int64_t>{0, 3, 4, 7, 2, 5, 1, 6}));
    q.OrderBy = {ByColumn(1), ByColumn(2, true)};  // ascending: NULLs first
    EXPECT_EQ(Ints(Run(q), 0), (std::vector<int64_t>{6, 1, 5, 2, 7, 4, 3, 0}));
    q.Offset = 2;
    q.Limit = 3;
    TQueryStatistics stats;
    EXPECT_EQ(Ints(Run(q, &stats), 0), (std::vector<int64_t>{5, 2, 7}));
    EXPECT_EQ(stats.RowsWritten, (int64_t)3);
    q.Offset = 7;
    EXPECT_EQ(Ints(Run(q), 0), (std::vector<int64_t>{0}));
    q.Offset = 8;
    EXPECT_EQ(Run(q).size(), (size_t)0);
    // an expression item: ORDER BY -d (-0.0 equals +0.0: ids 1 and 3 keep their order)
    TMultiGroupQuery e;
    e.Project = {0, 4};
    e.OrderBy = {By(TExpression().Column(1).Neg())};
    e.Limit = 8;
    EXPECT_EQ(Ints(Run(e), 0), (std::vector<int64_t>{4, 6, 2, 0, 7, 1, 3, 5}));
}

// SELECT k, sum(v) + 1 FROM t GROUP BY k HAVING count(v) > 1 ORDER BY sum(v) DESC LIMIT 2
void TestGroupByOrderBySumDesc() {
    TMultiGroupQuery q;
    q.GroupColumns = {1};
    q.AggregateItems = {{EAggregateFunction::Sum, 2}, {EAggregateFunction::Count, 2}};
    q.Having = TExpression().Column(2).Constant(I(1)).Compare(EBinaryOp::Greater);
    q.OrderBy = {ByColumn(1, true)};
    q.Limit = 2;
    q.Select = std::vector<TExpression>{TExpression().Column(0), TExpression().Column(1).Constant(I(1)).Add()};
    // groups first-seen: 3 (50), NULL (90), 1 (90), 2 (80); all have two rows; sum DESC, ties in first-seen order
    TQueryStatistics stats;
    const auto got = Run(q, &stats);
    EXPECT_EQ(Ints(got, 0), (std::vector<int64_t>{-999, 1}));
    EXPECT_EQ(Ints(got, 1), (std::vector<int64_t>{91, 91}));
    EXPECT_EQ(stats.RowsWritten, (int64_t)2);
    // LIMIT without ORDER BY: the first groups HAVING keeps, in first-seen order
    q.OrderBy.clear();
    q.Having = TExpression().Column(1).Constant(I(60)).Compare(EBinaryOp::Greater);
    EXPECT_EQ(Ints(Run(q), 0), (std::vector<int64_t>{-999, 1}));
    // an expression over the output row: ORDER BY sum(v) - 100 * k, and OFFSET
    q.Having.reset();
    q.OrderBy = {By(TExpression().Column(1).Constant(I(100)).Column(0).Mul().Sub())};
    q.Limit = 10;
    q.Offset = 1;
    EXPECT_EQ(Ints(Run(q), 0), (std::vector<int64_t>{3, 2, 1}));  // sums - 100k: 3 -> -250, NULL -> NULL, 1 -> -10, 2 -> -120
}

// SELECT name, count(v) FROM t GROUP BY name ORDER BY name LIMIT 10 / min(name) DESC
void TestOrderByStringGroupKey() {
    TMultiGroupQuery q;
    q.GroupColumns = {3};
    q.AggregateItems = {{EAggregateFunction::Count, 2}};
    q.OrderBy = {ByColumn(0)};
    q.Limit = 10;
    const auto got = Run(q);
    std::vector<std::string> names;
    for (const auto& r : got) names.push_back(Str(r[0]));
    EXPECT_EQ(names, (std::vector<std::string>{"<null>", "apple", "date", "fig", "kiwi", "pear"}));
    EXPECT_EQ(Ints(got, 1), (std::vector<int64_t>{1, 2, 1, 2, 1, 1}));
    // a string MIN by k, ordered DESC
    TMultiGroupQuery m;
    m.GroupColumns = {1};
    m.AggregateItems = {{EAggregateFunction::Min, 3}};
    m.OrderBy = {ByColumn(1, true)};
    m.Limit = 2;
    const auto got2 = Run(m);
    EXPECT_TRUE(got2.size() == 2 && Str(got2[0][1]) == "kiwi" && Str(got2[1][1]) == "fig");  // fig, apple, kiwi, apple
}

// SELECT concat(name, "!") AS c FROM t ORDER BY c DESC LIMIT 4
void TestProjectedStringComputedColumn() {
    TMultiGroupQuery q;
    q.Computed = {TExpression().Column(3).Constant(MakeUnversionedStringValue("!")).Concat()};
    q.Project = {TMultiGroupQuery::ComputedColumn(0), 0};
    q.OrderBy = {ByColumn(0, true)};
    q.Limit = 4;
    const auto got = Run(q);
    std::vector<std::string> names;
    for (const auto& r : got) names.push_back(Str(r[0]));
    EXPECT_EQ(names, (std::vector<std::string>{"pear!", "kiwi!", "fig!", "fig!"}));
    EXPECT_EQ(Ints(got, 1), (std::vector<int64_t>{0, 5, 3, 7}));
}

// SELECT t.id, d.w FROM t JOIN d ON t.k = d.k ORDER BY d.w DESC, t.id LIMIT 10
void TestJoinProjectionOrderedByForeignColumn() {
    std::vector<TUnversionedOwningRow> dims;
    for (auto [k, w] : std::vector<std::pair<int64_t, int64_t>>{{1, 5}, {2, 9}, {3, 7}}) {
        TUnversionedOwningRowBuilder b;
        b.AddValue(MakeUnversionedInt64Value(k, 0));
        b.AddValue(MakeUnversionedInt64Value(w, 1));
        dims.push_back(b.FinishRow());
    }
    TMultiGroupQuery q;
    q.Join = TMultiGroupQuery::TJoinClause{CreateInMemoryReader(dims), {1}, {0}, false};
    q.Project = {0, F(1)};
    q.OrderBy = {ByColumn(1, true), ByColumn(0)};
    q.Limit = 10;
    const auto got = Run(q);
    EXPECT_EQ(Ints(got, 0), (std::vector<int64_t>{4, 7, 0, 3, 2, 5}));
    EXPECT_EQ(Ints(got, 1), (std::vector<int64_t>{9, 9, 7, 7, 5, 5}));
}

// SELECT 100 / v FROM t ORDER BY v DESC LIMIT 3: row 4 has v = 0 but is not in the window; LIMIT 8 takes it in
void TestSelectDivisionOutsideWindow() {
    TMultiGroupQuery q;
    q.Project = {2};
    q.OrderBy = {ByColumn(0, true)};
    q.Limit = 3;
    q.Select = std::vector<TExpression>{TExpression().Constant(I(100)).Column(0).Div()};
    EXPECT_EQ(Ints(Run(q), 0), (std::vector<int64_t>{1, 1, 1}));
    q.Limit = 8;
    EXPECT_EQ(RunCode(q), (int)YTGPU_ERR_INVALID_ARGUMENT);
    // grouped: the group with sum 0 is outside the window
    TMultiGroupQuery g;
    g.GroupColumns = {0};
    g.AggregateItems = {{EAggregateFunction::Sum, 2}};
    g.OrderBy = {ByColumn(1, true)};
    g.Limit = 2;
    g.Select = std::vector<TExpression>{TExpression().Constant(I(800)).Column(1).Div()};
    EXPECT_EQ(Ints(Run(g), 0), (std::vector<int64_t>{10, 11}));
    g.Limit = 8;
    EXPECT_EQ(RunCode(g), (int)YTGPU_ERR_INVALID_ARGUMENT);
}

void TestRefusals() {
    auto base = [] {
        TMultiGroupQuery q;
        q.Project = {0};
        return q;
    };
    TMultiGroupQuery q = base();
    q.OrderBy = {ByColumn(0)};
    EXPECT_EQ(RunCode(q), (int)YTGPU_ERR_INVALID_ARGUMENT);  // ORDER BY used without LIMIT
    q = base();
    q.Offset = 1;
    q.Limit = 5;
    EXPECT_EQ(RunCode(q), (int)YTGPU_ERR_INVALID_ARGUMENT);  // OFFSET without ORDER BY
    q = base();
    q.Limit = -1;
    EXPECT_EQ(RunCode(q), (int)YTGPU_ERR_INVALID_ARGUMENT);
    q = base();
    q.OrderBy = {ByColumn(0)};
    q.Limit = 1;
    q.Offset = -1;
    EXPECT_EQ(RunCode(q), (int)YTGPU_ERR_INVALID_ARGUMENT);
    q = base();
    q.Having = TExpression().Column(0).Constant(I(0)).Compare(EBinaryOp::Greater);
    EXPECT_EQ(RunCode(q), (int)YTGPU_ERR_INVALID_ARGUMENT);  // HAVING without GROUP BY
    q = base();
    q.GroupColumns = {1};
    EXPECT_EQ(RunCode(q), (int)YTGPU_ERR_INVALID_ARGUMENT);  // Project with group items
    q = base();
    q.AggregateItems = {{EAggregateFunction::Sum, 2}};
    EXPECT_EQ(RunCode(q), (int)YTGPU_ERR_INVALID_ARGUMENT);
    q = TMultiGroupQuery{};
    q.Limit = 3;
    EXPECT_EQ(RunCode(q), (int)YTGPU_ERR_INVALID_ARGUMENT);  // neither Project nor GROUP BY
    q = base();
    q.OrderBy = {ByColumn(1)};
    q.Limit = 3;
    EXPECT_EQ(RunCode(q), (int)YTGPU_ERR_INVALID_ARGUMENT);  // no output position 1
    q = base();
    q.Project = {3};
    q.OrderBy = {By(TExpression().Column(0).Lower())};
    q.Limit = 3;
    EXPECT_EQ(RunCode(q), (int)YTGPU_ERR_UNSUPPORTED);  // a string function over the output row
    q = base();
    q.Project = {3};
    q.OrderBy = {By(TExpression().Column(0).Constant(I(1)).Add())};
    q.Limit = 3;
    EXPECT_EQ(RunCode(q), (int)YTGPU_ERR_UNSUPPORTED);  // arithmetic on a string position
    // the same items and Select over an empty input, or with an empty window, are refused alike
    auto emptyCode = [](const TMultiGroupQuery& query) {
        try {
            Run(query, nullptr, {});
        } catch (const TErrorException& e) {
            return e.GetCode();
        }
        return 0;
    };
    q = base();
    q.OrderBy = {ByColumn(1)};
    q.Limit = 3;
    EXPECT_EQ(emptyCode(q), (int)YTGPU_ERR_INVALID_ARGUMENT);  // no output position 1
    q.Limit = 0;
    EXPECT_EQ(RunCode(q), (int)YTGPU_ERR_INVALID_ARGUMENT);
    // a string position: without rows an input column has no type, a computed string column has one
    const auto concat = TExpression().Column(3).Constant(MakeUnversionedStringValue("!")).Concat();
    q = base();
    q.Computed = {concat};
    q.Project = {TMultiGroupQuery::ComputedColumn(0)};
    q.OrderBy = {By(TExpression().Column(0).Constant(I(1)).Add())};
    q.Limit = 3;
    EXPECT_EQ(emptyCode(q), (int)YTGPU_ERR_UNSUPPORTED);  // arithmetic on a string position
    q.Offset = 8;
    EXPECT_EQ(RunCode(q), (int)YTGPU_ERR_UNSUPPORTED);
    q = base();
    q.Computed = {concat};
    q.Project = {TMultiGroupQuery::ComputedColumn(0)};
    q.Select = std::vector<TExpression>{TExpression().Column(0).Lower()};
    EXPECT_EQ(emptyCode(q), (int)YTGPU_ERR_UNSUPPORTED);  // a string function in Select
    q.Limit = 0;
    EXPECT_EQ(RunCode(q), (int)YTGPU_ERR_UNSUPPORTED);
    q = base();
    q.Select = std::vector<TExpression>{TExpression().Column(2)};
    EXPECT_EQ(emptyCode(q), (int)YTGPU_ERR_INVALID_ARGUMENT);  // no output position 2
    q = base();  // a well-formed query over an empty input writes nothing
    q.Project = {0, 3};
    q.OrderBy = {ByColumn(1, true), By(TExpression().Column(0).Neg())};
    q.Limit = 3;
    q.Select = std::vector<TExpression>{TExpression().Column(0).Constant(I(1)).Add()};
    EXPECT_EQ(emptyCode(q), 0);
    EXPECT_EQ(Run(q, nullptr, {}).size(), (size_t)0);
    q = base();
    for (int i = 0; i < 33; ++i) q.OrderBy.push_back(ByColumn(0));
    q.Limit = 3;
    EXPECT_EQ(RunCode(q), (int)YTGPU_ERR_INVALID_ARGUMENT);  // more than 32 items
}

// The comparator of the random test, restated: NULL first, then the value; DESC reverses both; doubles with NaN above
// +inf (all NaNs equal) and -0.0 equal to +0.0; strings as unsigned bytes, a prefix first.
struct TRandomRow { int64_t Id; std::optional<int64_t> A; std::optional<double> B; std::optional<std::string> C; };

int CompareDouble(double x, double y) {
    const bool nx = std::isnan(x), ny = std::isnan(y);
    if (nx || ny) return (int)nx - (int)ny;
    return (x > y) - (x < y);
}

void TestRandomAgainstStableSort() {
    std::mt19937_64 rng(12345);
    const size_t n = 25000;  // three reader batches
    std::vector<TRandomRow> rows(n);
    std::vector<TUnversionedOwningRow> owned;
    const double doubles[] = {0.0, -0.0, 1.0, -1.0, INFINITY, -INFINITY, NAN, -NAN, 2.5, 1e-310};
    const char* strings[] = {"", "a", "ab", "abc", "b", "\xff", "a\x01", "zz"};
    for (size_t i = 0; i < n; ++i) {
        auto& r = rows[i];
        r.Id = (int64_t)i;
        if (rng() % 7) r.A = (int64_t)(rng() % 11) - 5;
        if (rng() % 9) r.B = doubles[rng() % 10];
        if (rng() % 5) r.C = strings[rng() % 8];
        TUnversionedOwningRowBuilder b;
        b.AddValue(MakeUnversionedInt64Value(r.Id, 0));
        b.AddValue(r.A ? MakeUnversionedInt64Value(*r.A, 1) : MakeUnversionedNullValue(1));
        b.AddValue(r.B ? MakeUnversionedDoubleValue(*r.B, 2) : MakeUnversionedNullValue(2));
        b.AddValue(r.C ? MakeUnversionedStringValue(*r.C, 3) : MakeUnversionedNullValue(3));
        owned.push_back(b.FinishRow());
    }
    TMultiGroupQuery q;
    q.Project = {0, 1, 2, 3};
    q.Where = TFilterExpression().Compare(0, EBinaryOp::NotEqual, I(7));
    q.OrderBy = {ByColumn(3), ByColumn(1, true), ByColumn(2)};
    q.Offset = 100;
    q.Limit = 20000;
    q.Select = std::vector<TExpression>{TExpression().Column(0)};
    const auto got = Run(q, nullptr, owned);

    auto cmpOpt = [](const auto& x, const auto& y, auto cmp) {
        if (!x || !y) return (int)(bool)x - (int)(bool)y;
        return cmp(*x, *y);
    };
    std::vector<TRandomRow> want;
    for (const auto& r : rows)
        if (r.Id != 7) want.push_back(r);
    std::stable_sort(want.begin(), want.end(), [&](const TRandomRow& x, const TRandomRow& y) {
        int c = cmpOpt(x.C, y.C, [](const std::string& a, const std::string& b) { return a.compare(b) < 0 ? -1 : a.compare(b) > 0 ? 1 : 0; });
        if (c == 0) c = -cmpOpt(x.A, y.A, [](int64_t a, int64_t b) { return (a > b) - (a < b); });
        if (c == 0) c = cmpOpt(x.B, y.B, CompareDouble);
        return c < 0;
    });
    std::vector<int64_t> wantIds;
    for (size_t i = 100; i < std::min<size_t>(want.size(), 20100); ++i) wantIds.push_back(want[i].Id);
    EXPECT_EQ(Ints(got, 0), wantIds);
}

}  // namespace

int main() {
    try {
        TestProjectionWhereLimit();
        TestOrderByTwoItemsWithNulls();
        TestGroupByOrderBySumDesc();
        TestOrderByStringGroupKey();
        TestProjectedStringComputedColumn();
        TestJoinProjectionOrderedByForeignColumn();
        TestSelectDivisionOutsideWindow();
        TestRefusals();
        TestRandomAgainstStableSort();
    } catch (const std::exception& e) {
        std::fprintf(stderr, "unexpected exception: %s\n", e.what());
        return 100;
    }
    std::printf("order_ut: %d failure(s)\n", Failures);
    return Failures;
}
