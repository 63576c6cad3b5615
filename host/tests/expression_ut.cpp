// expression_ut.cpp — the QL evaluator adapter (TGpuEvaluator::Run(TMultiGroupQuery)) with computed columns and Select:
//   * ql_query_ut.cpp Complex (:4162-4194) and ComplexWithNull (:4261-4300) verbatim: group by a % 2 as x, sum(b) + x,
//     with a % 2 and sum(b) + x evaluated by ytgpu_evaluate_expression;
//   * a Where expression over a computed column;
//   * b / a where a = 0 only in rows the WHERE drops (no exception), and with such a row kept (an exception);
//   * random rows with NULLs over several reader batches against a row-at-a-time restatement of the expressions.
// Runs on the GPU box (tests/test_expressions.py drives it); exit code = number of failed expectations.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <optional>
#include <random>
#include <string>
#include <tuple>

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

using TOptInt = std::optional<int64_t>;

TUnversionedValue IntOrNull(TOptInt v, int id) { return v ? MakeUnversionedInt64Value(*v, id) : MakeUnversionedNullValue(id); }

std::vector<TUnversionedOwningRow> Rows(const std::vector<std::vector<TOptInt>>& rows) {
    std::vector<TUnversionedOwningRow> owned;
    for (const auto& r : rows) {
        TUnversionedOwningRowBuilder b;
        for (size_t c = 0; c < r.size(); ++c) b.AddValue(IntOrNull(r[c], (int)c));
        owned.push_back(b.FinishRow());
    }
    return owned;
}

std::vector<TUnversionedOwningRow> Run(const TMultiGroupQuery& q, const std::vector<TUnversionedOwningRow>& rows) {
    auto writer = std::make_shared<TCollectingWriter>();
    CreateGpuEvaluator()->Run(q, CreateInMemoryReader(rows), writer);
    return writer->Rows;
}

bool IsInt(const TUnversionedValue& v, int64_t x) { return v.Type == EValueType::Int64 && v.Data.Int64 == x; }
bool IsNull(const TUnversionedValue& v) { return v.Type == EValueType::Null; }

TExpression AMod2() { return TExpression().Column(0).Constant(MakeUnversionedInt64Value(2)).Mod(); }

// select x, sum(b) + x as t FROM [//t] where a > 1 group by a % 2 as x   (a = 1..9, b = 10 a)
void TestComplex() {
    std::vector<std::vector<TOptInt>> rows;
    for (int64_t a = 1; a <= 9; ++a) rows.push_back({a, 10 * a});
    TMultiGroupQuery q;
    q.Computed = {AMod2()};
    q.GroupColumns = {TMultiGroupQuery::ComputedColumn(0)};
    q.AggregateItems = {{EAggregateFunction::Sum, 1}};
    q.Where = TFilterExpression().Compare(0, EBinaryOp::Greater, MakeUnversionedInt64Value(1));
    q.Select = std::vector<TExpression>{TExpression().Column(0), TExpression().Column(1).Column(0).Add()};
    const auto got = Run(q, Rows(rows));
    EXPECT_EQ(got.size(), (size_t)2);
    if (got.size() != 2) return;
    EXPECT_EQ(got[0].GetCount(), 2);
    EXPECT_TRUE(IsInt(got[0][0], 0) && IsInt(got[0][1], 200));  // first seen: a = 2
    EXPECT_TRUE(IsInt(got[1][0], 1) && IsInt(got[1][1], 241));
    EXPECT_TRUE(got[0][1].Id == 1 && got[1][0].Id == 0);
    // the same WHERE as the built-in WhereOp: it runs as a one-node filter program before the computed key
    TMultiGroupQuery op = q;
    op.Where.reset();
    op.WhereColumn = 0;
    op.WhereOp = EBinaryOp::Greater;
    op.WhereConstant = MakeUnversionedInt64Value(1);
    op.AggregateItems = {{EAggregateFunction::Sum, 1}, {EAggregateFunction::Count, 0}};
    const auto got2 = Run(op, Rows(rows));
    EXPECT_EQ(got2.size(), (size_t)2);
    if (got2.size() == 2) EXPECT_TRUE(IsInt(got2[0][0], 0) && IsInt(got2[0][1], 200) && IsInt(got2[1][0], 1) && IsInt(got2[1][1], 241));
}

// select x, sum(b) + x as t, sum(b) as y FROM [//t] group by a % 2 as x   (a NULL in three rows, b NULL in one)
void TestComplexWithNull() {
    std::vector<std::vector<TOptInt>> rows;
    for (int64_t a = 1; a <= 9; ++a) rows.push_back({a, 10 * a});
    rows.push_back({10, std::nullopt});
    rows.push_back({std::nullopt, 1});
    rows.push_back({std::nullopt, 2});
    rows.push_back({std::nullopt, 3});
    TMultiGroupQuery q;
    q.Computed = {AMod2()};
    q.GroupColumns = {TMultiGroupQuery::ComputedColumn(0)};
    q.AggregateItems = {{EAggregateFunction::Sum, 1}};
    q.Select = std::vector<TExpression>{TExpression().Column(0), TExpression().Column(1).Column(0).Add(), TExpression().Column(1)};
    const auto got = Run(q, Rows(rows));
    EXPECT_EQ(got.size(), (size_t)3);
    if (got.size() != 3) return;
    EXPECT_TRUE(IsInt(got[0][0], 1) && IsInt(got[0][1], 251) && IsInt(got[0][2], 250));
    EXPECT_TRUE(IsInt(got[1][0], 0) && IsInt(got[1][1], 200) && IsInt(got[1][2], 200));
    EXPECT_TRUE(IsNull(got[2][0]) && IsNull(got[2][1]) && IsInt(got[2][2], 6));
}

// b / a where a = 0 only in rows the WHERE drops, and with such a row kept; a Where expression over a computed column
void TestDivisionAndWhereOverComputed() {
    std::vector<std::vector<TOptInt>> rows;  // g, a, b
    for (int64_t i = 0; i < 100; ++i) rows.push_back({i % 3, i % 10 == 0 ? 0 : i - 50, 7 * i});
    auto code = [&](const TMultiGroupQuery& q, std::string* message) {
        try {
            Run(q, Rows(rows));
        } catch (const TErrorException& e) {
            if (message) *message = e.what();
            return e.GetCode();
        }
        return 0;
    };
    TMultiGroupQuery q;
    q.Computed = {TExpression().Column(2).Column(1).Div()};
    q.GroupColumns = {0};
    q.AggregateItems = {{EAggregateFunction::Sum, TMultiGroupQuery::ComputedColumn(0)}, {EAggregateFunction::Count, 1}};
    q.Where = TFilterExpression().Compare(1, EBinaryOp::NotEqual, MakeUnversionedInt64Value(0));
    const auto got = Run(q, Rows(rows));
    std::map<int64_t, std::pair<int64_t, int64_t>> want;
    for (const auto& r : rows)
        if (*r[1] != 0) {
            want[*r[0]].first += *r[2] / *r[1];
            ++want[*r[0]].second;
        }
    EXPECT_EQ(got.size(), want.size());
    for (const auto& row : got) EXPECT_TRUE(IsInt(row[1], want[row[0].Data.Int64].first) && IsInt(row[2], want[row[0].Data.Int64].second));
    // the built-in WhereOp form drops the same rows
    TMultiGroupQuery op = q;
    op.Where.reset();
    op.WhereColumn = 1;
    op.WhereOp = EBinaryOp::NotEqual;
    op.WhereConstant = MakeUnversionedInt64Value(0);
    EXPECT_EQ(code(op, nullptr), 0);
    // a row with a = 0 kept: the query fails
    TMultiGroupQuery kept = q;
    kept.Where = TFilterExpression().Compare(1, EBinaryOp::GreaterOrEqual, MakeUnversionedInt64Value(0));
    std::string message;
    EXPECT_EQ(code(kept, &message), (int)YTGPU_ERR_INVALID_ARGUMENT);
    EXPECT_TRUE(message.find("Division by zero") != std::string::npos);
    TMultiGroupQuery none = q;
    none.Where.reset();
    EXPECT_EQ(code(none, nullptr), (int)YTGPU_ERR_INVALID_ARGUMENT);
    // WHERE a + b > 100 over a computed column, grouped by it modulo 4
    TMultiGroupQuery w;
    w.Computed = {TExpression().Column(1).Column(2).Add(), TExpression().Column(1).Column(2).Add().Constant(MakeUnversionedInt64Value(4)).Mod()};
    w.GroupColumns = {TMultiGroupQuery::ComputedColumn(1)};
    w.AggregateItems = {{EAggregateFunction::Sum, 2}, {EAggregateFunction::Max, TMultiGroupQuery::ComputedColumn(0)}};
    w.Where = TFilterExpression().Compare(TMultiGroupQuery::ComputedColumn(0), EBinaryOp::Greater, MakeUnversionedInt64Value(100));
    const auto wgot = Run(w, Rows(rows));
    std::vector<int64_t> order;
    std::map<int64_t, std::pair<int64_t, int64_t>> wwant;
    for (const auto& r : rows) {
        const int64_t s = *r[1] + *r[2];
        if (s <= 100) continue;
        const int64_t k = s % 4;
        if (!wwant.count(k)) {
            order.push_back(k);
            wwant[k] = {0, s};
        }
        wwant[k].first += *r[2];
        wwant[k].second = std::max(wwant[k].second, s);
    }
    EXPECT_EQ(wgot.size(), order.size());
    for (size_t g = 0; g < std::min(order.size(), wgot.size()); ++g)
        EXPECT_TRUE(IsInt(wgot[g][0], order[g]) && IsInt(wgot[g][1], wwant[order[g]].first) && IsInt(wgot[g][2], wwant[order[g]].second));
    // mistyped expressions and arithmetic on a string are refused
    TMultiGroupQuery bad = q;
    bad.Computed = {TExpression().Column(2).Constant(MakeUnversionedUint64Value(2)).Add()};
    EXPECT_EQ(code(bad, nullptr), (int)YTGPU_ERR_INVALID_ARGUMENT);
    std::vector<TUnversionedOwningRow> strings;
    for (int i = 0; i < 4; ++i) {
        TUnversionedOwningRowBuilder b;
        b.AddValue(MakeUnversionedInt64Value(i % 2, 0));
        b.AddValue(MakeUnversionedStringValue(i % 2 ? "x" : "yy", 1));
        strings.push_back(b.FinishRow());
    }
    auto scode = [&](const TMultiGroupQuery& sq) {
        try {
            Run(sq, strings);
        } catch (const TErrorException& e) {
            return e.GetCode();
        }
        return 0;
    };
    TMultiGroupQuery s;
    s.GroupColumns = {0};
    s.AggregateItems = {{EAggregateFunction::Max, 1}};
    s.Select = std::vector<TExpression>{TExpression().Column(1), TExpression().Column(0)};
    EXPECT_EQ(scode(s), 0);
    const auto sgot = Run(s, strings);
    EXPECT_TRUE(sgot.size() == 2 && sgot[0][0].Type == EValueType::String && sgot[0][0].AsStringBuf() == "yy" && IsInt(sgot[0][1], 0));
    s.Select = std::vector<TExpression>{TExpression().Column(1).Column(1).Add()};
    EXPECT_EQ(scode(s), (int)YTGPU_ERR_UNSUPPORTED);
    TMultiGroupQuery sc;
    sc.Computed = {TExpression().Column(1).Neg()};
    sc.GroupColumns = {0};
    sc.AggregateItems = {{EAggregateFunction::Min, TMultiGroupQuery::ComputedColumn(0)}};
    EXPECT_EQ(scode(sc), (int)YTGPU_ERR_UNSUPPORTED);
}

// Random rows (g, a, b, d with NULLs) over several reader batches:
//   SELECT k, g, sum(c1), min(c2), max(a), count(c1) WHERE c1 > 0 OR is_null(c1) GROUP BY a % 5 AS k, g
//   with c1 = if_null(b, 0) * 3 - a, c2 = int64(d * 10.0)
void TestRandom() {
    std::mt19937_64 rng(41);
    struct TRow { int64_t G; TOptInt A, B; std::optional<double> D; };
    std::vector<TRow> rows;
    std::vector<TUnversionedOwningRow> owned;
    for (int i = 0; i < 25000; ++i) {
        TRow r{(int64_t)(rng() % 3), std::nullopt, std::nullopt, std::nullopt};
        if (rng() % 8) r.A = (int64_t)(rng() % 2001) - 1000;
        if (rng() % 6) r.B = (int64_t)(rng() % 2001) - 1000;
        if (rng() % 5) r.D = ((double)(int64_t)(rng() % 20001) - 10000) / 64.0;
        rows.push_back(r);
        TUnversionedOwningRowBuilder b;
        b.AddValue(MakeUnversionedInt64Value(r.G, 0));
        b.AddValue(IntOrNull(r.A, 1));
        b.AddValue(IntOrNull(r.B, 2));
        b.AddValue(r.D ? MakeUnversionedDoubleValue(*r.D, 3) : MakeUnversionedNullValue(3));
        owned.push_back(b.FinishRow());
    }
    TMultiGroupQuery q;
    q.Computed = {TExpression().Column(1).Constant(MakeUnversionedInt64Value(5)).Mod(),
                  TExpression().Column(2).Constant(MakeUnversionedInt64Value(0)).IfNull().Constant(MakeUnversionedInt64Value(3)).Mul().Column(1).Sub(),
                  TExpression().Column(3).Constant(MakeUnversionedDoubleValue(10.0)).Mul().Cast(EValueType::Int64)};
    const int k = TMultiGroupQuery::ComputedColumn(0), c1 = TMultiGroupQuery::ComputedColumn(1), c2 = TMultiGroupQuery::ComputedColumn(2);
    q.GroupColumns = {k, 0};
    q.AggregateItems = {{EAggregateFunction::Sum, c1}, {EAggregateFunction::Min, c2}, {EAggregateFunction::Max, 1}, {EAggregateFunction::Count, c1}};
    q.Where = TFilterExpression().Compare(c1, EBinaryOp::Greater, MakeUnversionedInt64Value(0)).IsNull(c1).Or();
    const auto got = Run(q, owned);
    struct TWant { TOptInt Sum, Min, Max; int64_t Count = 0; };
    std::vector<std::tuple<TOptInt, int64_t>> order;
    std::map<std::tuple<TOptInt, int64_t>, TWant> want;
    for (const auto& r : rows) {
        const TOptInt key = r.A ? TOptInt(*r.A % 5) : std::nullopt;
        const TOptInt v1 = r.A ? TOptInt((r.B ? *r.B : 0) * 3 - *r.A) : std::nullopt;
        const TOptInt v2 = r.D ? TOptInt((int64_t)(*r.D * 10.0)) : std::nullopt;
        if (!(v1 ? *v1 > 0 : true)) continue;
        const auto t = std::make_tuple(key, r.G);
        if (!want.count(t)) order.push_back(t);
        TWant& w = want[t];
        if (v1) { w.Sum = (w.Sum ? *w.Sum : 0) + *v1; ++w.Count; }
        if (v2 && (!w.Min || *v2 < *w.Min)) w.Min = v2;
        if (r.A && (!w.Max || *r.A > *w.Max)) w.Max = r.A;
    }
    auto same = [](const TUnversionedValue& v, TOptInt x) { return x ? IsInt(v, *x) : IsNull(v); };
    EXPECT_EQ(got.size(), order.size());
    EXPECT_TRUE(order.size() > 20);
    for (size_t g = 0; g < std::min(order.size(), got.size()); ++g) {
        const TWant& w = want[order[g]];
        EXPECT_TRUE(same(got[g][0], std::get<0>(order[g])) && IsInt(got[g][1], std::get<1>(order[g])));
        EXPECT_TRUE(same(got[g][2], w.Sum) && same(got[g][3], w.Min) && same(got[g][4], w.Max) && IsInt(got[g][5], w.Count));
        if (Failures > 5) break;
    }
}

}  // namespace

int main() {
    try {
        TestComplex();
        TestComplexWithNull();
        TestDivisionAndWhereOverComputed();
        TestRandom();
    } catch (const std::exception& e) {
        std::fprintf(stderr, "unexpected exception: %s\n", e.what());
        return 100;
    }
    std::printf("expression_ut: %d failure(s)\n", Failures);
    return Failures;
}
