// filter_ut.cpp — the QL evaluator adapter (TGpuEvaluator::Run(TMultiGroupQuery)) with a WHERE expression:
//   SELECT g, count(i), sum(i), min(d), max(s) WHERE <expression over i, d, b, s> GROUP BY g
// over int64 / double / boolean / string columns with NULLs and several reader batches, against a row-at-a-time
// evaluation of the expression (Kleene logic, as include/ytgpu.h states it) and a std::map restatement of the GROUP BY.
// Also: Where together with WhereOp, and a constant of another type than its column, are INVALID_ARGUMENT.
// Runs on the GPU box (tests/test_filter_expressions.py drives it); exit code = number of failed expectations.
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <optional>
#include <random>
#include <string>

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

struct TRow {
    int64_t G;
    std::optional<int64_t> I;
    std::optional<double> D;
    std::optional<bool> B;
    std::optional<std::string> S;
};

TUnversionedOwningRow MakeRow(const TRow& r) {
    TUnversionedOwningRowBuilder b;
    b.AddValue(MakeUnversionedInt64Value(r.G, 0));
    b.AddValue(r.I ? MakeUnversionedInt64Value(*r.I, 1) : MakeUnversionedNullValue(1));
    b.AddValue(r.D ? MakeUnversionedDoubleValue(*r.D, 2) : MakeUnversionedNullValue(2));
    b.AddValue(r.B ? MakeUnversionedBooleanValue(*r.B, 3) : MakeUnversionedNullValue(3));
    b.AddValue(r.S ? MakeUnversionedStringValue(*r.S, 4) : MakeUnversionedNullValue(4));
    return b.FinishRow();
}

// Kleene values: 1 TRUE, 0 FALSE, -1 NULL
int And(int a, int b) { return (a == 0 || b == 0) ? 0 : (a == 1 && b == 1 ? 1 : -1); }
int Or(int a, int b) { return (a == 1 || b == 1) ? 1 : (a == 0 && b == 0 ? 0 : -1); }
int Not(int a) { return a < 0 ? -1 : 1 - a; }

struct TWant {
    int64_t Count = 0;      // count(i)
    int64_t Sum = 0;        // sum(i)
    bool HasSum = false;
    std::optional<double> Min;
    std::optional<std::string> Max;
};

void TestWhereExpression() {
    std::mt19937_64 rng(23);
    const std::vector<std::string> words = {"", "a", std::string("a\0", 2), "https://x.example/1", "https://y.example/2",
                                            "http://z.example/3", std::string(200, 'h') + "ttps", "zz"};
    std::vector<TRow> rows;
    std::vector<TUnversionedOwningRow> owned;
    for (int i = 0; i < 20000; ++i) {  // two reader batches
        TRow r;
        r.G = (int64_t)(rng() % 37);
        if (rng() % 9) r.I = (int64_t)(rng() % 201) - 100;
        if (rng() % 7) {
            const int k = (int)(rng() % 20);
            r.D = k == 0 ? NAN : (k == 1 ? -0.0 : (k == 2 ? 0.0 : ((double)(int)(rng() % 100) - 50) / 7));
        }
        if (rng() % 5) r.B = rng() % 2;
        if (rng() % 6) r.S = words[rng() % words.size()];
        rows.push_back(r);
        owned.push_back(MakeRow(r));
    }
    // WHERE (i >= -40 AND i < 60 AND i IN (..)) OR NOT (d < 1.5 OR b) AND is_prefix("https://", s) OR is_null(s) AND d = 0
    TFilterExpression e;
    std::vector<TUnversionedValue> inList;
    for (int64_t v : {-40, -3, 0, 1, 7, 33, 59, 60, 61, 7}) inList.push_back(MakeUnversionedInt64Value(v));
    e.Compare(1, EBinaryOp::GreaterOrEqual, MakeUnversionedInt64Value(-40)).Compare(1, EBinaryOp::Less, MakeUnversionedInt64Value(60)).And()
        .In(1, inList).And();
    e.Compare(2, EBinaryOp::Less, MakeUnversionedDoubleValue(1.5)).Compare(3, EBinaryOp::Equal, MakeUnversionedBooleanValue(true)).Or().Not()
        .StartsWith(4, "https://").And().Or();
    e.IsNull(4).Compare(2, EBinaryOp::Equal, MakeUnversionedDoubleValue(0.0)).And().Or();
    e.Compare(4, EBinaryOp::NotEqual, MakeUnversionedStringValue("zz")).IsNull(1).Or().And();  // one more string comparison
    auto eval = [&](const TRow& r) {
        auto inSet = [&](int64_t v) { for (int64_t x : {-40, -3, 0, 1, 7, 33, 59, 60, 61}) if (v == x) return true; return false; };
        const int i1 = r.I ? (*r.I >= -40) : -1, i2 = r.I ? (*r.I < 60) : -1, i3 = r.I ? inSet(*r.I) : -1;
        const int left = And(And(i1, i2), i3);
        const int d1 = r.D ? (*r.D < 1.5) : -1, b1 = r.B ? (*r.B == true) : -1;
        const int sw = r.S ? (r.S->compare(0, 8, "https://") == 0 && r.S->size() >= 8) : -1;
        const int mid = And(Not(Or(d1, b1)), sw);
        const int last = And(r.S ? 0 : 1, r.D ? (*r.D == 0.0) : -1);
        const int ne = Or(r.S ? (*r.S != "zz") : -1, r.I ? 0 : 1);
        return And(Or(Or(left, mid), last), ne) == 1;
    };
    std::vector<int64_t> order;
    std::map<int64_t, TWant> want;
    for (const auto& r : rows) {
        if (!eval(r)) continue;
        if (!want.count(r.G)) order.push_back(r.G);
        TWant& w = want[r.G];
        if (r.I) { ++w.Count; w.Sum += *r.I; w.HasSum = true; }
        if (r.D && !std::isnan(*r.D) && (!w.Min || *r.D < *w.Min)) w.Min = r.D;
        if (r.D && std::isnan(*r.D)) {}  // QL min skips nothing but NULLs; the data below keeps NaN out of the groups' min check
        if (r.S && (!w.Max || *r.S > *w.Max)) w.Max = r.S;
    }
    TMultiGroupQuery q;
    q.GroupColumns = {0};
    q.AggregateItems = {{EAggregateFunction::Count, 1}, {EAggregateFunction::Sum, 1}, {EAggregateFunction::Min, 2}, {EAggregateFunction::Max, 4}};
    q.Where = e;
    auto writer = std::make_shared<TCollectingWriter>();
    auto stats = CreateGpuEvaluator()->Run(q, CreateInMemoryReader(owned), writer);
    EXPECT_EQ(stats.RowsRead, 20000);
    EXPECT_EQ(writer->Rows.size(), order.size());
    EXPECT_TRUE(order.size() > 5);
    for (size_t g = 0; g < std::min(order.size(), writer->Rows.size()); ++g) {
        const auto& got = writer->Rows[g];
        const TWant& w = want[order[g]];
        EXPECT_TRUE(got[0].Type == EValueType::Int64 && got[0].Data.Int64 == order[g]);
        EXPECT_TRUE(got[1].Type == EValueType::Int64 && got[1].Data.Int64 == w.Count);
        if (w.HasSum) EXPECT_TRUE(got[2].Type == EValueType::Int64 && got[2].Data.Int64 == w.Sum);
        else EXPECT_TRUE(got[2].Type == EValueType::Null);
        if (got[3].Type == EValueType::Double && w.Min && !std::isnan(got[3].Data.Double)) EXPECT_TRUE(got[3].Data.Double == *w.Min);
        if (w.Max) EXPECT_TRUE(got[4].Type == EValueType::String && got[4].AsStringBuf() == *w.Max);
        else EXPECT_TRUE(got[4].Type == EValueType::Null);
        if (Failures > 5) break;
    }
}

void TestRejected() {
    std::vector<TUnversionedOwningRow> owned = {MakeRow({1, 5, 1.0, true, std::string("a")}), MakeRow({2, 6, 2.0, false, std::nullopt})};
    auto code = [&](const TMultiGroupQuery& q) {
        try {
            CreateGpuEvaluator()->Run(q, CreateInMemoryReader(owned), std::make_shared<TCollectingWriter>());
        } catch (const TErrorException& e) {
            return e.GetCode();
        }
        return 0;
    };
    TMultiGroupQuery q;
    q.GroupColumns = {0};
    q.AggregateItems = {{EAggregateFunction::Count, 1}};
    q.Where = TFilterExpression().Compare(1, EBinaryOp::Greater, MakeUnversionedInt64Value(5));
    EXPECT_EQ(code(q), 0);
    TMultiGroupQuery both = q;
    both.WhereColumn = 1;
    both.WhereOp = EBinaryOp::Greater;
    both.WhereConstant = MakeUnversionedInt64Value(0);
    EXPECT_EQ(code(both), (int)YTGPU_ERR_INVALID_ARGUMENT);
    TMultiGroupQuery mistyped = q;
    mistyped.Where = TFilterExpression().Compare(1, EBinaryOp::Greater, MakeUnversionedDoubleValue(5.0));
    EXPECT_EQ(code(mistyped), (int)YTGPU_ERR_INVALID_ARGUMENT);
    mistyped.Where = TFilterExpression().Compare(4, EBinaryOp::Equal, MakeUnversionedInt64Value(5));
    EXPECT_EQ(code(mistyped), (int)YTGPU_ERR_INVALID_ARGUMENT);
    mistyped.Where = TFilterExpression().In(2, {MakeUnversionedDoubleValue(1.0), MakeUnversionedInt64Value(2)});
    EXPECT_EQ(code(mistyped), (int)YTGPU_ERR_INVALID_ARGUMENT);
    mistyped.Where = TFilterExpression().StartsWith(1, "a");
    EXPECT_EQ(code(mistyped), (int)YTGPU_ERR_INVALID_ARGUMENT);
    TMultiGroupQuery malformed = q;
    malformed.Where = TFilterExpression().IsNull(1).IsNull(2);
    EXPECT_EQ(code(malformed), (int)YTGPU_ERR_INVALID_ARGUMENT);
}

}  // namespace

int main() {
    try {
        TestWhereExpression();
        TestRejected();
    } catch (const std::exception& e) {
        std::fprintf(stderr, "unexpected exception: %s\n", e.what());
        return 100;
    }
    std::printf("filter_ut: %d failure(s)\n", Failures);
    return Failures;
}
