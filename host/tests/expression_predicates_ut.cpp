// expression_predicates_ut.cpp — the QL evaluator adapter (TGpuEvaluator::Run(TMultiGroupQuery)) with in / is_prefix /
// is_substr / like inside computed columns, Select and Having, against row-at-a-time restatements:
//   * sum(if(status in (200, 201, 204), 1, 0)) and sum(if(k in (1, 3), v, 0));
//   * GROUP BY lower(url) like '%/api/%' and GROUP BY if(is_prefix('https://', url), 'tls', 'plain');
//   * Having max(status) in (404, 500) and a Select item max(status) in (500);
//   * an input column that is NULL in every row under each op;
//   * a mistyped list entry (INVALID_ARGUMENT) and a string predicate over the output row (UNSUPPORTED).
// Runs on the GPU box (tests/test_expression_predicates.py drives it); exit code = number of failed expectations.
#include <algorithm>
#include <cctype>
#include <cstdio>
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

std::vector<TUnversionedOwningRow> Run(const TMultiGroupQuery& q, const std::vector<TUnversionedOwningRow>& rows) {
    auto writer = std::make_shared<TCollectingWriter>();
    CreateGpuEvaluator()->Run(q, CreateInMemoryReader(rows), writer);
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

TUnversionedValue I(int64_t x) { return MakeUnversionedInt64Value(x); }

// input positions: 0 k, 1 status (nullable), 2 v, 3 url (nullable string), 4 n (NULL in every row)
struct TRow { int64_t K; std::optional<int64_t> Status; int64_t V; std::optional<std::string> Url; };

std::vector<TUnversionedOwningRow> Owned(const std::vector<TRow>& rows) {
    std::vector<TUnversionedOwningRow> owned;
    for (const auto& r : rows) {
        TUnversionedOwningRowBuilder b;
        b.AddValue(MakeUnversionedInt64Value(r.K, 0));
        b.AddValue(r.Status ? MakeUnversionedInt64Value(*r.Status, 1) : MakeUnversionedNullValue(1));
        b.AddValue(MakeUnversionedInt64Value(r.V, 2));
        b.AddValue(r.Url ? MakeUnversionedStringValue(*r.Url, 3) : MakeUnversionedNullValue(3));
        b.AddValue(MakeUnversionedNullValue(4));
        owned.push_back(b.FinishRow());
    }
    return owned;
}

std::vector<TRow> RandomRows(size_t count, uint64_t seed) {
    static const char* urls[] = {"https://a.example.com/API/v1", "http://b.example.com/x", "https://c/", "HTTP://D/api/", ""};
    static const int64_t statuses[] = {200, 201, 204, 404, 500};
    std::mt19937_64 rng(seed);
    std::vector<TRow> rows;
    for (size_t i = 0; i < count; ++i) {
        TRow r{(int64_t)(rng() % 5), std::nullopt, (int64_t)(rng() % 2001) - 1000, std::nullopt};
        if (rng() % 9) r.Status = statuses[rng() % 5];
        if (rng() % 7) r.Url = urls[rng() % 5];
        rows.push_back(r);
    }
    return rows;
}

std::string Lower(std::string s) {
    for (auto& ch : s) ch = (char)std::tolower((unsigned char)ch);
    return s;
}

// SELECT k, sum(if(status in (200, 201, 204), 1, 0)), sum(if(k in (1, 3), v, 0)) GROUP BY k
void TestConditionalSumOverIn() {
    const auto rows = RandomRows(20000, 7);
    TMultiGroupQuery q;
    q.Computed = {
        TExpression().Column(1).In({I(200), I(201), I(204)}).Constant(I(1)).Constant(I(0)).If(),
        TExpression().Column(0).In({I(1), I(3)}).Column(2).Constant(I(0)).If(),
    };
    q.GroupColumns = {0};
    q.AggregateItems = {{EAggregateFunction::Sum, TMultiGroupQuery::ComputedColumn(0)}, {EAggregateFunction::Sum, TMultiGroupQuery::ComputedColumn(1)}};
    const auto got = Run(q, Owned(rows));
    std::map<int64_t, std::pair<int64_t, int64_t>> want;
    for (const auto& r : rows) {
        auto& w = want[r.K];
        // a NULL status makes in() NULL, so if() takes neither branch: NULL, which sum skips
        w.first += r.Status && (*r.Status == 200 || *r.Status == 201 || *r.Status == 204) ? 1 : 0;
        w.second += r.K == 1 || r.K == 3 ? r.V : 0;
    }
    EXPECT_EQ(got.size(), want.size());
    for (const auto& row : got) {
        const auto& w = want[row[0].Data.Int64];
        EXPECT_TRUE(row[1].Type == EValueType::Int64 && row[1].Data.Int64 == w.first);
        EXPECT_TRUE(row[2].Type == EValueType::Int64 && row[2].Data.Int64 == w.second);
    }
}

// SELECT key, count(v) GROUP BY lower(url) like '%/api/%'; GROUP BY if(is_prefix('https://', url), 'tls', 'plain')
void TestPatternKeys() {
    const auto rows = RandomRows(8000, 11);
    TMultiGroupQuery q;
    q.Computed = {TExpression().Column(3).Lower().Like("%/api/%")};
    q.GroupColumns = {TMultiGroupQuery::ComputedColumn(0)};
    q.AggregateItems = {{EAggregateFunction::Count, 2}};
    auto got = Run(q, Owned(rows));
    std::map<int, int64_t> want;  // 0 false, 1 true, 2 NULL
    for (const auto& r : rows) ++want[!r.Url ? 2 : Lower(*r.Url).find("/api/") != std::string::npos ? 1 : 0];
    EXPECT_EQ(got.size(), want.size());
    for (const auto& row : got) {
        const int key = row[0].Type == EValueType::Null ? 2 : row[0].Data.Boolean ? 1 : 0;
        EXPECT_TRUE(row[0].Type == EValueType::Null || row[0].Type == EValueType::Boolean);
        EXPECT_EQ(row[1].Data.Int64, want[key]);
    }
    q.Computed = {TExpression().Column(3).IsPrefix("https://").Constant(MakeUnversionedStringValue("tls"))
                      .Constant(MakeUnversionedStringValue("plain")).If()};
    got = Run(q, Owned(rows));
    std::map<std::string, int64_t> swant;  // "" for NULL
    for (const auto& r : rows) ++swant[!r.Url ? "" : r.Url->rfind("https://", 0) == 0 ? "tls" : "plain"];
    EXPECT_EQ(got.size(), swant.size());
    for (const auto& row : got) {
        const std::string key = row[0].Type == EValueType::Null ? "" : std::string(row[0].Data.String, row[0].Length);
        EXPECT_EQ(row[1].Data.Int64, swant[key]);
    }
}

// SELECT k, max(status), max(status) in (500) GROUP BY k HAVING max(status) in (404, 500)
void TestHavingWithIn() {
    std::vector<TRow> rows;
    for (int64_t k = 0; k < 6; ++k)
        for (int64_t s : {200, 404, 500})
            if (s <= 200 + 150 * k) rows.push_back({k, s, 1, std::nullopt});
    TMultiGroupQuery q;
    q.GroupColumns = {0};
    q.AggregateItems = {{EAggregateFunction::Max, 1}};
    q.Having = TExpression().Column(1).In({I(404), I(500)});
    q.Select = std::vector<TExpression>{TExpression().Column(0), TExpression().Column(1), TExpression().Column(1).In({I(500)})};
    const auto got = Run(q, Owned(rows));
    std::map<int64_t, int64_t> maxOf;
    for (const auto& r : rows) maxOf[r.K] = std::max(maxOf[r.K], *r.Status);
    size_t kept = 0;
    for (const auto& [k, m] : maxOf) kept += m == 404 || m == 500;
    EXPECT_EQ(got.size(), kept);
    for (const auto& row : got) {
        const int64_t m = maxOf[row[0].Data.Int64];
        EXPECT_TRUE(m == 404 || m == 500);
        EXPECT_EQ(row[1].Data.Int64, m);
        EXPECT_TRUE(row[2].Type == EValueType::Boolean && row[2].Data.Boolean == (m == 500));
    }
    // checked whatever the data: a mistyped list on an empty input, a string predicate over the output row
    q.Having = TExpression().Column(1).In({MakeUnversionedUint64Value(404)});
    EXPECT_EQ(Code(q, {}), (int)YTGPU_ERR_INVALID_ARGUMENT);
    EXPECT_EQ(Code(q, Owned(rows)), (int)YTGPU_ERR_INVALID_ARGUMENT);
    q.Having = std::nullopt;
    q.Select = std::vector<TExpression>{TExpression().Column(0).IsPrefix("x")};
    EXPECT_EQ(Code(q, Owned(rows)), (int)YTGPU_ERR_UNSUPPORTED);
}

// an input column that is NULL in every row under each op: NULL, so is_null(...) counts every row
void TestAllNullInputColumn() {
    const auto rows = RandomRows(3000, 13);
    std::map<int64_t, int64_t> count;
    for (const auto& r : rows) ++count[r.K];
    const std::vector<TExpression> ops = {
        TExpression().Column(4).In({I(1), I(2)}), TExpression().Column(4).In({MakeUnversionedStringValue("a")}),
        TExpression().Column(4).In({MakeUnversionedDoubleValue(0.5)}), TExpression().Column(4).IsPrefix("x"),
        TExpression().Column(4).IsSubstr("x"), TExpression().Column(4).Like("%x%"),
    };
    for (const auto& op : ops) {
        TMultiGroupQuery q;
        TExpression e = op;
        e.IsNull().Constant(I(1)).Constant(I(0)).If();
        q.Computed = {e};
        q.GroupColumns = {0};
        q.AggregateItems = {{EAggregateFunction::Sum, TMultiGroupQuery::ComputedColumn(0)}};
        const auto got = Run(q, Owned(rows));
        EXPECT_EQ(got.size(), count.size());
        for (const auto& row : got) EXPECT_EQ(row[1].Data.Int64, count[row[0].Data.Int64]);
    }
}

// a list entry of another type than its operand, or of two types, or NULL, throws INVALID_ARGUMENT
void TestMistypedLists() {
    const auto rows = RandomRows(100, 17);
    TMultiGroupQuery q;
    q.GroupColumns = {0};
    q.AggregateItems = {{EAggregateFunction::Count, TMultiGroupQuery::ComputedColumn(0)}};
    for (const auto& e : {TExpression().Column(1).In({MakeUnversionedStringValue("200")}),
                          TExpression().Column(1).In({MakeUnversionedUint64Value(200)}),
                          TExpression().Column(1).In({I(200), MakeUnversionedDoubleValue(1.0)}),
                          TExpression().Column(1).In({I(200), MakeUnversionedNullValue()}),
                          TExpression().Column(3).In({I(1)})}) {
        q.Computed = {e};
        EXPECT_EQ(Code(q, Owned(rows)), (int)YTGPU_ERR_INVALID_ARGUMENT);
    }
    q.Computed = {TExpression().Column(1).IsPrefix("2")};  // a string predicate over an Int64
    EXPECT_EQ(Code(q, Owned(rows)), (int)YTGPU_ERR_INVALID_ARGUMENT);
}

}  // namespace

int main() {
    try {
        TestConditionalSumOverIn();
        TestPatternKeys();
        TestHavingWithIn();
        TestAllNullInputColumn();
        TestMistypedLists();
    } catch (const std::exception& e) {
        std::fprintf(stderr, "unexpected exception: %s\n", e.what());
        return 100;
    }
    std::printf("expression_predicates_ut: %d failure(s)\n", Failures);
    return Failures;
}
