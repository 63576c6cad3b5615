// like_ut.cpp — the QL evaluator adapter (TGpuEvaluator::Run(TMultiGroupQuery)) with CONTAINS and LIKE in the WHERE:
//   SELECT g, count(i), sum(i) WHERE is_substr("site4", u) AND NOT (u LIKE '%/item/\_%' ESCAPE '\') GROUP BY g
// over URL-like rows with NULLs and several reader batches, against a row-at-a-time evaluation on the host (Kleene logic
// and the LIKE rules of include/ytgpu.h) and a std::map restatement of the GROUP BY.  Also: CONTAINS / LIKE over a column
// without values selects nothing, and over an int64 column they are INVALID_ARGUMENT.
// Runs on the GPU box (tests/test_filter_patterns.py drives it); exit code = number of failed expectations.
#include <cstdio>
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
    std::optional<std::string> U;
    std::optional<int64_t> I;
};

TUnversionedOwningRow MakeRow(const TRow& r) {
    TUnversionedOwningRowBuilder b;
    b.AddValue(MakeUnversionedInt64Value(r.G, 0));
    b.AddValue(r.U ? MakeUnversionedStringValue(*r.U, 1) : MakeUnversionedNullValue(1));
    b.AddValue(r.I ? MakeUnversionedInt64Value(*r.I, 2) : MakeUnversionedNullValue(2));
    b.AddValue(MakeUnversionedNullValue(3));  // a column without values
    return b.FinishRow();
}

// LIKE over ASCII values and patterns (the values below are ASCII, so _ is one byte): plain backtracking is fine here.
bool Like(const std::string& s, size_t i, const std::string& p, size_t k, int escape) {
    if (k == p.size()) return i == s.size();
    if (p[k] == '%') {
        for (size_t j = i; j <= s.size(); ++j)
            if (Like(s, j, p, k + 1, escape)) return true;
        return false;
    }
    if (i == s.size()) return false;
    if ((unsigned char)p[k] == escape) return s[i] == p[k + 1] && Like(s, i + 1, p, k + 2, escape);
    return (p[k] == '_' || s[i] == p[k]) && Like(s, i + 1, p, k + 1, escape);
}

int Code(const TMultiGroupQuery& q, const std::vector<TUnversionedOwningRow>& owned, size_t* rowsOut = nullptr) {
    auto writer = std::make_shared<TCollectingWriter>();
    try {
        CreateGpuEvaluator()->Run(q, CreateInMemoryReader(owned), writer);
    } catch (const TErrorException& e) {
        return e.GetCode();
    }
    if (rowsOut) *rowsOut = writer->Rows.size();
    return 0;
}

void TestContainsAndNotLike() {
    std::mt19937_64 rng(29);
    std::vector<TRow> rows;
    std::vector<TUnversionedOwningRow> owned;
    const char* paths[] = {"/item/", "/item/_x", "/item/ab", "/items", "/q/item/_", "/", ""};
    for (int i = 0; i < 20000; ++i) {  // two reader batches
        TRow r;
        r.G = (int64_t)(rng() % 23);
        if (rng() % 8) {
            r.U = std::string(rng() % 2 ? "https://" : "http://") + "www.site" + std::to_string(rng() % 10) + ".example.com" +
                  paths[rng() % 7] + std::string(rng() % 5, 'q');
        }
        if (rng() % 9) r.I = (int64_t)(rng() % 2001) - 1000;
        rows.push_back(r);
        owned.push_back(MakeRow(r));
    }
    const std::string pattern = "%/item/\\_%";
    std::vector<int64_t> order;
    std::map<int64_t, std::pair<int64_t, int64_t>> want;  // count(i), sum(i)
    for (const auto& r : rows) {
        // NULL u: both leaves NULL, so the conjunction is NULL and the row is dropped
        if (!r.U || r.U->find("site4") == std::string::npos || Like(*r.U, 0, pattern, 0, '\\')) continue;
        if (!want.count(r.G)) order.push_back(r.G);
        if (r.I) {
            ++want[r.G].first;
            want[r.G].second += *r.I;
        } else {
            want[r.G];
        }
    }
    TMultiGroupQuery q;
    q.GroupColumns = {0};
    q.AggregateItems = {{EAggregateFunction::Count, 2}, {EAggregateFunction::Sum, 2}};
    q.Where = TFilterExpression().Contains(1, "site4").Like(1, pattern, '\\').Not().And();
    auto writer = std::make_shared<TCollectingWriter>();
    auto stats = CreateGpuEvaluator()->Run(q, CreateInMemoryReader(owned), writer);
    EXPECT_EQ(stats.RowsRead, 20000);
    EXPECT_EQ(writer->Rows.size(), order.size());
    EXPECT_TRUE(order.size() > 5);
    for (size_t g = 0; g < std::min(order.size(), writer->Rows.size()); ++g) {
        const auto& got = writer->Rows[g];
        const auto& w = want[order[g]];
        EXPECT_TRUE(got[0].Type == EValueType::Int64 && got[0].Data.Int64 == order[g]);
        EXPECT_TRUE(got[1].Type == EValueType::Int64 && got[1].Data.Int64 == w.first);
        if (w.first) EXPECT_TRUE(got[2].Type == EValueType::Int64 && got[2].Data.Int64 == w.second);
        else EXPECT_TRUE(got[2].Type == EValueType::Null);
        if (Failures > 5) break;
    }

    // a column without values: every CONTAINS / LIKE over it is NULL, so nothing is selected
    TMultiGroupQuery none = q;
    size_t out = 1;
    none.Where = TFilterExpression().Like(3, "%");
    EXPECT_EQ(Code(none, owned, &out), 0);
    EXPECT_EQ(out, (size_t)0);
    none.Where = TFilterExpression().Contains(3, "").Not();
    out = 1;
    EXPECT_EQ(Code(none, owned, &out), 0);
    EXPECT_EQ(out, (size_t)0);

    // mistyped: over an int64 column; a pattern that ends in a lone escape
    TMultiGroupQuery bad = q;
    bad.Where = TFilterExpression().Contains(2, "1");
    EXPECT_EQ(Code(bad, owned), (int)YTGPU_ERR_INVALID_ARGUMENT);
    bad.Where = TFilterExpression().Like(2, "1%");
    EXPECT_EQ(Code(bad, owned), (int)YTGPU_ERR_INVALID_ARGUMENT);
    bad.Where = TFilterExpression().Like(1, "ab!", '!');
    EXPECT_EQ(Code(bad, owned), (int)YTGPU_ERR_INVALID_ARGUMENT);
}

}  // namespace

int main() {
    try {
        TestContainsAndNotLike();
    } catch (const std::exception& e) {
        std::fprintf(stderr, "unexpected exception: %s\n", e.what());
        return 100;
    }
    std::printf("like_ut: %d failure(s)\n", Failures);
    return Failures;
}
