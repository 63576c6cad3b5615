// string_expression_ut.cpp — the QL evaluator adapter (TGpuEvaluator::Run(TMultiGroupQuery)) with string computed columns:
//   * GROUP BY if_null(lower(s), 'none') with count / sum / max(s) against a row-at-a-time restatement;
//   * GROUP BY farm_hash(a, s) % 4 against ytgpu_farm_fingerprint_rowset over the rows (a, s);
//   * a WHERE over concat(s, '/', t): Compare, StartsWith and Like leaves on the computed string column;
//   * an input string column that is NULL in every row (if_null(lower(s), 'none'), concat(s, t), lower(s));
//   * lower of a non-ASCII value throws YTGPU_ERR_UNSUPPORTED, and does not when the WHERE drops that row.
// Runs on the GPU box (tests/test_string_expressions.py drives it); exit code = number of failed expectations.
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

using TOptStr = std::optional<std::string>;
struct TRow { int64_t A; TOptStr S, T; };

TUnversionedValue StrOrNull(const TOptStr& s, int id) { return s ? MakeUnversionedStringValue(*s, id) : MakeUnversionedNullValue(id); }

std::vector<TUnversionedOwningRow> Owned(const std::vector<TRow>& rows) {
    std::vector<TUnversionedOwningRow> owned;
    for (const auto& r : rows) {
        TUnversionedOwningRowBuilder b;
        b.AddValue(MakeUnversionedInt64Value(r.A, 0));
        b.AddValue(StrOrNull(r.S, 1));
        b.AddValue(StrOrNull(r.T, 2));
        owned.push_back(b.FinishRow());
    }
    return owned;
}

std::vector<TRow> RandomRows(size_t count, uint64_t seed) {
    static const char* hosts[] = {"Example.COM", "example.com", "YT.Tech", "yt.tech", "", "a-B_c.d", "LongHost-Name-Of-The-Cluster-0123456789.Example.Org"};
    static const char* paths[] = {"x", "Index.HTML", "", "api/v1/Rows"};
    std::mt19937_64 rng(seed);
    std::vector<TRow> rows;
    for (size_t i = 0; i < count; ++i) {
        TRow r{(int64_t)(rng() % 1000) - 500, std::nullopt, std::nullopt};
        if (rng() % 7) r.S = hosts[rng() % 7];
        if (rng() % 5) r.T = paths[rng() % 4];
        rows.push_back(r);
    }
    return rows;
}

std::string Lower(std::string s) {
    for (auto& c : s)
        if (c >= 'A' && c <= 'Z') c = (char)(c + 32);
    return s;
}

// SELECT k, count(a), sum(a), max(s) GROUP BY if_null(lower(s), 'none') AS k
void TestGroupByIfNullLower() {
    const auto rows = RandomRows(20000, 7);
    TMultiGroupQuery q;
    q.Computed = {TExpression().Column(1).Lower().Constant(MakeUnversionedStringValue("none")).IfNull()};
    q.GroupColumns = {TMultiGroupQuery::ComputedColumn(0)};
    q.AggregateItems = {{EAggregateFunction::Count, 0}, {EAggregateFunction::Sum, 0}, {EAggregateFunction::Max, 1}};
    const auto got = Run(q, Owned(rows));
    struct TWant { int64_t Count = 0, Sum = 0; TOptStr Max; };
    std::vector<std::string> order;
    std::map<std::string, TWant> want;
    for (const auto& r : rows) {
        const std::string k = r.S ? Lower(*r.S) : "none";
        if (!want.count(k)) order.push_back(k);
        TWant& w = want[k];
        ++w.Count;
        w.Sum += r.A;
        if (r.S && (!w.Max || *r.S > *w.Max)) w.Max = r.S;
    }
    EXPECT_EQ(got.size(), order.size());
    for (size_t g = 0; g < std::min(got.size(), order.size()); ++g) {
        const TWant& w = want[order[g]];
        EXPECT_TRUE(got[g][0].Type == EValueType::String && got[g][0].AsStringBuf() == order[g]);
        EXPECT_TRUE(got[g][1].Type == EValueType::Int64 && got[g][1].Data.Int64 == w.Count);
        EXPECT_TRUE(got[g][2].Type == EValueType::Int64 && got[g][2].Data.Int64 == w.Sum);
        EXPECT_TRUE(w.Max ? got[g][3].Type == EValueType::String && got[g][3].AsStringBuf() == *w.Max : got[g][3].Type == EValueType::Null);
    }
}

// SELECT k, count(a) GROUP BY farm_hash(a, s) % 4 AS k, the fingerprints from ytgpu_farm_fingerprint_rowset
void TestGroupByFarmHash() {
    const auto rows = RandomRows(5000, 11);
    TMultiGroupQuery q;
    q.Computed = {TExpression().Column(0).Column(1).FarmHash(2).Constant(MakeUnversionedUint64Value(4)).Mod()};
    q.GroupColumns = {TMultiGroupQuery::ComputedColumn(0)};
    q.AggregateItems = {{EAggregateFunction::Count, 0}};
    const auto got = Run(q, Owned(rows));
    std::string heap;
    std::vector<ytgpu_value> values;
    for (const auto& r : rows) {
        values.push_back(ytgpu_value{0, YTGPU_TYPE_INT64, 0, 0, (uint64_t)r.A});
        if (r.S) {
            values.push_back(ytgpu_value{1, YTGPU_TYPE_STRING, 0, (uint32_t)r.S->size(), heap.size()});
            heap += *r.S;
        } else {
            values.push_back(ytgpu_value{1, YTGPU_TYPE_NULL, 0, 0, 0});
        }
    }
    ytgpu_context* ctx = nullptr;
    ytgpu_error err{};
    EXPECT_EQ(ytgpu_context_create(0, nullptr, &ctx, &err), (int)YTGPU_OK);
    const ytgpu_rowset_view view{values.data(), rows.size(), 2, 0, reinterpret_cast<const uint8_t*>(heap.data()), heap.size(), YTGPU_MEM_HOST};
    std::vector<uint64_t> fp(rows.size());
    EXPECT_EQ(ytgpu_farm_fingerprint_rowset(ctx, &view, 2, fp.data(), YTGPU_MEM_HOST, &err), (int)YTGPU_OK);
    ytgpu_context_destroy(ctx);
    std::vector<uint64_t> order;
    std::map<uint64_t, int64_t> want;
    for (uint64_t h : fp) {
        if (!want.count(h % 4)) order.push_back(h % 4);
        ++want[h % 4];
    }
    EXPECT_EQ(got.size(), order.size());
    for (size_t g = 0; g < std::min(got.size(), order.size()); ++g) {
        EXPECT_TRUE(got[g][0].Type == EValueType::Uint64 && got[g][0].Data.Uint64 == order[g]);
        EXPECT_TRUE(got[g][1].Type == EValueType::Int64 && got[g][1].Data.Int64 == want[order[g]]);
    }
}

// SELECT t, count(a) WHERE concat(s, '/', t) > 'e' AND NOT concat(...) LIKE '%.HTML' OR starts_with(concat(...), 'yt') GROUP BY t
void TestWhereOverConcat() {
    const auto rows = RandomRows(20000, 13);
    TMultiGroupQuery q;
    q.Computed = {TExpression().Column(1).Constant(MakeUnversionedStringValue("/")).Concat().Column(2).Concat()};
    const int c = TMultiGroupQuery::ComputedColumn(0);
    q.GroupColumns = {2};
    q.AggregateItems = {{EAggregateFunction::Count, 0}, {EAggregateFunction::Min, c}};
    q.Where = TFilterExpression().Compare(c, EBinaryOp::Greater, MakeUnversionedStringValue("e")).Like(c, "%.HTML").Not().And()
                  .StartsWith(c, "yt").Or();
    const auto got = Run(q, Owned(rows));
    struct TWant { int64_t Count = 0; std::string Min; };
    std::vector<TOptStr> order;
    std::map<TOptStr, TWant> want;
    auto endsWith = [](const std::string& s, const std::string& x) { return s.size() >= x.size() && s.compare(s.size() - x.size(), x.size(), x) == 0; };
    for (const auto& r : rows) {
        if (!r.S || !r.T) continue;  // concat is NULL: the WHERE is NULL or FALSE
        const std::string v = *r.S + "/" + *r.T;
        if (!((v > "e" && !endsWith(v, ".HTML")) || v.rfind("yt", 0) == 0)) continue;
        if (!want.count(r.T)) order.push_back(r.T);
        TWant& w = want[r.T];
        if (w.Count == 0 || v < w.Min) w.Min = v;
        ++w.Count;
    }
    EXPECT_EQ(got.size(), order.size());
    EXPECT_TRUE(order.size() >= 3);
    for (size_t g = 0; g < std::min(got.size(), order.size()); ++g) {
        const TWant& w = want[order[g]];
        EXPECT_TRUE(got[g][0].Type == EValueType::String && got[g][0].AsStringBuf() == *order[g]);
        EXPECT_TRUE(got[g][1].Type == EValueType::Int64 && got[g][1].Data.Int64 == w.Count);
        EXPECT_TRUE(got[g][2].Type == EValueType::String && got[g][2].AsStringBuf() == w.Min);
    }
}

// an input string column without a non-NULL value in the fragment is an all-NULL string column: QL's 'none' group for
// if_null(lower(s), 'none'), one NULL group for concat(s, t) and lower(s)
void TestAllNullStringInput() {
    std::vector<TRow> rows = RandomRows(3000, 19);
    for (auto& r : rows) r.S.reset();
    TMultiGroupQuery q;
    q.Computed = {TExpression().Column(1).Lower().Constant(MakeUnversionedStringValue("none")).IfNull()};
    q.GroupColumns = {TMultiGroupQuery::ComputedColumn(0)};
    q.AggregateItems = {{EAggregateFunction::Count, 0}};
    auto got = Run(q, Owned(rows));
    EXPECT_EQ(got.size(), (size_t)1);
    if (got.size() == 1)
        EXPECT_TRUE(got[0][0].Type == EValueType::String && got[0][0].AsStringBuf() == "none" && got[0][1].Data.Int64 == 3000);
    for (const auto& e : {TExpression().Column(1).Column(2).Concat(), TExpression().Column(1).Lower(),
                          TExpression().Column(2).Column(1).IfNull().Upper()}) {
        q.Computed = {e};
        got = Run(q, Owned(rows));
        if (e.Nodes.size() == 4) {  // upper(if_null(t, s)): the groups of upper(t), t's NULL rows NULL
            std::map<TOptStr, int64_t> want;
            for (const auto& r : rows) {
                TOptStr k = r.T;
                if (k) for (auto& ch : *k) if (ch >= 'a' && ch <= 'z') ch = (char)(ch - 32);
                ++want[k];
            }
            EXPECT_EQ(got.size(), want.size());
            for (const auto& row : got) {
                const TOptStr k = row[0].Type == EValueType::Null ? TOptStr() : TOptStr(std::string(row[0].AsStringBuf()));
                EXPECT_TRUE(want.count(k) && row[1].Data.Int64 == want[k]);
            }
            continue;
        }
        EXPECT_EQ(got.size(), (size_t)1);
        if (got.size() == 1) EXPECT_TRUE(got[0][0].Type == EValueType::Null && got[0][1].Data.Int64 == 3000);
    }
    // a WHERE over concat(s, '/') of the all-NULL column selects nothing
    TMultiGroupQuery w;
    w.Computed = {TExpression().Column(1).Constant(MakeUnversionedStringValue("/")).Concat()};
    w.GroupColumns = {2};
    w.AggregateItems = {{EAggregateFunction::Count, 0}};
    w.Where = TFilterExpression().IsNull(TMultiGroupQuery::ComputedColumn(0)).Not();
    EXPECT_EQ(Run(w, Owned(rows)).size(), (size_t)0);
}

// lower() of a value with a byte >= 0x80: YTGPU_ERR_UNSUPPORTED (the caller's CPU path), unless the WHERE drops the row
void TestNonAsciiRefusal() {
    std::vector<TRow> rows = RandomRows(1000, 17);
    rows[500].S = "Stra\xc3\x9f" "e";
    rows[500].A = 100000;
    TMultiGroupQuery q;
    q.Computed = {TExpression().Column(1).Lower()};
    q.GroupColumns = {TMultiGroupQuery::ComputedColumn(0)};
    q.AggregateItems = {{EAggregateFunction::Count, 0}};
    EXPECT_EQ(Code(q, Owned(rows)), (int)YTGPU_ERR_UNSUPPORTED);
    q.Where = TFilterExpression().Compare(0, EBinaryOp::Less, MakeUnversionedInt64Value(1000));
    EXPECT_EQ(Code(q, Owned(rows)), 0);
    // numeric ops over a string and sum of a string result stay UNSUPPORTED, a mistyped concat is INVALID_ARGUMENT
    TMultiGroupQuery n;
    n.Computed = {TExpression().Column(1).Neg()};
    n.GroupColumns = {0};
    n.AggregateItems = {{EAggregateFunction::Min, TMultiGroupQuery::ComputedColumn(0)}};
    EXPECT_EQ(Code(n, Owned(rows)), (int)YTGPU_ERR_UNSUPPORTED);
    n.Computed = {TExpression().Column(1).Upper()};
    n.AggregateItems = {{EAggregateFunction::Sum, TMultiGroupQuery::ComputedColumn(0)}};
    EXPECT_EQ(Code(n, Owned(rows)), (int)YTGPU_ERR_UNSUPPORTED);
    n.Computed = {TExpression().Column(1).Column(0).Concat()};
    n.AggregateItems = {{EAggregateFunction::Min, TMultiGroupQuery::ComputedColumn(0)}};
    EXPECT_EQ(Code(n, Owned(rows)), (int)YTGPU_ERR_INVALID_ARGUMENT);
}

}  // namespace

int main() {
    try {
        TestGroupByIfNullLower();
        TestGroupByFarmHash();
        TestWhereOverConcat();
        TestAllNullStringInput();
        TestNonAsciiRefusal();
    } catch (const std::exception& e) {
        std::fprintf(stderr, "unexpected exception: %s\n", e.what());
        return 100;
    }
    std::printf("string_expression_ut: %d failure(s)\n", Failures);
    return Failures;
}
