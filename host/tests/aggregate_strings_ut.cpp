// aggregate_strings_ut.cpp — the QL evaluator adapter (TGpuEvaluator::Run(TMultiGroupQuery)) over string columns:
//   SELECT g, max(s), min(s), first(s), count(s), argmax(s, ts), argmin(ts, s) GROUP BY g
// with a string group item and string aggregate arguments over several reader batches with NULLs, against a std::map
// restatement in first-seen order (strings ordered as udf/min.c / max.c: memcmp over the common length, then length;
// argmin / argmax keep the first row on ties).  SUM of a string column and a string WHERE column are unsupported.
// Runs on the GPU box (tests/test_groupby_strings.py drives it); exit code = number of failed expectations.
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

using TOptString = std::optional<std::string>;

struct TRow {
    TOptString S, G;
    std::optional<int64_t> Ts;
};

TUnversionedOwningRow MakeRow(const TRow& r) {
    TUnversionedOwningRowBuilder b;
    b.AddValue(r.S ? MakeUnversionedStringValue(*r.S, 0) : MakeUnversionedNullValue(0));
    b.AddValue(r.G ? MakeUnversionedStringValue(*r.G, 1) : MakeUnversionedNullValue(1));
    b.AddValue(r.Ts ? MakeUnversionedInt64Value(*r.Ts, 2) : MakeUnversionedNullValue(2));
    return b.FinishRow();
}

bool IsString(const TUnversionedValue& v, const TOptString& want) {
    if (!want) return v.Type == EValueType::Null;
    return v.Type == EValueType::String && v.AsStringBuf() == *want;
}

struct TWant {
    TOptString Max, Min, First, ArgMax;
    int64_t Count = 0;
    std::optional<int64_t> ArgMaxBy, ArgMin;
    TOptString ArgMinBy;
};

void TestStringGroupByAndAggregates() {
    std::mt19937_64 rng(17);
    std::vector<std::string> words = {"", "a", std::string("a\0", 2), "ab", std::string(300, 'x') + "1", std::string(300, 'x') + "0",
                                      std::string("\xff", 1), "https://example.com/a", "https://example.com/b"};
    for (int i = 0; i < 40; ++i) {
        std::string w = "https://example.com/";
        const int len = (int)(rng() % 30);
        for (int j = 0; j < len; ++j) w += (char)(rng() % 256);
        words.push_back(w);
    }
    std::vector<std::string> groups = {"", "g1", std::string("g\0", 2), "g", std::string(500, 'k')};
    for (int i = 0; i < 60; ++i) groups.push_back("group-" + std::to_string(rng() % 1000));
    std::vector<TRow> rows;
    std::vector<TUnversionedOwningRow> owned;
    for (int i = 0; i < 25000; ++i) {  // three reader batches
        TRow r;
        if (rng() % 10) r.S = words[rng() % words.size()];
        if (rng() % 30) r.G = groups[rng() % groups.size()];
        if (rng() % 8) r.Ts = (int64_t)(rng() % 50) - 25;  // ties
        rows.push_back(r);
        owned.push_back(MakeRow(r));
    }
    // the restatement: first-seen order of the group items, NULL is a group of its own
    std::vector<TOptString> order;
    std::map<TOptString, TWant> want;
    for (const auto& r : rows) {
        if (!want.count(r.G)) order.push_back(r.G);
        TWant& w = want[r.G];
        if (r.S) {
            if (!w.Max || *r.S > *w.Max) w.Max = r.S;
            if (!w.Min || *r.S < *w.Min) w.Min = r.S;
            if (!w.First) w.First = r.S;
            ++w.Count;
        }
        if (r.S && r.Ts) {  // argmax(s, ts): strict comparison, the first row wins a tie
            if (!w.ArgMaxBy || *r.Ts > *w.ArgMaxBy) { w.ArgMaxBy = r.Ts; w.ArgMax = r.S; }
            if (!w.ArgMinBy || *r.S < *w.ArgMinBy) { w.ArgMinBy = r.S; w.ArgMin = r.Ts; }  // argmin(ts, s)
        }
    }
    TMultiGroupQuery q;
    q.GroupColumns = {1};
    q.AggregateItems = {{EAggregateFunction::Max, 0}, {EAggregateFunction::Min, 0}, {EAggregateFunction::First, 0},
                        {EAggregateFunction::Count, 0}, {EAggregateFunction::ArgMax, 0, 2}, {EAggregateFunction::ArgMin, 2, 0}};
    auto writer = std::make_shared<TCollectingWriter>();
    auto stats = CreateGpuEvaluator()->Run(q, CreateInMemoryReader(owned), writer);
    EXPECT_EQ(stats.RowsRead, 25000);
    EXPECT_EQ(writer->Rows.size(), order.size());
    for (size_t i = 0; i < std::min(order.size(), writer->Rows.size()); ++i) {
        const auto& got = writer->Rows[i];
        const TWant& w = want[order[i]];
        EXPECT_TRUE(IsString(got[0], order[i]));
        EXPECT_TRUE(IsString(got[1], w.Max));
        EXPECT_TRUE(IsString(got[2], w.Min));
        EXPECT_TRUE(IsString(got[3], w.First));
        EXPECT_TRUE(got[4].Type == EValueType::Int64 && got[4].Data.Int64 == w.Count);
        EXPECT_TRUE(IsString(got[5], w.ArgMax));
        if (w.ArgMin) EXPECT_TRUE(got[6].Type == EValueType::Int64 && got[6].Data.Int64 == *w.ArgMin);
        else EXPECT_TRUE(got[6].Type == EValueType::Null);
        if (Failures > 5) break;
    }
}

void TestUnsupported() {
    std::vector<TUnversionedOwningRow> owned = {MakeRow({std::string("a"), std::string("g"), 1}), MakeRow({std::string("b"), std::string("g"), 2})};
    auto code = [&](const TMultiGroupQuery& q) {
        try {
            CreateGpuEvaluator()->Run(q, CreateInMemoryReader(owned), std::make_shared<TCollectingWriter>());
        } catch (const TErrorException& e) {
            return e.GetCode();
        }
        return 0;
    };
    TMultiGroupQuery sum;
    sum.GroupColumns = {1};
    sum.AggregateItems = {{EAggregateFunction::Sum, 0}};
    EXPECT_EQ(code(sum), (int)YTGPU_ERR_UNSUPPORTED);
    TMultiGroupQuery where;
    where.GroupColumns = {2};
    where.AggregateItems = {{EAggregateFunction::Count, 2}};
    where.WhereColumn = 0;
    where.WhereOp = EBinaryOp::Greater;
    where.WhereConstant = MakeUnversionedInt64Value(0);
    EXPECT_EQ(code(where), (int)YTGPU_ERR_UNSUPPORTED);
}

}  // namespace

int main() {
    try {
        TestStringGroupByAndAggregates();
        TestUnsupported();
    } catch (const std::exception& e) {
        std::fprintf(stderr, "unexpected exception: %s\n", e.what());
        return 100;
    }
    std::printf("aggregate_strings_ut: %d failure(s)\n", Failures);
    return Failures;
}
