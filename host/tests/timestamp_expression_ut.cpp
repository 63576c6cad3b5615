// timestamp_expression_ut.cpp — the QL evaluator adapter (TGpuEvaluator::Run(TMultiGroupQuery)) with
// timestamp_floor_hour / day / week / month / year and format_timestamp, against a CPU restatement (integer arithmetic
// and the C library's strftime over gmtime_r in the C locale):
//   * GROUP BY timestamp_floor_day(ts) with COUNT and SUM, groups in first-seen order;
//   * GROUP BY format_timestamp(ts, '%Y-%m') with MIN(format_timestamp(ts, '%Y-%m-%d')) as a string aggregate;
//   * a WHERE leaf on a formatted value;
//   * floors in Select, Having and OrderBy; an all-NULL operand typed as Int64;
//   * FormatTimestamp refused in Select; an out-of-range row refused, and the same row dropped by WHERE not refused.
// Runs on the GPU box (tests/test_timestamp_expressions.py drives it); exit code = number of failed expectations.
#include <algorithm>
#include <climits>
#include <clocale>
#include <cstdio>
#include <ctime>
#include <map>
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
constexpr int C(int j) { return TMultiGroupQuery::ComputedColumn(j); }

// table: 0 ts (2015 .. 2025), 1 bytes, 2 ts with one value out of range (row Bad), 3 all NULL
constexpr int64_t T0 = 1420070400, T1 = 1735689600;
constexpr size_t N = 6000, Bad = 1234;
struct TRow { int64_t Ts, Bytes, Ts2; };
std::vector<TRow> MakeRows() {
    std::mt19937_64 rng(7);
    std::vector<TRow> rows;
    for (size_t i = 0; i < N; ++i) {
        const int64_t t = T0 + (int64_t)(rng() % (uint64_t)(T1 - T0));
        rows.push_back({t, (int64_t)(rng() % 1000), i == Bad ? -5 : t});
    }
    return rows;
}
const std::vector<TRow> Rows = MakeRows();

std::vector<TUnversionedOwningRow> TableRows() {
    std::vector<TUnversionedOwningRow> owned;
    for (const auto& r : Rows) {
        TUnversionedOwningRowBuilder b;
        b.AddValue(MakeUnversionedInt64Value(r.Ts, 0));
        b.AddValue(MakeUnversionedInt64Value(r.Bytes, 1));
        b.AddValue(MakeUnversionedInt64Value(r.Ts2, 2));
        b.AddValue(MakeUnversionedNullValue(3));
        owned.push_back(b.FinishRow());
    }
    return owned;
}

std::vector<TUnversionedOwningRow> Run(const TMultiGroupQuery& q) {
    auto writer = std::make_shared<TCollectingWriter>();
    CreateGpuEvaluator()->Run(q, CreateInMemoryReader(TableRows()), writer);
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

std::string Str(const TUnversionedValue& v) { return v.Type == EValueType::Null ? "<null>" : std::string(v.Data.String, v.Length); }

// the CPU restatement
int64_t FloorDay(int64_t t) { return t - t % 86400; }
int64_t FloorWeek(int64_t t) { const int64_t d = t / 86400; return (d - (d + 3) % 7) * 86400; }
int64_t FloorYear(int64_t t) {
    const time_t s = (time_t)t;
    std::tm tm{};
    gmtime_r(&s, &tm);
    tm.tm_mon = 0, tm.tm_mday = 1, tm.tm_hour = tm.tm_min = tm.tm_sec = 0;
    return (int64_t)timegm(&tm);
}
std::string Format(int64_t t, const char* fmt) {
    const time_t s = (time_t)t;
    std::tm tm{};
    gmtime_r(&s, &tm);
    char buf[128];
    return std::string(buf, std::strftime(buf, sizeof buf, fmt, &tm));
}

// SELECT timestamp_floor_day(ts) AS day, count(bytes), sum(bytes) FROM t GROUP BY day
void TestGroupByFloorDay() {
    TMultiGroupQuery q;
    q.Computed = {TExpression().Column(0).TimestampFloorDay()};
    q.GroupColumns = {C(0)};
    q.AggregateItems = {{EAggregateFunction::Count, 1}, {EAggregateFunction::Sum, 1}};
    std::vector<int64_t> order;
    std::map<int64_t, std::pair<int64_t, int64_t>> want;
    for (const auto& r : Rows) {
        const int64_t d = FloorDay(r.Ts);
        if (!want.count(d)) order.push_back(d);
        want[d].first += 1;
        want[d].second += r.Bytes;
    }
    const auto got = Run(q);
    EXPECT_EQ(got.size(), order.size());
    bool same = got.size() == order.size();
    for (size_t g = 0; same && g < got.size(); ++g)
        same = got[g][0].Data.Int64 == order[g] && got[g][1].Data.Int64 == want[order[g]].first && got[g][2].Data.Int64 == want[order[g]].second;
    EXPECT_TRUE(same);
}

// SELECT format_timestamp(ts, '%Y-%m') AS month, count(bytes), min(format_timestamp(ts, '%Y-%m-%d')) FROM t GROUP BY month
void TestGroupByFormattedMonth() {
    TMultiGroupQuery q;
    q.Computed = {TExpression().Column(0).FormatTimestamp("%Y-%m"), TExpression().Column(0).FormatTimestamp("%Y-%m-%d")};
    q.GroupColumns = {C(0)};
    q.AggregateItems = {{EAggregateFunction::Count, 1}, {EAggregateFunction::Min, C(1)}};
    std::vector<std::string> order;
    std::map<std::string, std::pair<int64_t, std::string>> want;
    for (const auto& r : Rows) {
        const std::string m = Format(r.Ts, "%Y-%m"), d = Format(r.Ts, "%Y-%m-%d");
        if (!want.count(m)) {
            order.push_back(m);
            want[m] = {0, d};
        }
        want[m].first += 1;
        if (d < want[m].second) want[m].second = d;
    }
    const auto got = Run(q);
    EXPECT_EQ(got.size(), order.size());
    bool same = got.size() == order.size();
    for (size_t g = 0; same && g < got.size(); ++g)
        same = Str(got[g][0]) == order[g] && got[g][1].Data.Int64 == want[order[g]].first && Str(got[g][2]) == want[order[g]].second;
    EXPECT_TRUE(same);
    EXPECT_EQ(order.size(), (size_t)120);
}

// SELECT bytes FROM t WHERE format_timestamp(ts, '%Y-%m') = '2024-03'
void TestWhereOnFormattedValue() {
    TMultiGroupQuery q;
    q.Computed = {TExpression().Column(0).FormatTimestamp("%Y-%m")};
    q.Where = TFilterExpression().Compare(C(0), EBinaryOp::Equal, MakeUnversionedStringValue("2024-03"));
    q.Project = {0};
    std::vector<int64_t> want, got;
    for (const auto& r : Rows)
        if (Format(r.Ts, "%Y-%m") == "2024-03") want.push_back(r.Ts);
    for (const auto& r : Run(q)) got.push_back(r[0].Data.Int64);
    EXPECT_EQ(got, want);
    EXPECT_TRUE(!want.empty());
}

// SELECT timestamp_floor_day(max(ts)), k FROM t GROUP BY timestamp_floor_month(ts) AS k
//   HAVING timestamp_floor_week(max(ts)) > X ORDER BY timestamp_floor_year(max(ts)) DESC, k LIMIT 30
void TestFloorsInSelectHavingOrderBy() {
    const int64_t x = 1600000000;
    TMultiGroupQuery q;
    q.Computed = {TExpression().Column(0).TimestampFloorMonth()};
    q.GroupColumns = {C(0)};
    q.AggregateItems = {{EAggregateFunction::Max, 0}};
    q.Having = TExpression().Column(1).TimestampFloorWeek().Constant(I(x)).Compare(EBinaryOp::Greater);
    q.OrderBy = {{TExpression().Column(1).TimestampFloorYear(), true}, {TExpression().Column(0), false}};
    q.Limit = 30;
    q.Select = std::vector<TExpression>{TExpression().Column(1).TimestampFloorDay(), TExpression().Column(0)};
    std::map<int64_t, int64_t> maxOf;  // month -> max ts
    for (const auto& r : Rows) {
        const time_t s = (time_t)r.Ts;
        std::tm tm{};
        gmtime_r(&s, &tm);
        tm.tm_mday = 1, tm.tm_hour = tm.tm_min = tm.tm_sec = 0;
        const int64_t month = (int64_t)timegm(&tm);
        maxOf[month] = std::max(maxOf.count(month) ? maxOf[month] : INT64_MIN, r.Ts);
    }
    std::vector<std::pair<int64_t, int64_t>> kept;  // (year of max, month)
    for (const auto& [month, mx] : maxOf)
        if (FloorWeek(mx) > x) kept.push_back({FloorYear(mx), month});
    std::stable_sort(kept.begin(), kept.end(), [](const auto& a, const auto& b) { return a.first != b.first ? a.first > b.first : a.second < b.second; });
    kept.resize(std::min<size_t>(kept.size(), 30));
    std::vector<int64_t> wantDay, wantMonth, gotDay, gotMonth;
    for (const auto& [year, month] : kept) {
        wantDay.push_back(FloorDay(maxOf[month]));
        wantMonth.push_back(month);
    }
    for (const auto& r : Run(q)) {
        gotDay.push_back(r[0].Data.Int64);
        gotMonth.push_back(r[1].Data.Int64);
    }
    EXPECT_EQ(gotDay, wantDay);
    EXPECT_EQ(gotMonth, wantMonth);
    EXPECT_EQ(wantDay.size(), (size_t)30);
}

// an all-NULL input column under a floor types as Int64: one NULL group
void TestAllNullOperand() {
    TMultiGroupQuery q;
    q.Computed = {TExpression().Column(3).TimestampFloorHour()};
    q.GroupColumns = {C(0)};
    q.AggregateItems = {{EAggregateFunction::Count, 1}};
    const auto got = Run(q);
    EXPECT_TRUE(got.size() == 1 && got[0][0].Type == EValueType::Null && got[0][1].Data.Int64 == (int64_t)N);
    TMultiGroupQuery f = q;
    f.Computed = {TExpression().Column(3).FormatTimestamp("%F")};
    const auto got2 = Run(f);
    EXPECT_TRUE(got2.size() == 1 && got2[0][0].Type == EValueType::Null);
}

void TestRefusals() {
    // format_timestamp over the output row
    TMultiGroupQuery s;
    s.GroupColumns = {1};
    s.AggregateItems = {{EAggregateFunction::Max, 0}};
    s.Select = std::vector<TExpression>{TExpression().Column(1).FormatTimestamp("%Y")};
    EXPECT_EQ(RunCode(s), (int)YTGPU_ERR_UNSUPPORTED);
    s.Select.reset();
    s.Having = TExpression().Column(1).FormatTimestamp("%Y").Constant(MakeUnversionedStringValue("2020")).Compare(EBinaryOp::Equal);
    EXPECT_EQ(RunCode(s), (int)YTGPU_ERR_UNSUPPORTED);
    // ts2 holds -5 in row Bad (bytes of that row: Rows[Bad].Bytes)
    TMultiGroupQuery q;
    q.Computed = {TExpression().Column(2).TimestampFloorDay()};
    q.GroupColumns = {C(0)};
    q.AggregateItems = {{EAggregateFunction::Count, 1}};
    EXPECT_EQ(RunCode(q), (int)YTGPU_ERR_UNSUPPORTED);
    q.Computed = {TExpression().Column(2).FormatTimestamp("%Y")};
    EXPECT_EQ(RunCode(q), (int)YTGPU_ERR_UNSUPPORTED);
    // the same row dropped by WHERE: no refusal
    q.Where = TFilterExpression().Compare(1, EBinaryOp::NotEqual, I(Rows[Bad].Bytes));
    EXPECT_EQ(RunCode(q), 0);
    q.Computed = {TExpression().Column(2).TimestampFloorDay()};
    EXPECT_EQ(RunCode(q), 0);
    // an unknown conversion is refused whatever the data
    TMultiGroupQuery c;
    c.Computed = {TExpression().Column(0).FormatTimestamp("%c")};
    c.GroupColumns = {C(0)};
    c.AggregateItems = {{EAggregateFunction::Count, 1}};
    EXPECT_EQ(RunCode(c), (int)YTGPU_ERR_UNSUPPORTED);
}

}  // namespace

int main() {
    std::setlocale(LC_TIME, "C");
    TestGroupByFloorDay();
    TestGroupByFormattedMonth();
    TestWhereOnFormattedValue();
    TestFloorsInSelectHavingOrderBy();
    TestAllNullOperand();
    TestRefusals();
    std::printf("timestamp_expression_ut: %d failure(s)\n", Failures);
    return Failures;
}
