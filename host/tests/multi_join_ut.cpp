// multi_join_ut.cpp — the QL evaluator adapter (TGpuEvaluator::Run(TMultiGroupQuery)) with several JOIN clauses and join
// keys that are expressions:
//   * hand-written queries over rows spelled out below: a snowflake chain, a star, LEFT then INNER on a column of the LEFT
//     table (the NULL rule), INNER then LEFT with fan-out in both clauses (the pair order through FIRST and LIMIT),
//     expression keys on either side, a self key expression over an earlier clause, a division by zero in a key, WHERE /
//     computed columns / HAVING / ORDER BY / LIMIT / Project over three clauses, every refusal, and one clause given
//     through Join alone;
//   * a randomized check against a CPU model of the chain (nested-loop joins in lexicographic order, NULL = NULL, doubles
//     by bit pattern, then a projection and a first-seen GROUP BY), from 0 to 10^6 primary rows;
//   * an equivalence check: two clauses give the rows of clause 0 alone, written to a table and joined by clause 1.
// Runs on the GPU box (tests/test_multi_join.py drives it); exit code = number of failed expectations.
#include <algorithm>
#include <cctype>
#include <cstdio>
#include <cstring>
#include <functional>
#include <random>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/ytgpu.h"
#include "../yt_query_client.h"

using namespace NYT::NTableClient;
using namespace NYT::NQueryClient;

static int Failures = 0;
#define EXPECT_EQ(a, b) do { auto _a = (a); auto _b = (b); if (!(_a == _b)) { ++Failures; std::fprintf(stderr, "%s:%d: EXPECT_EQ(%s, %s) failed\n", __FILE__, __LINE__, #a, #b); } } while (0)

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

// A typed value of a test table: doubles by bit pattern, so that -0.0 and NaN payloads compare exactly.
struct V {
    EValueType Type = EValueType::Null;
    uint64_t Bits = 0;
    std::string Str = {};
    bool operator==(const V& o) const {
        return Type == o.Type && (Type == EValueType::String ? Str == o.Str : Type == EValueType::Null || Bits == o.Bits);
    }
};
V Nul() { return {}; }
V I(int64_t x) { return {EValueType::Int64, (uint64_t)x}; }
V U(uint64_t x) { return {EValueType::Uint64, x}; }
V D(double x) { uint64_t b; std::memcpy(&b, &x, 8); return {EValueType::Double, b}; }
V DBits(uint64_t b) { return {EValueType::Double, b}; }
V B(bool x) { return {EValueType::Boolean, x ? 1u : 0u}; }
V S(std::string s) { return {EValueType::String, 0, std::move(s)}; }
using TRow = std::vector<V>;
using TTable = std::vector<TRow>;

TUnversionedValue IV(int64_t x) { return MakeUnversionedInt64Value(x); }
TUnversionedValue SV(const char* s) { return MakeUnversionedStringValue(s); }
constexpr int F(int clause, int j) { return TMultiGroupQuery::ForeignColumn(clause, j); }
constexpr int E(int e) { return TMultiGroupQuery::ComputedColumn(e); }

std::string Show(const V& v) {
    switch (v.Type) {
        case EValueType::Null: return "NULL";
        case EValueType::String: return "'" + v.Str + "'";
        case EValueType::Uint64: return std::to_string(v.Bits) + "u";
        case EValueType::Boolean: return v.Bits ? "true" : "false";
        case EValueType::Double: { char b[40]; std::snprintf(b, sizeof b, "d%016llx", (unsigned long long)v.Bits); return b; }
        default: return std::to_string((int64_t)v.Bits);
    }
}

std::string Show(const TRow& row) {
    std::string s = "(";
    for (size_t i = 0; i < row.size(); ++i) s += (i ? ", " : "") + Show(row[i]);
    return s + ")";
}

ISchemalessMultiChunkReaderPtr Reader(const TTable& table) {
    std::vector<TUnversionedOwningRow> owned;
    owned.reserve(table.size());
    for (const auto& row : table) {
        TUnversionedOwningRowBuilder b;
        for (int i = 0; i < (int)row.size(); ++i) {
            const V& v = row[i];
            switch (v.Type) {
                case EValueType::Null: b.AddValue(MakeUnversionedNullValue(i)); break;
                case EValueType::Int64: b.AddValue(MakeUnversionedInt64Value((int64_t)v.Bits, i)); break;
                case EValueType::Uint64: b.AddValue(MakeUnversionedUint64Value(v.Bits, i)); break;
                case EValueType::Double: { double d; std::memcpy(&d, &v.Bits, 8); b.AddValue(MakeUnversionedDoubleValue(d, i)); break; }
                case EValueType::Boolean: b.AddValue(MakeUnversionedBooleanValue(v.Bits != 0, i)); break;
                default: b.AddValue(MakeUnversionedStringValue(v.Str, i)); break;
            }
        }
        owned.push_back(b.FinishRow());
    }
    return CreateInMemoryReader(std::move(owned));
}

// The table behind each foreign reader Clause() makes: Run() reads a query's foreign tables afresh, so a query runs twice
std::unordered_map<const void*, TTable> ForeignTables;

TTable Run(const TMultiGroupQuery& q, const TTable& primary, TQueryStatistics* stats = nullptr) {
    TMultiGroupQuery fresh = q;
    auto refresh = [](TMultiGroupQuery::TJoinClause& clause) {
        if (auto it = ForeignTables.find(clause.Foreign.get()); it != ForeignTables.end()) clause.Foreign = Reader(it->second);
    };
    if (fresh.Join) refresh(*fresh.Join);
    for (auto& clause : fresh.NextJoins) refresh(clause);
    auto writer = std::make_shared<TCollectingWriter>();
    const auto s = CreateGpuEvaluator()->Run(fresh, Reader(primary), writer);
    if (stats) *stats = s;
    TTable out;
    out.reserve(writer->Rows.size());
    for (const auto& r : writer->Rows) {
        TRow row;
        for (const auto* x = r.Begin(); x != r.End(); ++x) {
            switch (x->Type) {
                case EValueType::Null: row.push_back(Nul()); break;
                case EValueType::String: row.push_back(S(std::string(x->Data.String, x->Length))); break;
                case EValueType::Boolean: row.push_back(B(x->Data.Boolean)); break;
                default: row.push_back({x->Type, x->Data.Uint64}); break;
            }
        }
        out.push_back(std::move(row));
    }
    return out;
}

void Expect(const TTable& got, const TTable& want, int line, const std::string& what = "") {
    if (got.size() != want.size()) {
        ++Failures;
        std::fprintf(stderr, "line %d %s: %zu rows, want %zu\n", line, what.c_str(), got.size(), want.size());
        for (size_t r = 0; r < std::min<size_t>(got.size(), 12); ++r) std::fprintf(stderr, "  got %s\n", Show(got[r]).c_str());
        return;
    }
    for (size_t r = 0; r < got.size(); ++r)
        if (!(got[r] == want[r])) {
            ++Failures;
            std::fprintf(stderr, "line %d %s: row %zu is %s, want %s\n", line, what.c_str(), r, Show(got[r]).c_str(), Show(want[r]).c_str());
            return;
        }
}

int CodeOf(const std::function<void()>& f) {
    try {
        f();
    } catch (const TErrorException& e) {
        return e.GetCode();
    }
    return 0;
}

TMultiGroupQuery::TJoinClause Clause(const TTable& foreign, std::vector<int> self, std::vector<int> keys, bool left = false) {
    auto reader = Reader(foreign);
    ForeignTables[reader.get()] = foreign;
    return TMultiGroupQuery::TJoinClause{reader, std::move(self), std::move(keys), left};
}

// facts (primary): 0 fact id, 1 user id (nullable), 2 amount, 3 product id
const TTable Facts = {
    {I(0), I(10), I(5), I(100)}, {I(1), I(11), I(7), I(101)}, {I(2), I(10), I(1), I(102)},
    {I(3), I(12), I(20), I(100)}, {I(4), Nul(), I(3), I(101)}, {I(5), I(13), I(9), I(103)},
};
// users: 0 id, 1 region id (nullable), 2 name; user 14 has no fact, user 13 no region
const TTable Users = {{I(10), I(1), S("ann")}, {I(11), I(2), S("bob")}, {I(12), I(1), S("cat")}, {I(13), Nul(), S("dan")}, {I(14), I(3), S("eve")}};
// regions: 0 id (one NULL), 1 name
const TTable Regions = {{I(1), S("eu")}, {I(2), S("us")}, {I(3), S("asia")}, {Nul(), S("nowhere")}};
const TTable RegionsWithoutNull = {{I(1), S("eu")}, {I(2), S("us")}, {I(3), S("asia")}};
// products: 0 id, 1 category; product 103 has none
const TTable Products = {{I(100), S("toys")}, {I(101), S("books")}, {I(102), S("toys")}};

// SELECT r.name, sum(f.amount), count(f.amount) FROM facts f JOIN users u ON f.user_id = u.id JOIN regions r
// ON u.region_id = r.id GROUP BY r.name.  Fact 4 has no user; fact 5's user has a NULL region, which matches the NULL id.
void TestSnowflake() {
    TMultiGroupQuery q;
    q.Join = Clause(Users, {1}, {0});
    q.NextJoins = {Clause(Regions, {F(0, 1)}, {0})};
    q.GroupColumns = {F(1, 1)};
    q.AggregateItems = {{EAggregateFunction::Sum, 2}, {EAggregateFunction::Count, 2}};
    TQueryStatistics stats;
    Expect(Run(q, Facts, &stats), {{S("eu"), I(26), I(3)}, {S("us"), I(7), I(1)}, {S("nowhere"), I(9), I(1)}}, __LINE__);
    EXPECT_EQ(stats.RowsRead, (int64_t)Facts.size());
    EXPECT_EQ(stats.RowsWritten, (int64_t)3);
}

// ... FROM facts f JOIN users u ON f.user_id = u.id JOIN products p ON f.product_id = p.id GROUP BY p.category, u.name
void TestStar() {
    TMultiGroupQuery q;
    q.Join = Clause(Users, {1}, {0});
    q.NextJoins = {Clause(Products, {3}, {0})};
    q.GroupColumns = {F(1, 1), F(0, 2)};
    q.AggregateItems = {{EAggregateFunction::Sum, 2}};
    Expect(Run(q, Facts), {{S("toys"), S("ann"), I(6)}, {S("books"), S("bob"), I(7)}, {S("toys"), S("cat"), I(20)}}, __LINE__);
}

// facts LEFT JOIN users, then JOIN regions ON u.region_id = r.id: fact 4 missed its user, so its region id is NULL and
// matches the NULL id, as does fact 5's user's NULL region.  Without a NULL id both rows go.
void TestLeftThenInnerNullRule() {
    TMultiGroupQuery q;
    q.Join = Clause(Users, {1}, {0}, true);
    q.NextJoins = {Clause(Regions, {F(0, 1)}, {0})};
    q.Project = {0, F(0, 2), F(1, 1)};
    Expect(Run(q, Facts),
           {{I(0), S("ann"), S("eu")}, {I(1), S("bob"), S("us")}, {I(2), S("ann"), S("eu")}, {I(3), S("cat"), S("eu")},
            {I(4), Nul(), S("nowhere")}, {I(5), S("dan"), S("nowhere")}},
           __LINE__);
    q.NextJoins = {Clause(RegionsWithoutNull, {F(0, 1)}, {0})};
    Expect(Run(q, Facts), {{I(0), S("ann"), S("eu")}, {I(1), S("bob"), S("us")}, {I(2), S("ann"), S("eu")}, {I(3), S("cat"), S("eu")}},
           __LINE__);
}

// INNER then LEFT, fan-out 2 in both clauses: the joined rows are ordered by (primary row, clause 0 row, clause 1 row)
void TestPairOrder() {
    const TTable p = {{I(0), I(1)}, {I(1), I(2)}, {I(2), I(1)}};                          // 0 id, 1 k
    const TTable a = {{I(1), I(10), I(7)}, {I(2), I(20), I(8)}, {I(1), I(11), I(9)}};     // 0 k, 1 tag, 2 g
    const TTable b = {{I(7), I(100)}, {I(9), I(300)}, {I(7), I(101)}, {I(9), I(301)}};    // 0 g, 1 val; g 8 has none
    TMultiGroupQuery q;
    q.Join = Clause(a, {1}, {0});
    q.NextJoins = {Clause(b, {F(0, 2)}, {0}, true)};
    q.Project = {0, F(0, 1), F(1, 1)};
    const TTable all = {{I(0), I(10), I(100)}, {I(0), I(10), I(101)}, {I(0), I(11), I(300)}, {I(0), I(11), I(301)}, {I(1), I(20), Nul()},
                        {I(2), I(10), I(100)}, {I(2), I(10), I(101)}, {I(2), I(11), I(300)}, {I(2), I(11), I(301)}};
    Expect(Run(q, p), all, __LINE__);
    q.Limit = 5;  // LIMIT without ORDER BY: the first joined rows
    Expect(Run(q, p), TTable(all.begin(), all.begin() + 5), __LINE__);
    // GROUP BY the primary row with first(): the first joined row of each
    TMultiGroupQuery g;
    g.Join = Clause(a, {1}, {0});
    g.NextJoins = {Clause(b, {F(0, 2)}, {0}, true)};
    g.GroupColumns = {0};
    g.AggregateItems = {{EAggregateFunction::First, F(1, 1)}, {EAggregateFunction::First, F(0, 1)}, {EAggregateFunction::Count, F(1, 1)}};
    Expect(Run(g, p), {{I(0), I(100), I(10), I(4)}, {I(1), Nul(), I(20), I(0)}, {I(2), I(100), I(10), I(4)}}, __LINE__);
    // GROUP BY the clause 1 value: groups in the order their first joined row comes
    g.GroupColumns = {F(1, 1)};
    g.AggregateItems = {{EAggregateFunction::First, 0}, {EAggregateFunction::Count, 0}};
    Expect(Run(g, p), {{I(100), I(0), I(2)}, {I(101), I(0), I(2)}, {I(300), I(0), I(2)}, {I(301), I(0), I(2)}, {Nul(), I(1), I(1)}}, __LINE__);
}

void TestExpressionKeys() {
    const TTable dims = {{I(5), S("five")}, {I(7), S("seven")}, {I(-3), S("neg")}};  // 0 id, 1 name
    {   // ON f.k % 1000 = d.id
        TMultiGroupQuery q;
        q.Join = Clause(dims, {E(0)}, {0});
        q.Join->SelfExpressions = {TExpression().Column(0).Constant(IV(1000)).Mod()};
        q.Project = {0, F(0, 1)};
        Expect(Run(q, {{I(1005)}, {I(2007)}, {I(-3)}, {I(5)}, {Nul()}}),
               {{I(1005), S("five")}, {I(2007), S("seven")}, {I(-3), S("neg")}, {I(5), S("five")}}, __LINE__);
    }
    {   // ON cast(f.u as int64) = d.id; without the cast the key types differ
        const TTable facts = {{U(5)}, {U(7)}, {U(8)}};
        TMultiGroupQuery q;
        q.Join = Clause(dims, {E(0)}, {0});
        q.Join->SelfExpressions = {TExpression().Column(0).Cast(EValueType::Int64)};
        q.Project = {0, F(0, 1)};
        Expect(Run(q, facts), {{U(5), S("five")}, {U(7), S("seven")}}, __LINE__);
        q.Join = Clause(dims, {0}, {0});
        EXPECT_EQ(CodeOf([&] { Run(q, facts); }), (int)YTGPU_ERR_INVALID_ARGUMENT);
    }
    {   // ON lower(f.host) = d.host: a string result against a string column
        TMultiGroupQuery q;
        q.Join = Clause({{S("a.com"), I(1)}, {S("b.com"), I(2)}}, {E(0)}, {0});
        q.Join->SelfExpressions = {TExpression().Column(0).Lower()};
        q.Project = {0, F(0, 1)};
        Expect(Run(q, {{S("A.com")}, {S("B.COM")}, {S("c.com")}, {Nul()}}), {{S("A.com"), I(1)}, {S("B.COM"), I(2)}}, __LINE__);
    }
    {   // ON concat(f.a, f.b) = concat(d.a, d.b)
        TMultiGroupQuery q;
        q.Join = Clause({{S("a"), S("bc"), I(1)}, {S("xy"), S(""), I(2)}}, {E(0)}, {E(0)});
        q.Join->SelfExpressions = {TExpression().Column(0).Column(1).Concat()};
        q.Join->ForeignExpressions = {TExpression().Column(0).Column(1).Concat()};
        q.Project = {0, 1, F(0, 2)};
        Expect(Run(q, {{S("ab"), S("c")}, {S("a"), S("bc")}, {S("x"), S("y")}}),
               {{S("ab"), S("c"), I(1)}, {S("a"), S("bc"), I(1)}, {S("x"), S("y"), I(2)}}, __LINE__);
    }
    {   // ON (f.a, f.b % 10) = (d.a, d.b % 10): a column and an expression in one tuple
        TMultiGroupQuery q;
        q.Join = Clause({{I(1), I(5), S("x")}, {I(2), I(5), S("y")}, {I(1), I(15), S("z")}}, {0, E(0)}, {0, E(0)});
        q.Join->SelfExpressions = {TExpression().Column(1).Constant(IV(10)).Mod()};
        q.Join->ForeignExpressions = {TExpression().Column(1).Constant(IV(10)).Mod()};
        q.Project = {1, F(0, 2)};
        Expect(Run(q, {{I(1), I(15)}, {I(1), I(25)}, {I(2), I(15)}}),
               {{I(15), S("x")}, {I(15), S("z")}, {I(25), S("x")}, {I(25), S("z")}, {I(15), S("y")}}, __LINE__);
    }
    {   // ON timestamp_floor_day(f.ts) = d.day
        TMultiGroupQuery q;
        q.Join = Clause({{I(3 * 86400), S("d3")}, {I(4 * 86400), S("d4")}}, {E(0)}, {0});
        q.Join->SelfExpressions = {TExpression().Column(0).TimestampFloorDay()};
        q.Project = {0, F(0, 1)};
        Expect(Run(q, {{I(3 * 86400 + 5)}, {I(3 * 86400 + 7000)}, {I(4 * 86400 + 1)}, {I(5 * 86400)}}),
               {{I(3 * 86400 + 5), S("d3")}, {I(3 * 86400 + 7000), S("d3")}, {I(4 * 86400 + 1), S("d4")}}, __LINE__);
    }
    {   // the key types follow the results: a string result against an integer column is refused
        TMultiGroupQuery q;
        q.Join = Clause(dims, {E(0)}, {0});
        q.Join->SelfExpressions = {TExpression().Column(0).Lower()};
        q.Project = {0};
        EXPECT_EQ(CodeOf([&] { Run(q, {{S("x")}}); }), (int)YTGPU_ERR_INVALID_ARGUMENT);
    }
}

// ... JOIN users u ON f.user_id = u.id JOIN r2 ON u.region_id + 1 = r2.id: a self key expression over clause 0's columns
void TestSelfExpressionOverEarlierClause() {
    TMultiGroupQuery q;
    q.Join = Clause(Users, {1}, {0});
    q.NextJoins = {Clause({{I(2), S("two")}, {I(3), S("three")}}, {E(0)}, {0})};
    q.NextJoins[0].SelfExpressions = {TExpression().Column(F(0, 1)).Constant(IV(1)).Add()};
    q.Project = {0, F(1, 1)};
    Expect(Run(q, Facts), {{I(0), S("two")}, {I(1), S("three")}, {I(2), S("two")}, {I(3), S("two")}}, __LINE__);
}

// A key expression is evaluated over every row before the join and the WHERE: 100 / 0 throws though WHERE drops the row
void TestDivisionByZeroInKey() {
    TMultiGroupQuery q;
    q.Join = Clause({{I(20)}}, {E(0)}, {0});
    q.Join->SelfExpressions = {TExpression().Constant(IV(100)).Column(1).Div()};
    q.Where = TFilterExpression().Compare(1, EBinaryOp::Greater, IV(0));
    q.Project = {0};
    EXPECT_EQ(CodeOf([&] { Run(q, {{I(1), I(0)}, {I(2), I(5)}}); }), (int)YTGPU_ERR_INVALID_ARGUMENT);
    Expect(Run(q, {{I(1), I(4)}, {I(2), I(5)}}), {{I(2)}}, __LINE__);  // 100 / 5 = 20
}

// users INNER, regions LEFT, products INNER: rows f0 (ann, eu, toys, 5), f1 (bob, us, books, 7), f2 (ann, eu, toys, 1),
// f3 (cat, eu, toys, 20); f4 has no user, f5 (dan, no region) has no product
void TestClausesDownstream() {
    TMultiGroupQuery q;
    q.Join = Clause(Users, {1}, {0});
    q.NextJoins = {Clause(RegionsWithoutNull, {F(0, 1)}, {0}, true), Clause(Products, {3}, {0})};
    // WHERE p.category = 'toys' GROUP BY concat(r.name, u.name) HAVING sum(f.amount) > 5 ORDER BY sum(f.amount) DESC LIMIT 10
    q.Where = TFilterExpression().Compare(F(2, 1), EBinaryOp::Equal, SV("toys"));
    q.Computed = {TExpression().Column(F(1, 1)).Column(F(0, 2)).Concat()};
    q.GroupColumns = {E(0)};
    q.AggregateItems = {{EAggregateFunction::Sum, 2}};
    q.Having = TExpression().Column(1).Constant(IV(5)).Compare(EBinaryOp::Greater);
    q.OrderBy = {{TExpression().Column(1), true}};
    q.Limit = 10;
    Expect(Run(q, Facts), {{S("eucat"), I(20)}, {S("euann"), I(6)}}, __LINE__);
    q.Having.reset();
    q.Where = TFilterExpression().Compare(F(2, 1), EBinaryOp::Equal, SV("books"));
    Expect(Run(q, Facts), {{S("usbob"), I(7)}}, __LINE__);
    // SELECT f.id, u.name, r.name, p.category ... WHERE u.name != 'bob' ORDER BY f.id DESC LIMIT 2
    TMultiGroupQuery p;
    p.Join = Clause(Users, {1}, {0});
    p.NextJoins = {Clause(RegionsWithoutNull, {F(0, 1)}, {0}, true), Clause(Products, {3}, {0})};
    p.Where = TFilterExpression().Compare(F(0, 2), EBinaryOp::NotEqual, SV("bob"));
    p.Project = {0, F(0, 2), F(1, 1), F(2, 1)};
    p.OrderBy = {{TExpression().Column(0), true}};
    p.Limit = 2;
    Expect(Run(p, Facts), {{I(3), S("cat"), S("eu"), S("toys")}, {I(2), S("ann"), S("eu"), S("toys")}}, __LINE__);
    // Select over the projection: amount * 2 with the region's name
    p.OrderBy.clear();
    p.Limit.reset();
    p.Where.reset();
    p.Project = {2, F(1, 1)};
    p.Select = std::vector<TExpression>{TExpression().Column(0).Constant(IV(2)).Mul(), TExpression().Column(1)};
    Expect(Run(p, Facts), {{I(10), S("eu")}, {I(14), S("us")}, {I(2), S("eu")}, {I(40), S("eu")}}, __LINE__);
}

void TestRefusals() {
    auto base = [] {
        TMultiGroupQuery q;
        q.Join = Clause(Users, {1}, {0});
        q.NextJoins = {Clause(Regions, {F(0, 1)}, {0})};
        q.Project = {0};
        return q;
    };
    auto refused = [&](const TMultiGroupQuery& q, int line) {
        const int code = CodeOf([&] { Run(q, Facts); });
        if (code != YTGPU_ERR_INVALID_ARGUMENT) {
            ++Failures;
            std::fprintf(stderr, "line %d: code %d, want INVALID_ARGUMENT\n", line, code);
        }
    };
    {   // a self column of the current clause's foreign rows
        auto q = base();
        q.NextJoins[0].SelfColumns = {F(1, 0)};
        refused(q, __LINE__);
    }
    {   // a self column of a later clause's foreign rows
        auto q = base();
        q.Join->SelfColumns = {F(1, 0)};
        refused(q, __LINE__);
    }
    {   // a self expression over the current clause's foreign rows
        auto q = base();
        q.NextJoins[0].SelfColumns = {E(0)};
        q.NextJoins[0].SelfExpressions = {TExpression().Column(F(1, 0))};
        refused(q, __LINE__);
    }
    {   // a self expression over a query.Computed position
        auto q = base();
        q.Computed = {TExpression().Column(2)};
        q.Join->SelfColumns = {E(0)};
        q.Join->SelfExpressions = {TExpression().Column(E(0))};
        refused(q, __LINE__);
    }
    {   // a foreign expression over a foreign position of the clause (it reads plain positions)
        auto q = base();
        q.Join->ForeignColumns = {E(0)};
        q.Join->ForeignExpressions = {TExpression().Column(F(0, 0))};
        refused(q, __LINE__);
    }
    {   // ComputedColumn(e) beyond the side's list
        auto q = base();
        q.Join->SelfColumns = {E(1)};
        q.Join->SelfExpressions = {TExpression().Column(1)};
        refused(q, __LINE__);
        auto r = base();
        r.NextJoins[0].ForeignColumns = {E(0)};
        refused(r, __LINE__);
    }
    {   // a foreign position of a clause that does not exist
        auto q = base();
        q.Project = {F(2, 0)};
        refused(q, __LINE__);
        q.Project = {0};
        q.NextJoins[0].SelfColumns = {F(5, 1)};
        refused(q, __LINE__);
    }
    {   // NextJoins without Join
        auto q = base();
        q.Join.reset();
        refused(q, __LINE__);
    }
    {   // 8 clauses run, 9 are refused: the star facts -> users, eight times
        TMultiGroupQuery q;
        q.Join = Clause(Users, {1}, {0});
        for (int c = 1; c < 8; ++c) q.NextJoins.push_back(Clause(Users, {1}, {0}));
        q.Project = {0, F(7, 2)};
        Expect(Run(q, Facts), {{I(0), S("ann")}, {I(1), S("bob")}, {I(2), S("ann")}, {I(3), S("cat")}, {I(5), S("dan")}}, __LINE__);
        q.NextJoins.push_back(Clause(Users, {1}, {0}));
        refused(q, __LINE__);
    }
}

// One clause through Join alone: the rows of join_ut's star and LEFT queries over its tables
void TestSingleClause() {
    const TTable facts = {{I(1), I(10), S("a")}, {I(2), I(20), S("b")}, {I(1), I(30), S("a")}, {I(3), I(40), S("zz")}, {I(2), I(50), S("b")},
                          {Nul(), I(60), Nul()}};
    const TTable dims = {{I(1), S("eu"), I(7), S("a")}, {I(2), S("us"), I(8), S("b")}, {I(4), S("eu"), I(9), S("c")}, {I(2), S("asia"), I(5), S("b")}};
    TMultiGroupQuery q;
    q.Join = Clause(dims, {0}, {0});
    q.GroupColumns = {TMultiGroupQuery::ForeignColumn(1)};
    q.AggregateItems = {{EAggregateFunction::Sum, 1}, {EAggregateFunction::Count, 1}};
    Expect(Run(q, facts), {{S("eu"), I(40), I(2)}, {S("us"), I(70), I(2)}, {S("asia"), I(70), I(2)}}, __LINE__);
    q.Join = Clause(dims, {0}, {0}, true);
    q.GroupColumns = {2};
    q.AggregateItems = {{EAggregateFunction::Count, F(0, 2)}, {EAggregateFunction::First, F(0, 1)}, {EAggregateFunction::Sum, 1}};
    Expect(Run(q, facts), {{S("a"), I(2), S("eu"), I(40)}, {S("b"), I(4), S("us"), I(140)}, {S("zz"), I(0), Nul(), I(40)}, {Nul(), I(0), Nul(), I(60)}},
           __LINE__);
}

// ---- the randomized model check ----
// Every table has the columns 0 int64, 1 uint64, 2 double (+-0.0, NaNs), 3 boolean, 4 string (mixed case), all with NULLs,
// and 5 the row's index.  A clause joins on one of these key kinds; its self side reads the primary table or an earlier
// clause's foreign table.
enum EKind { KInt, KCastUint, KMod, KModBoth, KDouble, KBool, KString, KLower, KPair, KindCount };
struct TSpec {
    EKind Kind;
    int SelfSource;  // 0: the primary rows, s > 0: clause s - 1's foreign rows
    bool Left;
};

// NULLs: one value in 12 of the primary table; about one per column of a foreign table, since NULL keys match each other
// and many of them on both sides would multiply the joined rows
TTable MakeTable(std::mt19937_64& rng, size_t rows, int64_t range, bool foreign) {
    auto pick = [&](uint64_t n) { return rng() % n; };
    const uint64_t nullEvery = foreign ? std::max<uint64_t>(12, rows) : 12;
    auto null = [&] { return pick(nullEvery) == 0; };
    const V doubles[] = {D(0.0), D(-0.0), DBits(0x7ff8000000000000ull), DBits(0x7ff8000000000123ull), D(1.5), D(-2.25)};
    TTable t(rows);
    for (size_t i = 0; i < rows; ++i) {
        const int64_t k = (int64_t)pick((uint64_t)range + 2) - 2;
        t[i] = {null() ? Nul() : I(k), null() ? Nul() : U(pick((uint64_t)range)), null() ? Nul() : doubles[pick(6)], null() ? Nul() : B(pick(2)),
                null() ? Nul() : S((pick(3) == 0 ? "K" : "k") + std::to_string(pick((uint64_t)range))), I((int64_t)i)};
    }
    return t;
}

// The clause of `spec` over `foreign`; position(s, j) names column j of source s in the self side's rows
TMultiGroupQuery::TJoinClause MakeClause(const TSpec& spec, const TTable& foreign, const std::function<int(int, int)>& position) {
    const int s = spec.SelfSource;
    auto clause = Clause(foreign, {}, {}, spec.Left);
    switch (spec.Kind) {
        case KInt: clause.SelfColumns = {position(s, 0)}; clause.ForeignColumns = {0}; break;
        case KCastUint:
            clause.SelfExpressions = {TExpression().Column(position(s, 1)).Cast(EValueType::Int64)};
            clause.SelfColumns = {E(0)};
            clause.ForeignColumns = {0};
            break;
        case KMod:
        case KModBoth:
            clause.SelfExpressions = {TExpression().Column(position(s, 0)).Constant(IV(7)).Mod()};
            clause.SelfColumns = {E(0)};
            clause.ForeignColumns = {0};
            if (spec.Kind == KModBoth) {
                clause.ForeignExpressions = {TExpression().Column(0).Constant(IV(7)).Mod()};
                clause.ForeignColumns = {E(0)};
            }
            break;
        case KDouble: clause.SelfColumns = {position(s, 2)}; clause.ForeignColumns = {2}; break;
        case KBool: clause.SelfColumns = {position(s, 3)}; clause.ForeignColumns = {3}; break;
        case KString: clause.SelfColumns = {position(s, 4)}; clause.ForeignColumns = {4}; break;
        case KLower:
            clause.SelfExpressions = {TExpression().Column(position(s, 4)).Lower()};
            clause.SelfColumns = {E(0)};
            clause.ForeignColumns = {4};
            break;
        default: clause.SelfColumns = {position(s, 0), position(s, 4)}; clause.ForeignColumns = {0, 4}; break;
    }
    return clause;
}

// The key tuple of a row as bytes: equal exactly when the tuples are equal under the join's rule (NULL = NULL, doubles by
// bit pattern)
void AppendKey(std::string* key, const V& v) {
    if (v.Type == EValueType::Null) {
        *key += 'N';
        return;
    }
    *key += 'V';
    if (v.Type == EValueType::String) {
        const uint64_t n = v.Str.size();
        key->append(reinterpret_cast<const char*>(&n), 8);
        *key += v.Str;
    } else {
        key->append(reinterpret_cast<const char*>(&v.Bits), 8);
    }
}

std::string SelfKey(EKind kind, const TRow* row) {
    auto at = [&](int j) { return row ? (*row)[j] : Nul(); };
    std::string key;
    switch (kind) {
        case KInt: AppendKey(&key, at(0)); break;
        case KCastUint: { const V v = at(1); AppendKey(&key, v.Type == EValueType::Null ? v : I((int64_t)v.Bits)); break; }
        case KMod: case KModBoth: { const V v = at(0); AppendKey(&key, v.Type == EValueType::Null ? v : I((int64_t)v.Bits % 7)); break; }
        case KDouble: AppendKey(&key, at(2)); break;
        case KBool: AppendKey(&key, at(3)); break;
        case KString: AppendKey(&key, at(4)); break;
        case KLower: {
            V v = at(4);
            for (auto& ch : v.Str) ch = (char)std::tolower((unsigned char)ch);
            AppendKey(&key, v);
            break;
        }
        default: AppendKey(&key, at(0)); AppendKey(&key, at(4)); break;
    }
    return key;
}

std::string ForeignKey(EKind kind, const TRow& row) {
    if (kind == KModBoth) return SelfKey(KMod, &row);
    if (kind == KCastUint || kind == KMod || kind == KLower) return SelfKey(kind == KLower ? KString : KInt, &row);
    return SelfKey(kind, &row);
}

// The joined rows of the chain: per joined row, the row of every source (-1: a LEFT clause's miss), in lexicographic order
std::vector<std::vector<int64_t>> ModelJoin(const TTable& primary, const std::vector<TTable>& foreign, const std::vector<TSpec>& specs) {
    std::vector<std::vector<int64_t>> joined;
    for (size_t p = 0; p < primary.size(); ++p) joined.push_back({(int64_t)p});
    for (size_t c = 0; c < specs.size(); ++c) {
        std::unordered_map<std::string, std::vector<int64_t>> index;  // the foreign rows of each key, ascending: a nested loop's order
        for (size_t f = 0; f < foreign[c].size(); ++f) index[ForeignKey(specs[c].Kind, foreign[c][f])].push_back((int64_t)f);
        std::vector<std::vector<int64_t>> next;
        for (const auto& row : joined) {
            const int s = specs[c].SelfSource;
            const int64_t r = row[s];
            const TRow* self = r < 0 ? nullptr : s == 0 ? &primary[r] : &foreign[s - 1][r];
            const auto it = index.find(SelfKey(specs[c].Kind, self));
            if (it == index.end()) {
                if (!specs[c].Left) continue;
                next.push_back(row);
                next.back().push_back(-1);
                continue;
            }
            for (int64_t f : it->second) {
                next.push_back(row);
                next.back().push_back(f);
            }
        }
        joined = std::move(next);
    }
    return joined;
}

void CheckRandom(uint64_t seed, size_t rows, int clauses, bool wide) {
    std::mt19937_64 rng(seed);
    const int64_t range = std::max<int64_t>(8, (int64_t)rows / 2);
    const TTable primary = MakeTable(rng, rows, range, false);
    std::vector<TSpec> specs;
    std::vector<TTable> foreign;
    for (int c = 0; c < clauses; ++c) {
        const EKind narrow[] = {KInt, KString, KCastUint, KLower};
        const EKind kind = wide ? (EKind)(rng() % KindCount) : narrow[rng() % 4];
        specs.push_back({kind, (int)(rng() % (uint64_t)(c + 1)), rng() % 2 == 0});
        // a small table for the small key domains keeps the fan-out near 1
        const size_t size = kind == KDouble || kind == KModBoth ? 1 + rng() % 7 : kind == KBool ? 1 + rng() % 2 : (size_t)(rng() % 4 == 0 ? 0 : range);
        foreign.push_back(MakeTable(rng, size, range, true));
    }
    const auto joined = ModelJoin(primary, foreign, specs);
    const std::string what = "seed " + std::to_string(seed) + ", " + std::to_string(rows) + " rows, " + std::to_string(clauses) + " clauses";
    auto value = [&](const std::vector<int64_t>& row, int s, int j) {
        const int64_t r = row[s];
        return r < 0 ? Nul() : s == 0 ? primary[r][j] : foreign[s - 1][r][j];
    };
    TMultiGroupQuery q;
    const auto position = [](int s, int j) { return s == 0 ? j : F(s - 1, j); };
    for (int c = 0; c < clauses; ++c) {
        auto clause = MakeClause(specs[c], foreign[c], position);
        if (c == 0) q.Join = std::move(clause);
        else q.NextJoins.push_back(std::move(clause));
    }
    // the projection: every source's row index and the last clause's string
    for (int s = 0; s <= clauses; ++s) q.Project.push_back(position(s, 5));
    q.Project.push_back(position(clauses, 4));
    TTable want;
    want.reserve(joined.size());
    for (const auto& row : joined) {
        TRow w;
        for (int s = 0; s <= clauses; ++s) w.push_back(value(row, s, 5));
        w.push_back(value(row, clauses, 4));
        want.push_back(std::move(w));
    }
    TQueryStatistics stats;
    Expect(Run(q, primary, &stats), want, __LINE__, what + ", projection");
    EXPECT_EQ(stats.RowsRead, (int64_t)rows);
    // GROUP BY the last clause's string with sum(primary int64), count(clause 0's row index): first-seen groups
    q.Project.clear();
    q.GroupColumns = {position(clauses, 4)};
    q.AggregateItems = {{EAggregateFunction::Sum, 0}, {EAggregateFunction::Count, position(1, 5)}};
    std::unordered_map<std::string, size_t> group;
    TTable groups;
    for (const auto& row : joined) {
        const V k = value(row, clauses, 4);
        std::string key;
        AppendKey(&key, k);
        auto [it, inserted] = group.try_emplace(key, groups.size());
        if (inserted) groups.push_back({k, Nul(), I(0)});
        TRow& g = groups[it->second];
        const V a = value(row, 0, 0);
        if (a.Type != EValueType::Null) g[1] = I((int64_t)((g[1].Type == EValueType::Null ? 0 : g[1].Bits) + a.Bits));
        if (value(row, 1, 5).Type != EValueType::Null) g[2].Bits += 1;
    }
    Expect(Run(q, primary), groups, __LINE__, what + ", group by");
}

// Two clauses against clause 0 alone, its joined rows written to a table (the primary columns, then clause 0's) and
// joined by clause 1 as a single-Join query
void CheckEquivalence(uint64_t seed, size_t rows) {
    std::mt19937_64 rng(seed);
    const int64_t range = std::max<int64_t>(8, (int64_t)rows / 2);
    const TTable primary = MakeTable(rng, rows, range, false);
    const TSpec s0{(EKind)(rng() % KindCount), 0, rng() % 2 == 0}, s1{(EKind)(rng() % KindCount), (int)(rng() % 2), rng() % 2 == 0};
    auto size = [&](EKind kind) { return kind == KDouble || kind == KModBoth ? (size_t)5 : kind == KBool ? (size_t)2 : (size_t)range; };
    const TTable f0 = MakeTable(rng, size(s0.Kind), range, true), f1 = MakeTable(rng, size(s1.Kind), range, true);
    const auto chained = [](int s, int j) { return s == 0 ? j : F(s - 1, j); };
    TMultiGroupQuery two;
    two.Join = MakeClause(s0, f0, chained);
    two.NextJoins = {MakeClause(s1, f1, chained)};
    two.Project = {5, F(0, 5), F(1, 5), F(1, 4)};
    TMultiGroupQuery first;
    first.Join = MakeClause(s0, f0, chained);
    for (int j = 0; j < 6; ++j) first.Project.push_back(j);
    for (int j = 0; j < 6; ++j) first.Project.push_back(F(0, j));
    const TTable staged = Run(first, primary);
    TMultiGroupQuery second;
    second.Join = MakeClause(s1, f1, [](int s, int j) { return s * 6 + j; });
    second.Project = {5, 11, F(0, 5), F(0, 4)};
    Expect(Run(two, primary), Run(second, staged), __LINE__, "equivalence, seed " + std::to_string(seed) + ", " + std::to_string(rows) + " rows");
}

}  // namespace

int main() {
    try {
        TestSnowflake();
        TestStar();
        TestLeftThenInnerNullRule();
        TestPairOrder();
        TestExpressionKeys();
        TestSelfExpressionOverEarlierClause();
        TestDivisionByZeroInKey();
        TestClausesDownstream();
        TestRefusals();
        TestSingleClause();
        uint64_t seed = 1;
        for (size_t rows : {0, 1, 7, 100, 3000, 25000})
            for (int clauses = 2; clauses <= 4; ++clauses)
                for (int rep = 0; rep < 3; ++rep) CheckRandom(seed++, rows, clauses, true);
        CheckRandom(seed++, 1000000, 2, false);
        CheckRandom(seed++, 200000, 3, false);
        for (size_t rows : {0, 5, 300, 20000})
            for (int rep = 0; rep < 4; ++rep) CheckEquivalence(seed++, rows);
    } catch (const std::exception& e) {
        std::fprintf(stderr, "unexpected exception: %s\n", e.what());
        return 100;
    }
    std::printf("multi_join_ut: %d failure(s)\n", Failures);
    return Failures;
}
