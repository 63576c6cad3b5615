// block_combine_keys_strings_ut.cpp — STRING values in the YQL BlockCombineHashed adapter over key tuples
// (CreateGpuBlockCombineHashedKeys): MIN, MAX, FIRST and COUNT of a string against a std::map GROUP BY spelled out below,
// over more rows than BlockCombineHashedKeysStageRows in blocks that straddle it, with a numeric value column between
// the string ones; then decreasing offsets in a string value (INVALID_ARGUMENT) and a string value without offsets
// (UNSUPPORTED), after which the result still holds every accepted block.
// Runs on the GPU box (tests/test_groupby_table_strings.py drives it); exit code = number of failed expectations.
#include <cstdio>
#include <cstring>
#include <functional>
#include <map>
#include <optional>
#include <random>
#include <string>
#include <vector>

#include "../../include/ytgpu.h"
#include "../yt_query_client.h"

using namespace NYT::NTableClient;
using namespace NYql::NMiniKQL;
using namespace NYT::NQueryClient;

static int Failures = 0;
#define EXPECT_EQ(a, b) do { auto _a = (a); auto _b = (b); if (!(_a == _b)) { ++Failures; std::fprintf(stderr, "%s:%d: EXPECT_EQ(%s, %s) failed\n", __FILE__, __LINE__, #a, #b); } } while (0)

namespace {

//! One Arrow column of `n` rows at offset `off` (the rows before it are garbage).
struct TCol {
    std::vector<uint64_t> Values;
    std::vector<uint8_t> Data;
    std::vector<int32_t> Offsets;
    std::vector<uint8_t> Validity;
    TArrowColumn A;
};

TCol Numeric(uint8_t type, const std::vector<std::optional<uint64_t>>& v, int64_t off) {
    TCol c;
    c.Values.assign(off, 0xdeadbeefull);
    c.Validity.assign((off + v.size() + 7) / 8 + 1, 0xff);
    for (size_t i = 0; i < v.size(); ++i) {
        c.Values.push_back(v[i].value_or(0x5a5a));
        const int64_t bit = off + (int64_t)i;
        if (!v[i]) c.Validity[bit >> 3] &= (uint8_t)~(1u << (bit & 7));
    }
    c.A.Values = c.Values.data();
    c.A.Validity = c.Validity.data();
    c.A.Offset = off;
    c.A.Length = (int64_t)v.size();
    c.A.ValueType = type;
    return c;
}

TCol Strings(const std::vector<std::optional<std::string>>& v, int64_t off) {
    TCol c;
    c.Data.assign(5, 'g');
    c.Offsets.assign(off, 0);
    for (int64_t i = 0; i < off; ++i) c.Offsets[i] = (int32_t)i;
    c.Validity.assign((off + v.size() + 7) / 8 + 1, 0xff);
    for (size_t i = 0; i < v.size(); ++i) {
        c.Offsets.push_back((int32_t)c.Data.size());
        if (v[i]) c.Data.insert(c.Data.end(), v[i]->begin(), v[i]->end());
        else c.Data.insert(c.Data.end(), {'n', 'u'});  // a NULL row's bytes are ignored
        const int64_t bit = off + (int64_t)i;
        if (!v[i]) c.Validity[bit >> 3] &= (uint8_t)~(1u << (bit & 7));
    }
    c.Offsets.push_back((int32_t)c.Data.size());
    c.A.Values = c.Data.data();
    c.A.Validity = c.Validity.data();
    c.A.Offset = off;
    c.A.Length = (int64_t)v.size();
    c.A.ValueType = YTGPU_TYPE_STRING;
    c.A.Offsets = c.Offsets.data();
    return c;
}

struct TGroup {
    uint64_t Count = 0;
    std::optional<std::string> Min, Max, First;
    uint64_t FirstRow = 0;
};

//! The reference: groups in first-seen order (an INT64 key) with MIN, MAX, FIRST and COUNT of a string.
struct TReference {
    std::map<uint64_t, size_t> Index;
    std::vector<std::pair<uint64_t, TGroup>> Groups;
    uint64_t Rows = 0;
    void Add(uint64_t k, const std::optional<std::string>& v) {
        auto it = Index.find(k);
        if (it == Index.end()) {
            it = Index.emplace(k, Groups.size()).first;
            Groups.push_back({k, TGroup{}});
        }
        TGroup& g = Groups[it->second].second;
        if (v) {
            ++g.Count;
            if (!g.Min || *v < *g.Min) g.Min = v;  // std::string compares bytes as unsigned char, the shorter first
            if (!g.Max || *v > *g.Max) g.Max = v;
            if (!g.First) {
                g.First = v;
                g.FirstRow = Rows;
            }
        }
        ++Rows;
    }
};

// values: 0 = a string, 1 = an INT64, 2 = a string; MIN / MAX / FIRST of value 0, COUNT of value 0, MAX of value 2
std::vector<TAggregateItem> Aggregates() {
    return {{EAggregateFunction::Min, 0, -1}, {EAggregateFunction::Max, 0, -1}, {EAggregateFunction::First, 0, -1},
            {EAggregateFunction::Count, 0, -1}, {EAggregateFunction::Sum, 1, -1}, {EAggregateFunction::Max, 2, -1}};
}

std::optional<std::string> At(const IBlockCombineHashedKeys::TResult& r, size_t j, size_t o) {
    if (!r.StringValueValid[j][o]) return std::nullopt;
    const auto& off = r.StringValueOffsets[j];
    return r.StringValueBytes[j].substr(off[o], off[o + 1] - off[o]);
}

int Code(const std::function<void()>& f) {
    try {
        f();
    } catch (const TErrorException& e) {
        return e.GetCode();
    }
    return YTGPU_OK;
}

void StringValues() {
    std::mt19937_64 rng(21);
    const std::vector<std::string> pool = {"", "a", "ab", std::string("a\0", 2), std::string("\0", 1), "\x80\xff", "zz", std::string(300, 'q'),
                                           "http://example.com/a", "http://example.com/ab"};
    auto agg = CreateGpuBlockCombineHashedKeys(Aggregates(), 1000);
    TReference ref, ref2;
    const uint64_t total = BlockCombineHashedKeysStageRows + BlockCombineHashedKeysStageRows / 3;
    const uint64_t block = 100003;  // blocks straddle the staging threshold
    for (uint64_t done = 0; done < total; done += block) {
        const size_t n = (size_t)std::min<uint64_t>(block, total - done);
        std::vector<std::optional<uint64_t>> k, num;
        std::vector<std::optional<std::string>> s, s2;
        for (size_t i = 0; i < n; ++i) {
            k.push_back(rng() % 1500);
            const uint64_t x = rng();
            s.push_back(x % 7 == 0 ? std::nullopt
                                   : std::optional<std::string>(x % 3 ? pool[(x >> 8) % pool.size()] : "u/" + std::to_string((x >> 16) % 100000)));
            s2.push_back(x % 5 == 0 ? std::nullopt : std::optional<std::string>(std::to_string(x >> 40)));
            num.push_back(1);
        }
        const TCol kc = Numeric(YTGPU_TYPE_INT64, k, 1), sc = Strings(s, 3), nc = Numeric(YTGPU_TYPE_INT64, num, 0), sc2 = Strings(s2, 0);
        agg->AddBlock({kc.A}, {sc.A, nc.A, sc2.A});
        for (size_t i = 0; i < n; ++i) {
            ref.Add(*k[i], s[i]);
            ref2.Add(*k[i], s2[i]);
        }
        if (done == 0) {  // the refusals, between accepted blocks
            const TCol k2 = Numeric(YTGPU_TYPE_INT64, {1, 2}, 0), n2 = Numeric(YTGPU_TYPE_INT64, {1, 2}, 0);
            TCol bad = Strings({std::string("abc"), std::string("d")}, 0);
            bad.Offsets[1] = 20;  // decreasing offsets
            bad.A.Offsets = bad.Offsets.data();
            EXPECT_EQ(Code([&] { agg->AddBlock({k2.A}, {bad.A, n2.A, bad.A}); }), YTGPU_ERR_INVALID_ARGUMENT);
            TCol plain = Strings({std::string("abc"), std::string("d")}, 0);
            plain.A.Offsets = nullptr;  // a STRING value without offsets
            EXPECT_EQ(Code([&] { agg->AddBlock({k2.A}, {plain.A, n2.A, plain.A}); }), YTGPU_ERR_UNSUPPORTED);
        }
    }
    const IBlockCombineHashedKeys::TResult r = agg->Finish();
    EXPECT_EQ(r.StringValueBytes.size(), (size_t)4);  // MIN, MAX, FIRST of value 0 and MAX of value 2
    EXPECT_EQ(r.Values.size(), (size_t)6);
    if (r.StringValueBytes.size() != 4 || r.Values.size() != 6) return;
    EXPECT_EQ(r.Keys[0].size(), ref.Groups.size());
    if (r.Keys[0].size() != ref.Groups.size()) return;
    for (size_t o = 0; o < ref.Groups.size(); ++o) {
        const TGroup& g = ref.Groups[o].second;
        EXPECT_EQ(r.Keys[0][o], ref.Groups[o].first);
        EXPECT_EQ(At(r, 0, o), g.Min);
        EXPECT_EQ(At(r, 1, o), g.Max);
        EXPECT_EQ(At(r, 2, o), g.First);
        EXPECT_EQ(At(r, 3, o), ref2.Groups[o].second.Max);
        EXPECT_EQ(r.ValueValid[2][o], (uint8_t)(g.First ? 1 : 0));
        if (g.First) EXPECT_EQ(r.Values[2][o], g.FirstRow);  // a string-valued result's value is its global row
        EXPECT_EQ(r.Values[3][o], g.Count);
    }
}

}  // namespace

int main() {
    StringValues();
    std::printf("block_combine_keys_strings_ut: %d failure(s)\n", Failures);
    return Failures;
}
