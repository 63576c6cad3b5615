// block_combine_keys_ut.cpp — the YQL BlockCombineHashed adapter over key tuples (CreateGpuBlockCombineHashedKeys) against a
// std::map GROUP BY spelled out below, row by row:
//   * (INT64, STRING) keys over three Arrow blocks with non-zero offsets, validity bitmaps and NULLs in keys and values;
//     the strings include "", prefixes of each other, embedded zeros and bytes >= 0x80;
//   * STRING-only keys over more rows than BlockCombineHashedKeysStageRows, in blocks that straddle the threshold;
//   * the refusals: a key whose type changes between blocks, a value count that changes, decreasing offsets
//     (INVALID_ARGUMENT), a BOOLEAN key (UNSUPPORTED); after them the result still holds every accepted block.
// Runs on the GPU box (tests/test_groupby_table.py drives it); exit code = number of failed expectations.
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

using TKey = std::vector<std::optional<std::string>>;  // INT64 components as their 8 bytes

//! One Arrow column of `n` rows at offset `off` (the rows before it are garbage).
struct TCol {
    std::vector<uint64_t> Values;
    std::vector<uint8_t> Data;
    std::vector<int32_t> Offsets;
    std::vector<uint8_t> Validity;
    TArrowColumn Arrow() const { return A; }
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

std::string I(uint64_t v) { return std::string(reinterpret_cast<const char*>(&v), 8); }

struct TGroup {
    uint64_t First = 0, Sum = 0, Count = 0;
    std::optional<int64_t> Min;
};

//! The reference: groups in first-seen order with SUM, COUNT and MIN of an INT64 value.
struct TReference {
    std::map<TKey, size_t> Index;
    std::vector<std::pair<TKey, TGroup>> Groups;
    uint64_t Rows = 0;
    void Add(const TKey& k, std::optional<uint64_t> v) {
        auto it = Index.find(k);
        if (it == Index.end()) {
            it = Index.emplace(k, Groups.size()).first;
            Groups.push_back({k, TGroup{Rows}});
        }
        TGroup& g = Groups[it->second].second;
        if (v) {
            g.Sum += *v;
            ++g.Count;
            const int64_t x = (int64_t)*v;
            g.Min = g.Min ? std::min(*g.Min, x) : x;
        }
        ++Rows;
    }
};

std::vector<TAggregateItem> Aggregates() {
    return {{EAggregateFunction::Sum, 0, -1}, {EAggregateFunction::Count, 0, -1}, {EAggregateFunction::Min, 0, -1}};
}

//! Result row o against the reference, key components in the block's column order (stringAt: which are strings).
void Compare(const IBlockCombineHashedKeys::TResult& r, const TReference& ref, const std::vector<bool>& stringAt) {
    EXPECT_EQ(r.Values.size(), (size_t)3);
    if (r.Values.size() != 3) return;
    EXPECT_EQ(r.Values[0].size(), ref.Groups.size());
    if (r.Values[0].size() != ref.Groups.size()) return;
    for (size_t o = 0; o < ref.Groups.size(); ++o) {
        TKey got;
        size_t ni = 0, si = 0;
        for (bool s : stringAt) {
            if (s) {
                const auto& off = r.StringKeyOffsets[si];
                got.push_back(r.StringKeyValid[si][o] ? std::optional<std::string>(r.StringKeyBytes[si].substr(off[o], off[o + 1] - off[o]))
                                                      : std::nullopt);
                ++si;
            } else {
                got.push_back(r.KeyValid[ni][o] ? std::optional<std::string>(I(r.Keys[ni][o])) : std::nullopt);
                ++ni;
            }
        }
        const TGroup& g = ref.Groups[o].second;
        EXPECT_EQ(got == ref.Groups[o].first, true);
        EXPECT_EQ(r.ValueValid[1][o], (uint8_t)1);
        EXPECT_EQ(r.Values[1][o], g.Count);
        EXPECT_EQ(r.ValueValid[0][o], (uint8_t)(g.Count ? 1 : 0));
        if (g.Count) {
            EXPECT_EQ(r.Values[0][o], g.Sum);
            EXPECT_EQ((int64_t)r.Values[2][o], *g.Min);
        }
    }
}

int Code(const std::function<void()>& f) {
    try {
        f();
    } catch (const TErrorException& e) {
        return e.GetCode();
    }
    return YTGPU_OK;
}

void TupleKeys() {
    std::mt19937_64 rng(11);
    const std::vector<std::string> pool = {"", "a", "ab", "abc", std::string("a\0b", 3), "\x80\xff", "zz", std::string(300, 'q')};
    auto agg = CreateGpuBlockCombineHashedKeys(Aggregates(), 0);
    TReference ref;
    for (int b = 0; b < 3; ++b) {
        const size_t n = 500 + 300 * b;
        std::vector<std::optional<uint64_t>> k0, val;
        std::vector<std::optional<std::string>> k1;
        for (size_t i = 0; i < n; ++i) {
            k0.push_back(rng() % 9 == 0 ? std::nullopt : std::optional<uint64_t>(rng() % 7));
            k1.push_back(rng() % 11 == 0 ? std::nullopt : std::optional<std::string>(pool[rng() % pool.size()]));
            val.push_back(rng() % 5 == 0 ? std::nullopt : std::optional<uint64_t>((uint64_t)((int64_t)(rng() % 2001) - 1000)));
        }
        const TCol c0 = Numeric(YTGPU_TYPE_INT64, k0, 3 + b), c1 = Strings(k1, 5 + b), v0 = Numeric(YTGPU_TYPE_INT64, val, 1 + b);
        agg->AddBlock({c0.Arrow(), c1.Arrow()}, {v0.Arrow()});
        for (size_t i = 0; i < n; ++i) ref.Add({k0[i] ? std::optional<std::string>(I(*k0[i])) : std::nullopt, k1[i]}, val[i]);
    }
    Compare(agg->Finish(), ref, {false, true});
}

void StagingAndRefusals() {
    std::mt19937_64 rng(12);
    auto agg = CreateGpuBlockCombineHashedKeys(Aggregates(), 1000);
    TReference ref;
    const uint64_t total = BlockCombineHashedKeysStageRows + BlockCombineHashedKeysStageRows / 3;
    const uint64_t block = 100003;  // blocks straddle the staging threshold
    for (uint64_t done = 0; done < total; done += block) {
        const size_t n = (size_t)std::min<uint64_t>(block, total - done);
        std::vector<std::optional<std::string>> k;
        std::vector<std::optional<uint64_t>> val;
        for (size_t i = 0; i < n; ++i) {
            k.push_back(rng() % 50 == 0 ? std::nullopt : std::optional<std::string>("url/" + std::to_string(rng() % 1500)));
            val.push_back((uint64_t)(rng() % 1000));
        }
        const TCol c = Strings(k, 2), v = Numeric(YTGPU_TYPE_INT64, val, 0);
        agg->AddBlock({c.Arrow()}, {v.Arrow()});
        for (size_t i = 0; i < n; ++i) ref.Add({k[i]}, val[i]);
        if (done == 0) {  // the refusals, between accepted blocks
            const TCol num = Numeric(YTGPU_TYPE_INT64, {1, 2}, 0), vv = Numeric(YTGPU_TYPE_INT64, {1, 2}, 0);
            EXPECT_EQ(Code([&] { agg->AddBlock({num.Arrow()}, {vv.Arrow()}); }), YTGPU_ERR_INVALID_ARGUMENT);
            const TCol s2 = Strings({std::string("a"), std::string("b")}, 0);
            EXPECT_EQ(Code([&] { agg->AddBlock({s2.Arrow()}, {vv.Arrow(), vv.Arrow()}); }), YTGPU_ERR_INVALID_ARGUMENT);
            TCol bad = Strings({std::string("abc"), std::string("d")}, 0);
            bad.Offsets[1] = 20;  // decreasing offsets
            bad.A.Offsets = bad.Offsets.data();
            EXPECT_EQ(Code([&] { agg->AddBlock({bad.Arrow()}, {vv.Arrow()}); }), YTGPU_ERR_INVALID_ARGUMENT);
            TCol boolean = Numeric(YTGPU_TYPE_BOOLEAN, {1, 0}, 0);
            EXPECT_EQ(Code([&] { agg->AddBlock({boolean.Arrow()}, {vv.Arrow()}); }), YTGPU_ERR_UNSUPPORTED);
        }
    }
    Compare(agg->Finish(), ref, {true});
}

}  // namespace

int main() {
    TupleKeys();
    StagingAndRefusals();
    std::printf("block_combine_keys_ut: %d failure(s)\n", Failures);
    return Failures;
}
