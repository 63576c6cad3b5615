// map_join_strings_ut.cpp — the YQL block map join adapter (CreateGpuBlockMapJoin) with STRING keys against a nested-loop
// join spelled out below:
//   * the four kinds with STRING-only keys and with (INT64, STRING) keys, over two right blocks and three left blocks, as
//     Arrow blocks with non-zero offsets, validity bitmaps and NULLs on both sides; the values include "", prefixes of each
//     other, embedded zeros and bytes >= 0x80;
//   * the refusals: decreasing offsets (INVALID_ARGUMENT), a STRING key on one side against a numeric key on the other
//     (INVALID_ARGUMENT).
// Runs on the GPU box (tests/test_join_table_strings.py drives it); exit code = number of failed expectations.
#include <cstdio>
#include <cstring>
#include <optional>
#include <string>
#include <vector>

#include "../../include/ytgpu.h"
#include "../yt_query_client.h"

using namespace NYT::NTableClient;
using namespace NYql::NMiniKQL;

static int Failures = 0;
#define EXPECT_EQ(a, b) do { auto _a = (a); auto _b = (b); if (!(_a == _b)) { ++Failures; std::fprintf(stderr, "%s:%d: EXPECT_EQ(%s, %s) failed\n", __FILE__, __LINE__, #a, #b); } } while (0)

namespace {

// A key component: NULL, or its bytes (an INT64 component as its 8 little-endian bytes, so byte equality is value equality).
using TKey = std::optional<std::string>;
using TRow = std::vector<TKey>;

std::string I(uint64_t v) { return std::string(reinterpret_cast<const char*>(&v), 8); }
std::string S(const char* p, size_t n) { return std::string(p, n); }

//! One Arrow column holding `keys` at `offset` (the rows before it are garbage), with a validity bitmap when any is NULL.
struct TBlockColumn {
    std::vector<uint64_t> Values;  // INT64
    std::vector<uint8_t> Data;     // STRING
    std::vector<int32_t> Offsets;
    std::vector<uint8_t> Validity;
    int64_t Offset = 0, Length = 0;
    uint8_t Type = 0;

    TArrowColumn Column() const {
        TArrowColumn c;
        c.Values = Type == YTGPU_TYPE_STRING ? (const void*)Data.data() : (const void*)Values.data();
        c.Validity = Validity.empty() ? nullptr : Validity.data();
        c.Offset = Offset;
        c.Length = Length;
        c.ValueType = Type;
        c.Offsets = Type == YTGPU_TYPE_STRING ? Offsets.data() : nullptr;
        return c;
    }
};

TBlockColumn MakeColumn(uint8_t type, const std::vector<TKey>& keys, int64_t offset) {
    TBlockColumn c;
    c.Type = type;
    c.Offset = offset;
    c.Length = (int64_t)keys.size();
    bool anyNull = false;
    for (const auto& k : keys) anyNull = anyNull || !k;
    if (anyNull) c.Validity.assign((offset + keys.size() + 7) / 8, 0xff);  // the rows before the offset read as valid
    if (type == YTGPU_TYPE_STRING) {
        for (int64_t i = 0; i < offset; ++i) {  // garbage values before the window
            c.Offsets.push_back((int32_t)c.Data.size());
            c.Data.insert(c.Data.end(), {'g', 'a', 'r'});
        }
    } else {
        c.Values.assign(offset, 0xdeadbeefull);
    }
    for (size_t i = 0; i < keys.size(); ++i) {
        const size_t at = offset + i;
        if (!keys[i]) c.Validity[at >> 3] &= (uint8_t)~(1u << (at & 7));
        if (type == YTGPU_TYPE_STRING) {
            c.Offsets.push_back((int32_t)c.Data.size());
            if (keys[i]) c.Data.insert(c.Data.end(), keys[i]->begin(), keys[i]->end());
            else c.Data.insert(c.Data.end(), {'n', 'u'});  // a NULL row's bytes are ignored
        } else {
            uint64_t v = 0xdeadbeefull;
            if (keys[i]) std::memcpy(&v, keys[i]->data(), 8);
            c.Values.push_back(v);
        }
    }
    if (type == YTGPU_TYPE_STRING) {
        c.Offsets.push_back((int32_t)c.Data.size());
        c.Data.insert(c.Data.end(), {'t', 'a', 'i', 'l'});  // bytes past the window
    }
    return c;
}

struct TBlock {
    std::vector<TBlockColumn> Columns;
    std::vector<TArrowColumn> Arrow;
};

TBlock MakeBlock(const std::vector<uint8_t>& types, const std::vector<TRow>& rows, int64_t offset) {
    TBlock b;
    for (size_t k = 0; k < types.size(); ++k) {
        std::vector<TKey> col;
        for (const auto& r : rows) col.push_back(r[k]);
        b.Columns.push_back(MakeColumn(types[k], col, offset + (int64_t)k));
    }
    for (const auto& c : b.Columns) b.Arrow.push_back(c.Column());
    return b;
}

bool Matches(const TRow& a, const TRow& b) {
    for (size_t k = 0; k < a.size(); ++k)
        if (!a[k] || !b[k] || *a[k] != *b[k]) return false;  // SQL: NULL matches nothing; bytes compare as bytes
    return true;
}

IBlockMapJoin::TResult Reference(EBlockJoinKind kind, const std::vector<TRow>& left, const std::vector<TRow>& right) {
    IBlockMapJoin::TResult r;
    for (uint32_t l = 0; l < left.size(); ++l) {
        std::vector<uint32_t> hits;
        for (uint32_t f = 0; f < right.size(); ++f)
            if (Matches(left[l], right[f])) hits.push_back(f);
        switch (kind) {
            case EBlockJoinKind::Inner:
            case EBlockJoinKind::Left:
                for (uint32_t f : hits) {
                    r.LeftRows.push_back(l);
                    r.RightRows.push_back(f);
                }
                if (hits.empty() && kind == EBlockJoinKind::Left) {
                    r.LeftRows.push_back(l);
                    r.RightRows.push_back(YTGPU_JOIN_NO_ROW);
                }
                break;
            case EBlockJoinKind::LeftSemi:
                if (!hits.empty()) r.LeftRows.push_back(l);
                break;
            case EBlockJoinKind::LeftOnly:
                if (hits.empty()) r.LeftRows.push_back(l);
                break;
        }
    }
    return r;
}

const std::string Zero = S("a\0b", 3), High = S("\xff\x80z", 3);

// STRING-only keys: right rows 0..4 and 5..7
const std::vector<std::vector<TRow>> RightStrings = {
    {{"a"}, {""}, {std::nullopt}, {"ab"}, {"a"}},
    {{Zero}, {High}, {S("a\0", 2)}},
};
const std::vector<std::vector<TRow>> LeftStrings = {
    {{"a"}, {std::nullopt}, {""}, {"abc"}},
    {{Zero}, {S("a", 1)}, {S("a\0", 2)}, {High}, {"b"}},
    {{"ab"}, {std::nullopt}, {S("a\0c", 3)}},
};

// (INT64, STRING) keys
const std::vector<std::vector<TRow>> RightMixed = {
    {{I(1), "x"}, {I(2), ""}, {std::nullopt, "x"}, {I(1), "x"}},
    {{I(3), std::nullopt}, {I(2), Zero}, {I(1), "y"}},
};
const std::vector<std::vector<TRow>> LeftMixed = {
    {{I(1), "x"}, {I(3), std::nullopt}, {std::nullopt, "x"}, {I(2), ""}},
    {{I(2), Zero}, {I(2), "a"}, {I(1), "y"}},
    {{I(1), "y"}, {I(1), "x"}, {std::nullopt, std::nullopt}, {I(7), "x"}, {I(2), S("a\0b\0", 4)}},
};

void TestKinds(EBlockJoinKind kind, const std::vector<uint8_t>& types, const std::vector<std::vector<TRow>>& rightBlocks,
               const std::vector<std::vector<TRow>>& leftBlocks) {
    auto join = CreateGpuBlockMapJoin(kind, (uint32_t)types.size());
    std::vector<TRow> right;
    for (size_t b = 0; b < rightBlocks.size(); ++b) {
        TBlock block = MakeBlock(types, rightBlocks[b], 3 + (int64_t)b);
        join->AddRightBlock(block.Arrow);  // the block's buffers die here: the adapter copies them
        right.insert(right.end(), rightBlocks[b].begin(), rightBlocks[b].end());
    }
    for (size_t b = 0; b < leftBlocks.size(); ++b) {
        TBlock block = MakeBlock(types, leftBlocks[b], 5 + 2 * (int64_t)b);
        auto got = join->ProbeBlock(block.Arrow);
        auto want = Reference(kind, leftBlocks[b], right);
        EXPECT_EQ(got.LeftRows, want.LeftRows);
        EXPECT_EQ(got.RightRows, want.RightRows);
    }
}

int CodeOf(void (*fn)()) {
    try {
        fn();
    } catch (const TErrorException& e) {
        return e.GetCode();
    }
    return 0;
}

void TestRefusals() {
    EXPECT_EQ(CodeOf([] {  // decreasing offsets in a left block
        auto join = CreateGpuBlockMapJoin(EBlockJoinKind::Inner, 1);
        TBlockColumn r = MakeColumn(YTGPU_TYPE_STRING, {TKey{"a"}, TKey{"b"}}, 0);
        join->AddRightBlock({r.Column()});
        TBlockColumn l = MakeColumn(YTGPU_TYPE_STRING, {TKey{"ab"}, TKey{"cd"}}, 1);
        l.Offsets[2] = l.Offsets[3] + 1;
        join->ProbeBlock({l.Column()});
    }), (int)YTGPU_ERR_INVALID_ARGUMENT);
    EXPECT_EQ(CodeOf([] {  // decreasing offsets in a right block
        auto join = CreateGpuBlockMapJoin(EBlockJoinKind::LeftSemi, 1);
        TBlockColumn r = MakeColumn(YTGPU_TYPE_STRING, {TKey{"a"}, TKey{"b"}, TKey{"c"}}, 0);
        r.Offsets[1] = 3;
        join->AddRightBlock({r.Column()});
    }), (int)YTGPU_ERR_INVALID_ARGUMENT);
    EXPECT_EQ(CodeOf([] {  // a STRING right key against an INT64 left key
        auto join = CreateGpuBlockMapJoin(EBlockJoinKind::Inner, 1);
        TBlockColumn r = MakeColumn(YTGPU_TYPE_STRING, {TKey{"a"}}, 0);
        join->AddRightBlock({r.Column()});
        TBlockColumn l = MakeColumn(YTGPU_TYPE_INT64, {TKey{I(1)}}, 0);
        join->ProbeBlock({l.Column()});
    }), (int)YTGPU_ERR_INVALID_ARGUMENT);
    EXPECT_EQ(CodeOf([] {  // an INT64 right key against a STRING left key
        auto join = CreateGpuBlockMapJoin(EBlockJoinKind::LeftOnly, 1);
        TBlockColumn r = MakeColumn(YTGPU_TYPE_INT64, {TKey{I(1)}}, 0);
        join->AddRightBlock({r.Column()});
        TBlockColumn l = MakeColumn(YTGPU_TYPE_STRING, {TKey{"a"}}, 0);
        join->ProbeBlock({l.Column()});
    }), (int)YTGPU_ERR_INVALID_ARGUMENT);
    EXPECT_EQ(CodeOf([] {  // a STRING key without offsets stays unsupported
        auto join = CreateGpuBlockMapJoin(EBlockJoinKind::Inner, 1);
        TBlockColumn r = MakeColumn(YTGPU_TYPE_STRING, {TKey{"a"}}, 0);
        TArrowColumn c = r.Column();
        c.Offsets = nullptr;
        join->AddRightBlock({c});
    }), (int)YTGPU_ERR_UNSUPPORTED);
}

}  // namespace

int main() {
    try {
        for (auto kind : {EBlockJoinKind::Inner, EBlockJoinKind::Left, EBlockJoinKind::LeftSemi, EBlockJoinKind::LeftOnly}) {
            TestKinds(kind, {YTGPU_TYPE_STRING}, RightStrings, LeftStrings);
            TestKinds(kind, {YTGPU_TYPE_INT64, YTGPU_TYPE_STRING}, RightMixed, LeftMixed);
            TestKinds(kind, {YTGPU_TYPE_STRING}, {}, LeftStrings);  // no right block
        }
        // the expected rows, spelled out for the second STRING-only left block against both right blocks
        std::vector<TRow> right = RightStrings[0];
        right.insert(right.end(), RightStrings[1].begin(), RightStrings[1].end());
        auto want = Reference(EBlockJoinKind::Left, LeftStrings[1], right);
        EXPECT_EQ(want.LeftRows, (std::vector<uint32_t>{0, 1, 1, 2, 3, 4}));
        EXPECT_EQ(want.RightRows, (std::vector<uint32_t>{5, 0, 4, 7, 6, YTGPU_JOIN_NO_ROW}));
        TestRefusals();
    } catch (const std::exception& e) {
        std::fprintf(stderr, "unexpected exception: %s\n", e.what());
        return 100;
    }
    std::printf("map_join_strings_ut: %d failure(s)\n", Failures);
    return Failures;
}
