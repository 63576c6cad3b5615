// map_join_ut.cpp — the YQL block map join adapter (CreateGpuBlockMapJoin) against a nested-loop join spelled out below:
//   * the four kinds over two right blocks and three left blocks, as Arrow blocks with validity bitmaps and non-zero
//     offsets, two key columns (INT64, DOUBLE) with NULLs on both sides: the SQL rule makes a NULL left key a Left miss and
//     a LeftOnly row, and a NULL right key match nothing;
//   * an empty right side;
//   * a right block of another key type than the left block (throws INVALID_ARGUMENT), and a string key (UNSUPPORTED).
// Runs on the GPU box (tests/test_join_table.py drives it); exit code = number of failed expectations.
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

using TKey = std::optional<uint64_t>;  // a key column's value: payload bits or NULL

//! One Arrow column holding `keys` at `offset` (the rows before it are garbage), with a validity bitmap when any is NULL.
struct TBlockColumn {
    std::vector<uint64_t> Values;
    std::vector<uint8_t> Validity;
    TArrowColumn Column(uint8_t type) const {
        TArrowColumn c;
        c.Values = Values.data();
        c.Validity = Validity.empty() ? nullptr : Validity.data();
        c.Offset = Offset;
        c.Length = Length;
        c.ValueType = type;
        return c;
    }
    int64_t Offset = 0, Length = 0;
};

TBlockColumn MakeColumn(const std::vector<TKey>& keys, int64_t offset) {
    TBlockColumn c;
    c.Offset = offset;
    c.Length = (int64_t)keys.size();
    c.Values.assign(offset + keys.size(), 0xdeadbeefull);
    bool anyNull = false;
    for (const auto& k : keys) anyNull = anyNull || !k;
    if (anyNull) c.Validity.assign((offset + keys.size() + 7) / 8, 0xff);  // the rows before the offset read as valid
    for (size_t i = 0; i < keys.size(); ++i) {
        const size_t at = offset + i;
        if (keys[i]) c.Values[at] = *keys[i];
        else c.Validity[at >> 3] &= (uint8_t)~(1u << (at & 7));
    }
    return c;
}

uint64_t D(double x) {
    uint64_t b;
    std::memcpy(&b, &x, 8);
    return b;
}

using TRow = std::vector<TKey>;  // one key tuple
const uint8_t Types[2] = {YTGPU_TYPE_INT64, YTGPU_TYPE_DOUBLE};

struct TBlock {
    std::vector<TBlockColumn> Columns;
    std::vector<TArrowColumn> Arrow;
};

TBlock MakeBlock(const std::vector<TRow>& rows, int64_t offset) {
    TBlock b;
    for (size_t k = 0; k < 2; ++k) {
        std::vector<TKey> col;
        for (const auto& r : rows) col.push_back(r[k]);
        b.Columns.push_back(MakeColumn(col, offset + (int64_t)k));
    }
    for (size_t k = 0; k < 2; ++k) b.Arrow.push_back(b.Columns[k].Column(Types[k]));
    return b;
}

// right rows (two blocks), over all blocks in order: 0..3 and 4..6
const std::vector<std::vector<TRow>> RightBlocks = {
    {{1, D(1.5)}, {2, D(2.5)}, {std::nullopt, D(1.5)}, {1, D(1.5)}},
    {{3, std::nullopt}, {2, D(2.5)}, {5, D(-0.0)}},
};
const std::vector<std::vector<TRow>> LeftBlocks = {
    {{1, D(1.5)}, {3, std::nullopt}, {std::nullopt, D(1.5)}, {2, D(2.5)}},
    {{5, D(0.0)}, {5, D(-0.0)}, {4, D(4.0)}},
    {{2, D(2.5)}, {1, D(1.5)}, {std::nullopt, std::nullopt}, {7, D(7.0)}, {1, D(2.5)}},
};

bool Matches(const TRow& a, const TRow& b) {
    for (size_t k = 0; k < a.size(); ++k)
        if (!a[k] || !b[k] || *a[k] != *b[k]) return false;  // SQL: NULL matches nothing; doubles by bit pattern
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

void TestKinds(EBlockJoinKind kind, bool emptyRight) {
    auto join = CreateGpuBlockMapJoin(kind, 2);
    std::vector<TRow> right;
    if (!emptyRight) {
        for (size_t b = 0; b < RightBlocks.size(); ++b) {
            TBlock block = MakeBlock(RightBlocks[b], 3 + (int64_t)b);
            join->AddRightBlock(block.Arrow);  // the block's buffers die here: the adapter copies them
            right.insert(right.end(), RightBlocks[b].begin(), RightBlocks[b].end());
        }
    }
    for (size_t b = 0; b < LeftBlocks.size(); ++b) {
        TBlock block = MakeBlock(LeftBlocks[b], 5 + 2 * (int64_t)b);
        auto got = join->ProbeBlock(block.Arrow);
        auto want = Reference(kind, LeftBlocks[b], right);
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

void TestTypeMismatchThrows() {
    EXPECT_EQ(CodeOf([] {
        auto join = CreateGpuBlockMapJoin(EBlockJoinKind::Inner, 1);
        TBlockColumn c = MakeColumn({1, 2, 3}, 1);
        join->AddRightBlock({c.Column(YTGPU_TYPE_UINT64)});
        join->ProbeBlock({c.Column(YTGPU_TYPE_INT64)});
    }), (int)YTGPU_ERR_INVALID_ARGUMENT);
    EXPECT_EQ(CodeOf([] {
        auto join = CreateGpuBlockMapJoin(EBlockJoinKind::LeftSemi, 1);
        TBlockColumn c = MakeColumn({1, 2, 3}, 0);
        join->AddRightBlock({c.Column(YTGPU_TYPE_STRING)});
    }), (int)YTGPU_ERR_UNSUPPORTED);
}

}  // namespace

int main() {
    try {
        for (auto kind : {EBlockJoinKind::Inner, EBlockJoinKind::Left, EBlockJoinKind::LeftSemi, EBlockJoinKind::LeftOnly}) {
            TestKinds(kind, false);
            TestKinds(kind, true);
        }
        // the expected rows of the SQL rule, spelled out for the first left block against both right blocks
        auto want = Reference(EBlockJoinKind::Left, LeftBlocks[0], {RightBlocks[0][0], RightBlocks[0][1], RightBlocks[0][2], RightBlocks[0][3],
                                                                     RightBlocks[1][0], RightBlocks[1][1], RightBlocks[1][2]});
        EXPECT_EQ(want.LeftRows, (std::vector<uint32_t>{0, 0, 1, 2, 3, 3}));
        EXPECT_EQ(want.RightRows, (std::vector<uint32_t>{0, 3, YTGPU_JOIN_NO_ROW, YTGPU_JOIN_NO_ROW, 1, 5}));
        TestTypeMismatchThrows();
    } catch (const std::exception& e) {
        std::fprintf(stderr, "unexpected exception: %s\n", e.what());
        return 100;
    }
    std::printf("map_join_ut: %d failure(s)\n", Failures);
    return Failures;
}
