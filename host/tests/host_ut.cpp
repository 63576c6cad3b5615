// host_ut.cpp — the reference's own unit tests for this path, re-stated against the GPU-backed adapters
// (same factories, same expectations):
//   TPartitionerTest.{Ordered,Hash,ColumnBased}   yt/yt/ytlib/unittests/partitioner_ut.cpp:31-124
//   sorting / merging reader behaviour             sorting_reader.cpp:58-81,163-188; sorted_merging_reader_ut.cpp
// Runs on the GPU box (pytest -m gpu drives it); exit code = number of failed expectations.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <array>
#include <random>
#include <set>
#include <string>

#include "../../include/ytgpu.h"
#include "../yt_table_client.h"

using namespace NYT::NTableClient;

static int Failures = 0;
#define EXPECT_EQ(a, b) do { auto _a = (a); auto _b = (b); if (!(_a == _b)) { ++Failures; std::fprintf(stderr, "%s:%d: EXPECT_EQ(%s, %s) failed\n", __FILE__, __LINE__, #a, #b); } } while (0)
#define EXPECT_TRUE(a) do { if (!(a)) { ++Failures; std::fprintf(stderr, "%s:%d: EXPECT_TRUE(%s) failed\n", __FILE__, __LINE__, #a); } } while (0)
#define EXPECT_THROW_WITH_SUBSTRING(stmt, sub) do { bool _t = false; try { stmt; } catch (const TErrorException& e) { _t = std::string(e.what()).find(sub) != std::string::npos; if (!_t) std::fprintf(stderr, "  got message: %s\n", e.what()); } if (!_t) { ++Failures; std::fprintf(stderr, "%s:%d: expected error containing \"%s\"\n", __FILE__, __LINE__, sub); } } while (0)

static TUnversionedOwningRow MakeRow(std::vector<int64_t> values) {
    TUnversionedOwningRowBuilder b;
    for (auto v : values) b.AddValue(MakeUnversionedInt64Value(v));
    return b.FinishRow();
}

static void TestOrdered() {  // partitioner_ut.cpp:31-51
    std::vector<TOwningKeyBound> bounds;
    bounds.push_back(TOwningKeyBound::MakeUniversal(false));
    bounds.push_back(TOwningKeyBound::FromRow(MakeRow({1}), true, false));
    bounds.push_back(TOwningKeyBound::FromRow(MakeRow({6}), false, false));
    bounds.push_back(TOwningKeyBound::FromRow(MakeRow({8}), true, false));
    bounds.push_back(TOwningKeyBound::FromRow(MakeRow({8}), true, false));
    auto partitioner = CreateOrderedPartitioner(std::move(bounds), TComparator({ESortOrder::Ascending}));
    EXPECT_EQ(5, partitioner->GetPartitionCount());
    EXPECT_EQ(0, partitioner->GetPartitionIndex(MakeRow({0})));
    EXPECT_EQ(1, partitioner->GetPartitionIndex(MakeRow({1})));
    EXPECT_EQ(1, partitioner->GetPartitionIndex(MakeRow({5})));
    EXPECT_EQ(1, partitioner->GetPartitionIndex(MakeRow({6})));
    EXPECT_EQ(1, partitioner->GetPartitionIndex(MakeRow({6, 42})));
    EXPECT_EQ(2, partitioner->GetPartitionIndex(MakeRow({7})));
    EXPECT_EQ(4, partitioner->GetPartitionIndex(MakeRow({42})));
}

static void TestHash() {  // partitioner_ut.cpp:53-67
    auto p0 = CreateHashPartitioner(10, 1, 0);
    auto p42 = CreateHashPartitioner(7, 1, 42);
    EXPECT_EQ(10, p0->GetPartitionCount());
    EXPECT_EQ(7, p42->GetPartitionCount());
    EXPECT_EQ(1, p0->GetPartitionIndex(MakeRow({0})));
    EXPECT_EQ(1, p0->GetPartitionIndex(MakeRow({0, 7})));
    EXPECT_EQ(9, p0->GetPartitionIndex(MakeRow({35})));
    EXPECT_EQ(6, p42->GetPartitionIndex(MakeRow({0})));
    EXPECT_EQ(5, p42->GetPartitionIndex(MakeRow({37})));
    EXPECT_EQ(1, p42->GetPartitionIndex(MakeRow({39})));
    // batched form == per-row form
    std::vector<TUnversionedOwningRow> keep;
    std::vector<TUnversionedRow> rows;
    for (int i = 0; i < 1000; ++i) keep.push_back(MakeRow({i * 7919LL, i}));
    for (auto& r : keep) rows.push_back(r);
    auto batched = p42->GetPartitionIndexes(rows);
    for (int i = 0; i < 1000; i += 97) EXPECT_EQ(batched[i], p42->GetPartitionIndex(rows[i]));
}

static void TestColumnBased() {  // partitioner_ut.cpp:69-124
    auto partitioner = CreateColumnBasedPartitioner(5, 1);
    auto makeRow = [](TUnversionedValue partitionValue) {
        TUnversionedOwningRowBuilder b;
        b.AddValue(MakeUnversionedStringValue("foo", 0));
        partitionValue.Id = 1;
        b.AddValue(partitionValue);
        b.AddValue(MakeUnversionedInt64Value(42, 2));
        return b.FinishRow();
    };
    EXPECT_EQ(5, partitioner->GetPartitionCount());
    EXPECT_EQ(3, partitioner->GetPartitionIndex(makeRow(MakeUnversionedInt64Value(3))));
    EXPECT_EQ(0, partitioner->GetPartitionIndex(makeRow(MakeUnversionedUint64Value(0))));
    EXPECT_THROW_WITH_SUBSTRING(partitioner->GetPartitionIndex(makeRow(MakeUnversionedDoubleValue(1.5))), "Invalid partition column value type");
    EXPECT_THROW_WITH_SUBSTRING(partitioner->GetPartitionIndex(makeRow(MakeUnversionedInt64Value(-1))), "Received negative partition index");
    EXPECT_THROW_WITH_SUBSTRING(partitioner->GetPartitionIndex(makeRow(MakeUnversionedUint64Value(5))), "Partition index is out of bounds");
    TUnversionedOwningRowBuilder b;
    b.AddValue(MakeUnversionedStringValue("foo", 0));
    EXPECT_THROW_WITH_SUBSTRING(partitioner->GetPartitionIndex(b.FinishRow()), "Row does not contain partition column");
}

// local 3-way compare used only to CHECK the reader outputs here (type order first, then value)
static int CompareValues(const TUnversionedValue& l, const TUnversionedValue& r) {
    if (l.Type != r.Type) return l.Type < r.Type ? -1 : 1;
    switch (l.Type) {
        case EValueType::Int64: return l.Data.Int64 < r.Data.Int64 ? -1 : l.Data.Int64 > r.Data.Int64;
        case EValueType::Uint64: return l.Data.Uint64 < r.Data.Uint64 ? -1 : l.Data.Uint64 > r.Data.Uint64;
        case EValueType::Double: {
            double a = l.Data.Double, b = r.Data.Double;
            if (a < b) return -1;
            if (a > b) return 1;
            if (std::isnan(a)) return std::isnan(b) ? 0 : 1;
            return std::isnan(b) ? -1 : 0;
        }
        case EValueType::Boolean: return (int)l.Data.Boolean - (int)r.Data.Boolean;
        case EValueType::String: { int c = l.AsStringBuf().compare(r.AsStringBuf()); return (c > 0) - (c < 0); }
        default: return 0;
    }
}

static std::vector<TUnversionedOwningRow> RandomRows(int n, uint32_t seed, int tag) {
    std::mt19937 rng(seed);
    std::vector<TUnversionedOwningRow> rows;
    std::vector<std::string> words = {"", "a", "ab", "abc", "b", std::string("a\0", 2), "zz"};
    for (int i = 0; i < n; ++i) {
        TUnversionedOwningRowBuilder b;
        switch (rng() % 5) {
            case 0: b.AddValue(MakeUnversionedNullValue()); break;
            case 1: b.AddValue(MakeUnversionedInt64Value((int64_t)(rng() % 7) - 3)); break;
            case 2: b.AddValue(MakeUnversionedUint64Value(rng() % 3)); break;
            case 3: b.AddValue(MakeUnversionedDoubleValue((rng() % 2) ? -0.0 : (double)(rng() % 3))); break;
            default: b.AddValue(MakeUnversionedStringValue(words[rng() % words.size()])); break;
        }
        b.AddValue(MakeUnversionedStringValue(words[rng() % words.size()]));
        b.AddValue(MakeUnversionedInt64Value(tag * 1000000 + i));  // payload: origin
        rows.push_back(b.FinishRow());
    }
    return rows;
}

static std::vector<TUnversionedRow> ReadAll(ISchemalessMultiChunkReaderPtr reader, int maxRows) {
    std::vector<TUnversionedRow> out;
    static std::vector<IUnversionedRowBatchPtr> keep;  // keep batches (and their holders) alive for the checks
    TRowBatchReadOptions opts;
    opts.MaxRowsPerRead = maxRows;
    while (auto batch = reader->Read(opts)) {
        EXPECT_TRUE(batch->GetRowCount() <= maxRows);
        for (auto row : batch->MaterializeRows()) out.push_back(row);
        keep.push_back(batch);
    }
    EXPECT_TRUE(reader->Read(opts) == nullptr);  // stays at end of stream
    return out;
}

static void TestSortingReader() {
    for (auto orders : {std::vector<ESortOrder>{ESortOrder::Ascending, ESortOrder::Ascending},
                        std::vector<ESortOrder>{ESortOrder::Descending, ESortOrder::Ascending}}) {
        auto input = RandomRows(25000, 7, 0);
        std::vector<size_t> expect(input.size());
        for (size_t i = 0; i < expect.size(); ++i) expect[i] = i;
        auto less = [&](size_t a, size_t b) {
            for (int c = 0; c < 2; ++c) {
                int r = CompareValues(input[a][c], input[b][c]);
                if (orders[c] == ESortOrder::Descending) r = -r;
                if (r) return r < 0;
            }
            return false;
        };
        std::stable_sort(expect.begin(), expect.end(), less);
        auto reader = CreateSortingReader(CreateInMemoryReader(input), TComparator(orders));
        auto rows = ReadAll(reader, 1000);
        EXPECT_EQ(rows.size(), input.size());
        bool same = rows.size() == input.size();
        for (size_t i = 0; same && i < rows.size(); ++i) same = rows[i][2].Data.Int64 == (int64_t)expect[i];
        EXPECT_TRUE(same);  // identical to the stable CPU sort (one of the orders std::sort may produce)
    }
    auto empty = CreateSortingReader(CreateInMemoryReader({}), TComparator({ESortOrder::Ascending}));
    EXPECT_TRUE(empty->Read() == nullptr);
}

// 1 KB string keys: the normalised key would exceed 256 bytes, the rowset sort refines by key words instead
static void TestSortingReaderLongKeys() {
    std::mt19937 rng(11);
    const std::string prefix(1000, 'p');
    std::vector<TUnversionedOwningRow> input;
    for (int i = 0; i < 5000; ++i) {
        std::string key = prefix.substr(0, 900 + rng() % 100);
        for (int k = rng() % 40; k > 0; --k) key.push_back("ab\0"[rng() % 3]);
        TUnversionedOwningRowBuilder b;
        b.AddValue(MakeUnversionedStringValue(key));
        b.AddValue(MakeUnversionedInt64Value(i));
        input.push_back(b.FinishRow());
    }
    for (auto order : {ESortOrder::Ascending, ESortOrder::Descending}) {
        std::vector<size_t> expect(input.size());
        for (size_t i = 0; i < expect.size(); ++i) expect[i] = i;
        std::stable_sort(expect.begin(), expect.end(), [&](size_t a, size_t b) {
            int r = CompareValues(input[a][0], input[b][0]);
            return (order == ESortOrder::Descending ? -r : r) < 0;
        });
        auto rows = ReadAll(CreateSortingReader(CreateInMemoryReader(input), TComparator({order})), 1000);
        bool same = rows.size() == input.size();
        for (size_t i = 0; same && i < rows.size(); ++i) same = rows[i][1].Data.Int64 == (int64_t)expect[i];
        EXPECT_TRUE(same);
    }
}

static void TestSortedMergingReader() {
    TComparator comparator({ESortOrder::Ascending, ESortOrder::Ascending});
    std::vector<ISchemalessMultiChunkReaderPtr> readers;
    std::vector<std::vector<TUnversionedOwningRow>> runs;
    for (int r = 0; r < 5; ++r) {
        auto rows = RandomRows(r == 3 ? 0 : 3000 + 500 * r, 100 + r, r);
        std::stable_sort(rows.begin(), rows.end(), [](const auto& a, const auto& b) {
            for (int c = 0; c < 2; ++c) { int x = CompareValues(a[c], b[c]); if (x) return x < 0; }
            return false;
        });
        runs.push_back(rows);
        readers.push_back(CreateInMemoryReader(rows));
    }
    auto rows = ReadAll(CreateSortedMergingReader(readers, comparator), 10000);
    size_t total = 0;
    for (auto& r : runs) total += r.size();
    EXPECT_EQ(rows.size(), total);
    bool ok = true;
    for (size_t i = 1; ok && i < rows.size(); ++i) {
        int c = 0;
        for (int k = 0; k < 2 && !c; ++k) c = CompareValues(rows[i - 1][k], rows[i][k]);
        if (c > 0) ok = false;
        if (c == 0) {  // CompareStreams: ties by table (reader) index, then stream order
            int64_t a = rows[i - 1][2].Data.Int64, b = rows[i][2].Data.Int64;
            if (a / 1000000 > b / 1000000) ok = false;
        }
    }
    EXPECT_TRUE(ok);
}

// TSortedJoiningReader: sorted_merging_reader_ut.cpp:353-395 (table data), :698-1350 (the expected sequences in the tests'
// comments), :1499-1640 (stress test: emitted foreign rows == foreign rows whose join key occurs among the primary rows).
namespace {
constexpr int TableIndexId = 3;
struct TRawRow { const char* C0; int64_t C1; uint64_t C2; };
const std::vector<TRawRow> JoinTable0 = {{"ab", 1, 21}, {"ab", 1, 22}, {"bb", 2, 23}, {"bb", 2, 24}, {"cb", 3, 25}, {"cb", 3, 26}};
const std::vector<TRawRow> JoinTable1 = {{"aa", 1, 1}, {"ab", 3, 3}, {"ac", 5, 5}, {"ba", 7, 7}, {"bb", 9, 9}, {"bc", 11, 11}, {"ca", 13, 13}, {"cb", 15, 15}, {"cc", 17, 17}};
const std::vector<TRawRow> JoinTable2 = {{"aa", 2, 2}, {"ab", 4, 4}, {"ac", 6, 6}, {"ba", 8, 8}, {"bb", 10, 10}, {"bc", 12, 12}, {"ca", 14, 14}, {"cb", 16, 16}, {"cc", 18, 18}};

ISchemalessMultiChunkReaderPtr FakeReader(const std::vector<TRawRow>& table, int tableIndex) {  // TSchemalessMultiChunkFakeReader
    std::vector<TUnversionedOwningRow> rows;
    for (auto& r : table) {
        TUnversionedOwningRowBuilder b;
        b.AddValue(MakeUnversionedStringValue(r.C0, 0));
        b.AddValue(MakeUnversionedInt64Value(r.C1, 1));
        b.AddValue(MakeUnversionedUint64Value(r.C2, 2));
        b.AddValue(MakeUnversionedInt64Value(tableIndex, TableIndexId));
        rows.push_back(b.FinishRow());
    }
    return CreateInMemoryReader(rows);
}

std::string RowToString(TUnversionedRow row) {
    char buf[128];
    std::snprintf(buf, sizeof(buf), "%.*s %lld %llu %lld", (int)row[0].Length, row[0].Data.String, (long long)row[1].Data.Int64,
                  (unsigned long long)row[2].Data.Uint64, (long long)row[3].Data.Int64);
    return buf;
}
}  // namespace

static void TestSortedJoiningReader() {
    auto asc = [](int n) { return TComparator(std::vector<ESortOrder>(n, ESortOrder::Ascending)); };
    auto run = [&](std::vector<ISchemalessMultiChunkReaderPtr> primary, std::vector<ISchemalessMultiChunkReaderPtr> foreign, int sortLen) {
        std::vector<IUnversionedRowBatchPtr> keep;
        std::vector<std::string> out;
        auto reader = CreateSortedJoiningReader(primary, asc(sortLen), asc(std::min(sortLen, 2)), foreign, asc(1), true, TableIndexId);
        TRowBatchReadOptions opts;
        opts.MaxRowsPerRead = 5;
        while (auto batch = reader->Read(opts)) {
            for (auto row : batch->MaterializeRows()) out.push_back(RowToString(row));
            keep.push_back(batch);
        }
        return out;
    };
    {  // SortedJoiningReaderForeignBeforeMultiplePrimary (:698-745)
        auto rows = run({FakeReader(JoinTable0, 1), FakeReader(JoinTable1, 2)}, {FakeReader(JoinTable2, 0)}, 3);
        std::vector<std::string> expect = {
            "aa 2 2 0", "aa 1 1 2", "ab 4 4 0", "ab 1 21 1", "ab 1 22 1", "ab 3 3 2", "ac 6 6 0", "ac 5 5 2", "ba 8 8 0", "ba 7 7 2",
            "bb 10 10 0", "bb 2 23 1", "bb 2 24 1", "bb 9 9 2", "bc 12 12 0", "bc 11 11 2", "ca 14 14 0", "ca 13 13 2",
            "cb 16 16 0", "cb 3 25 1", "cb 3 26 1", "cb 15 15 2", "cc 18 18 0", "cc 17 17 2"};
        EXPECT_TRUE(rows == expect);
    }
    {  // SortedJoiningReaderMultiplePrimaryBeforeForeign (:820-868)
        auto rows = run({FakeReader(JoinTable0, 0), FakeReader(JoinTable1, 1)}, {FakeReader(JoinTable2, 2)}, 3);
        std::vector<std::string> expect = {
            "aa 1 1 1", "aa 2 2 2", "ab 1 21 0", "ab 1 22 0", "ab 3 3 1", "ab 4 4 2", "ac 5 5 1", "ac 6 6 2", "ba 7 7 1", "ba 8 8 2",
            "bb 2 23 0", "bb 2 24 0", "bb 9 9 1", "bb 10 10 2", "bc 11 11 1", "bc 12 12 2", "ca 13 13 1", "ca 14 14 2",
            "cb 3 25 0", "cb 3 26 0", "cb 15 15 1", "cb 16 16 2", "cc 17 17 1", "cc 18 18 2"};
        EXPECT_TRUE(rows == expect);
    }
    {  // SortedJoiningReaderMultipleForeignBeforePrimary (:940-976) and ...ForeignBeforePrimary (:1146-1182)
        std::vector<std::string> expect = {"ab 3 3 0", "ab 4 4 1", "ab 1 21 2", "ab 1 22 2", "bb 9 9 0", "bb 10 10 1", "bb 2 23 2", "bb 2 24 2",
                                           "cb 15 15 0", "cb 16 16 1", "cb 3 25 2", "cb 3 26 2"};
        EXPECT_TRUE(run({FakeReader(JoinTable0, 2)}, {FakeReader(JoinTable1, 0), FakeReader(JoinTable2, 1)}, 3) == expect);
        EXPECT_TRUE(run({FakeReader(JoinTable0, 2)}, {FakeReader(JoinTable1, 0), FakeReader(JoinTable2, 1)}, 1) == expect);
    }
    {  // SortedJoiningReaderPrimaryBeforeMultipleForeign (:1043-1079) and ...PrimaryBeforeForeign (:1249-1285)
        std::vector<std::string> expect = {"ab 1 21 0", "ab 1 22 0", "ab 3 3 1", "ab 4 4 2", "bb 2 23 0", "bb 2 24 0", "bb 9 9 1", "bb 10 10 2",
                                           "cb 3 25 0", "cb 3 26 0", "cb 15 15 1", "cb 16 16 2"};
        EXPECT_TRUE(run({FakeReader(JoinTable0, 0)}, {FakeReader(JoinTable1, 1), FakeReader(JoinTable2, 2)}, 3) == expect);
        EXPECT_TRUE(run({FakeReader(JoinTable0, 0)}, {FakeReader(JoinTable1, 1), FakeReader(JoinTable2, 2)}, 1) == expect);
    }
    {  // stress (:1499-1640): random int64 tables; the foreign rows that survive are exactly those with a primary key
        std::mt19937 rng(42);
        for (int it = 0; it < 5; ++it) {
            auto table = [&](int rows, int range, int tableIndex) {
                std::vector<int64_t> keys(rows);
                for (auto& k : keys) k = rng() % range;
                std::sort(keys.begin(), keys.end());
                std::vector<TUnversionedOwningRow> out;
                for (int i = 0; i < rows; ++i) {
                    TUnversionedOwningRowBuilder b;
                    b.AddValue(MakeUnversionedInt64Value(keys[i], 0));
                    b.AddValue(MakeUnversionedInt64Value(i, 1));
                    b.AddValue(MakeUnversionedInt64Value(tableIndex, 2));
                    out.push_back(b.FinishRow());
                }
                return out;
            };
            const int range = 1 + rng() % 400;
            auto primary = table(rng() % 3000, range, 0), foreign1 = table(rng() % 3000, range, 1), foreign2 = table(rng() % 3000, range, 2);
            std::set<int64_t> primaryKeys;
            for (auto& r : primary) primaryKeys.insert(r[0].Data.Int64);
            std::vector<std::array<int64_t, 3>> expect;
            for (auto* t : {&primary, &foreign1, &foreign2})
                for (auto& r : *t)
                    if (t == &primary || primaryKeys.count(r[0].Data.Int64)) expect.push_back({r[0].Data.Int64, r[2].Data.Int64, r[1].Data.Int64});
            std::sort(expect.begin(), expect.end());
            auto reader = CreateSortedJoiningReader({CreateInMemoryReader(primary)}, asc(1), asc(1),
                                                    {CreateInMemoryReader(foreign1), CreateInMemoryReader(foreign2)}, asc(1), false, 2);
            std::vector<IUnversionedRowBatchPtr> keep;
            std::vector<std::array<int64_t, 3>> got;
            while (auto batch = reader->Read()) {
                for (auto row : batch->MaterializeRows()) got.push_back({row[0].Data.Int64, row[2].Data.Int64, row[1].Data.Int64});
                keep.push_back(batch);
            }
            EXPECT_TRUE(got == expect);
        }
    }
}

// TPartitionMultiChunkWriter (schemaless_chunk_writer.cpp:1509-1535,1604-1667): rows reach the sink as horizontal blocks
// tagged with their partition, in input order per partition; blocks are cut by the size threshold and the buffer limit.
static void TestPartitionMultiChunkWriter() {
    struct TSink : IPartitionBlockSink {
        std::vector<TPartitionBlock> Blocks;
        bool WriteBlock(TPartitionBlock block) override {
            Blocks.push_back(std::move(block));
            return true;
        }
    };
    auto sink = std::make_shared<TSink>();
    auto partitioner = CreateHashPartitioner(4, 1, 0);
    TPartitionWriterConfig config;
    config.BlockSize = 3000;
    config.MaxBufferSize = 7000;
    auto writer = CreatePartitionMultiChunkWriter(config, partitioner, sink);
    std::mt19937_64 rng(17);
    std::vector<TUnversionedOwningRow> keep;
    for (int i = 0; i < 5000; ++i) {
        TUnversionedOwningRowBuilder b;
        b.AddValue(MakeUnversionedInt64Value((int64_t)(rng() % 1000) - 500, 0));
        b.AddValue(MakeUnversionedInt64Value(i, 1));
        b.AddValue(MakeUnversionedStringValue(std::string(rng() % 20, 'a' + (char)(i % 26)), 2));
        keep.push_back(b.FinishRow());
    }
    size_t blocksBeforeClose = 0;
    for (size_t off = 0; off < keep.size(); off += 700) {
        std::vector<TUnversionedRow> batch(keep.begin() + off, keep.begin() + std::min(keep.size(), off + 700));
        (void)writer->Write(batch);
    }
    blocksBeforeClose = sink->Blocks.size();
    writer->Close();
    EXPECT_TRUE(blocksBeforeClose > 4);                    // the thresholds cut blocks while writing
    EXPECT_TRUE(sink->Blocks.size() >= blocksBeforeClose);  // Close flushes the rest
    ytgpu_context* ctx = nullptr;
    ytgpu_error err{};
    EXPECT_EQ(ytgpu_context_create(0, nullptr, &ctx, &err), (int)YTGPU_OK);
    std::vector<std::vector<int64_t>> seen(4);  // per partition: the sequence numbers in arrival order
    int64_t total = 0;
    for (auto& block : sink->Blocks) {
        // a partition is flushed by DumpLargeBlocks AFTER the rows of one Write() were appended (as in the reference):
        // a block may exceed BlockSize by at most that batch's bytes
        EXPECT_TRUE((int64_t)block.Data.size() <= config.BlockSize + 700 * 48);
        std::vector<ytgpu_value> values((size_t)block.RowCount * 3);
        std::vector<uint32_t> counts((size_t)block.RowCount);
        EXPECT_EQ(ytgpu_decode_horizontal_block(ctx, block.Data.data(), block.Data.size(), (uint32_t)block.RowCount, 3, values.data(),
                                                counts.data(), YTGPU_MEM_HOST, &err), (int)YTGPU_OK);
        for (int64_t r = 0; r < block.RowCount; ++r) {
            EXPECT_EQ(counts[r], 3u);
            const int64_t key = (int64_t)values[r * 3].data, seq = (int64_t)values[r * 3 + 1].data;
            EXPECT_EQ(partitioner->GetPartitionIndex(MakeRow({key})), block.PartitionIndex);
            EXPECT_EQ(keep[seq][0].Data.Int64, key);
            EXPECT_EQ(values[r * 3 + 2].length, keep[seq][2].Length);
            seen[block.PartitionIndex].push_back(seq);
            ++total;
            if (Failures > 10) break;
        }
    }
    EXPECT_EQ(total, 5000);
    for (auto& s : seen) EXPECT_TRUE(std::is_sorted(s.begin(), s.end()));  // input order inside every partition
    ytgpu_context_destroy(ctx);
}

// 1 KB string keys and bounds: the ordered partitioner compares key words (the normalised key would exceed 256 bytes).
// Every row written through the partition writer lands in the partition a CPU upper_bound over TestKey gives it.
static void TestPartitionMultiChunkWriterLongKeys() {
    std::mt19937 rng(13);
    const std::string prefix(1000, 'p');
    auto makeKey = [&] {
        std::string key = prefix.substr(0, 900 + rng() % 100);
        for (int k = rng() % 40; k > 0; --k) key.push_back("ab\0"[rng() % 3]);
        return key;
    };
    std::vector<TUnversionedOwningRow> keep;
    for (int i = 0; i < 3000; ++i) {
        TUnversionedOwningRowBuilder b;
        b.AddValue(MakeUnversionedStringValue(makeKey(), 0));
        b.AddValue(MakeUnversionedInt64Value(i, 1));
        keep.push_back(b.FinishRow());
    }
    std::vector<TUnversionedOwningRow> pivots;
    for (int j = 0; j < 15; ++j) {
        TUnversionedOwningRowBuilder b;
        b.AddValue(MakeUnversionedStringValue(makeKey()));
        pivots.push_back(b.FinishRow());
    }
    std::sort(pivots.begin(), pivots.end(), [](const auto& a, const auto& b) { return CompareValues(a[0], b[0]) < 0; });
    std::vector<TOwningKeyBound> bounds{TOwningKeyBound::MakeUniversal(false)};
    for (size_t j = 0; j < pivots.size(); ++j) bounds.push_back(TOwningKeyBound::FromRow(pivots[j], j % 3 != 0, false));
    // TOrderedPartitioner::GetPartitionIndex (partitioner.cpp:41-57) on the CPU: upper_bound with !TestKey, minus one
    auto testKey = [](const TUnversionedOwningRow& row, const TOwningKeyBound& bound) {
        const int c = bound.Prefix.GetCount() ? CompareValues(row[0], bound.Prefix[0]) : 0;
        return c > 0 || (c == 0 && bound.IsInclusive);
    };
    std::vector<int> expect;
    for (auto& row : keep) {
        auto it = std::upper_bound(bounds.begin(), bounds.end(), row, [&](const auto& r, const auto& b) { return !testKey(r, b); });
        expect.push_back((int)(it - bounds.begin()) - 1);
    }
    struct TSink : IPartitionBlockSink {
        std::vector<TPartitionBlock> Blocks;
        bool WriteBlock(TPartitionBlock block) override {
            Blocks.push_back(std::move(block));
            return true;
        }
    };
    auto sink = std::make_shared<TSink>();
    TPartitionWriterConfig config;
    config.BlockSize = 64 << 10;
    config.MaxBufferSize = 256 << 10;
    auto writer = CreatePartitionMultiChunkWriter(config, CreateOrderedPartitioner(bounds, TComparator({ESortOrder::Ascending})), sink);
    for (size_t off = 0; off < keep.size(); off += 500) {
        std::vector<TUnversionedRow> batch(keep.begin() + off, keep.begin() + std::min(keep.size(), off + 500));
        (void)writer->Write(batch);
    }
    writer->Close();
    ytgpu_context* ctx = nullptr;
    ytgpu_error err{};
    EXPECT_EQ(ytgpu_context_create(0, nullptr, &ctx, &err), (int)YTGPU_OK);
    std::vector<int> got(keep.size(), -1);
    for (auto& block : sink->Blocks) {
        std::vector<ytgpu_value> values((size_t)block.RowCount * 2);
        std::vector<uint32_t> counts((size_t)block.RowCount);
        EXPECT_EQ(ytgpu_decode_horizontal_block(ctx, block.Data.data(), block.Data.size(), (uint32_t)block.RowCount, 2, values.data(),
                                                counts.data(), YTGPU_MEM_HOST, &err), (int)YTGPU_OK);
        for (int64_t r = 0; r < block.RowCount; ++r) got[(size_t)values[r * 2 + 1].data] = block.PartitionIndex;
    }
    EXPECT_TRUE(got == expect);
    EXPECT_TRUE(std::set<int>(expect.begin(), expect.end()).size() > 8);  // the keys spread over the partitions
    ytgpu_context_destroy(ctx);
}

int main() {
    try {
        TestOrdered();
        TestHash();
        TestColumnBased();
        TestSortingReader();
        TestSortingReaderLongKeys();
        TestSortedMergingReader();
        TestSortedJoiningReader();
        TestPartitionMultiChunkWriter();
        TestPartitionMultiChunkWriterLongKeys();
    } catch (const std::exception& e) {
        std::fprintf(stderr, "unexpected exception: %s\n", e.what());
        return 100;
    }
    std::printf("host_ut: %d failure(s)\n", Failures);
    return Failures;
}
