// yt_query_client.h — the aggregate-side interfaces of the reference that the GPU path plugs into, reduced to what
// the scan -> filter -> GROUP BY hot path touches (interface mirror; a real integration includes the reference's own
// headers instead):
//   columnar batches   IUnversionedColumnarRowBatch::TColumn              yt/yt/client/table_client/row_batch.h:49-202
//   rowset writer      IUnversionedRowsetWriter::Write / Close            yt/yt/client/table_client/unversioned_writer.h:21-45
//   YT QL evaluator    IEvaluator::Run(query, reader, writer, ...)        yt/yt/library/query/engine_api/evaluator.h:17-31
//   CHYT source        ISource::generate() -> DB::Chunk                   yt/chyt/server/secondary_query_source.cpp:293-400
//   YQL block agg      IBlockAggregatorCombineKeys (batched here)         yql/essentials/minikql/comp_nodes/mkql_block_agg_factory.h:46-58
#pragma once

#include <cstdint>
#include <memory>
#include <optional>
#include <string>
#include <vector>

#include "yt_table_client.h"

namespace NYT::NTableClient {

//! One column of a columnar batch: the fields of IUnversionedColumnarRowBatch::TColumn the integer / double decoders
//! read (row_batch.h:49-191).  Pointers borrow the reader's block memory for the life of the batch.
struct TColumnarColumn {
    int Id = 0;
    EValueType Type = EValueType::Int64;
    int64_t StartIndex = 0;
    int64_t ValueCount = 0;
    // TValueBuffer
    const void* Values = nullptr;    // null: the column is all-NULL
    int BitWidth = 64;               // 8/16/32/64, 0 = TBitPackedUnsignedVector
    uint64_t ValuesCount = 0;
    uint64_t BaseValue = 0;
    bool ZigZagEncoded = false;
    const uint8_t* NullBitmap = nullptr;        // TBitmap: bit set = NULL
    const uint32_t* DictionaryIndexes = nullptr;  // TDictionaryEncoding (ZeroMeansNull)
    uint64_t DictionaryIndexCount = 0;
    const uint64_t* RleIndexes = nullptr;         // TRleEncoding
    uint64_t RleCount = 0;
};

struct IUnversionedColumnarRowBatch {
    virtual ~IUnversionedColumnarRowBatch() = default;
    virtual int64_t GetRowCount() const = 0;
    //! MaterializeColumns (row_batch.h:195): the root columns of the batch.
    virtual const std::vector<TColumnarColumn>& MaterializeColumns() = 0;
};
using IUnversionedColumnarRowBatchPtr = std::shared_ptr<IUnversionedColumnarRowBatch>;

//! Pull protocol as everywhere else: nullptr = end of stream, an empty batch = not ready yet.
struct IColumnarReader {
    virtual ~IColumnarReader() = default;
    virtual IUnversionedColumnarRowBatchPtr Read(const TRowBatchReadOptions& options = {}) = 0;
};
using IColumnarReaderPtr = std::shared_ptr<IColumnarReader>;

//! unversioned_writer.h:21-45 (+ IWriterBase::Close).
struct IUnversionedRowsetWriter {
    virtual ~IUnversionedRowsetWriter() = default;
    [[nodiscard]] virtual bool Write(const std::vector<TUnversionedRow>& rows) = 0;
    virtual void Close() = 0;
};
using IUnversionedRowsetWriterPtr = std::shared_ptr<IUnversionedRowsetWriter>;

//! PipeReaderToWriter (yt/yt/client/table_client/adapters.cpp:155-215), the pump of TSimpleJobBase::Run: reads batches of
//! at most BufferRowCount rows / BufferDataWeight bytes and hands them to the writer until the reader is exhausted, then
//! closes the writer.  (The reference waits on the reader's / writer's ready events where this synchronous mirror loops.)
struct TPipeReaderToWriterOptions {
    int64_t BufferRowCount = 10000;
    int64_t BufferDataWeight = 16LL * 1024 * 1024;
};
void PipeReaderToWriter(const ISchemalessMultiChunkReaderPtr& reader, const IUnversionedRowsetWriterPtr& writer,
                        const TPipeReaderToWriterOptions& options = {});

}  // namespace NYT::NTableClient

namespace NYT::NQueryClient {

using namespace NTableClient;

enum class EBinaryOp { None, Less, LessOrEqual, Greater, GreaterOrEqual, Equal, NotEqual };

//! The query shape the GPU path evaluates: SELECT key, sum(value) [, sum(1)] FROM [...] WHERE value <op> constant GROUP BY key.
//! (The reference compiles arbitrary expressions with LLVM; everything else stays on its CPU evaluator.)
struct TGroupQuery {
    int KeyColumn = 0;       // position of the key in the input rows / id of the key column in columnar batches
    int ValueColumn = 1;     // position / id of the aggregated column
    EValueType ValueType = EValueType::Int64;
    EBinaryOp WhereOp = EBinaryOp::None;
    TUnversionedValue WhereConstant{};
    bool WithCount = false;  // adds sum(1): QL has no COUNT (SURVEY appendix 6)
    bool WithMinMax = false; // adds min(value), max(value) (udf/min.c, udf/max.c) after the count column
};

//! The general GROUP BY shape: SELECT g1, .., gK, f1(c1), .., fN(cN) FROM [...] WHERE c <op> constant GROUP BY g1, .., gK with
//! the reference's built-in aggregates (library/query/base/builtin_function_types.cpp:201-254).  Output row = the group
//! items followed by the aggregate items, ids 0..n-1, groups in first-seen order.
enum class EAggregateFunction { Sum, Min, Max, Count /* sum(if(is_null(c), 0, 1)) */, Avg, ArgMin, ArgMax, First };
struct TAggregateItem {
    EAggregateFunction Function = EAggregateFunction::Sum;
    int Column = 0;     // position of the argument in the input rows (argmin / argmax: the returned column)
    int ByColumn = -1;  // argmin / argmax: the minimised / maximised column
};
//! A WHERE expression of AND / OR / NOT over comparisons, IN lists, NULL tests, prefix and substring tests and LIKE
//! patterns, evaluated on the GPU
//! (ytgpu_evaluate_filter: the semantics, three-valued logic included, are in include/ytgpu.h).  Nodes are in postfix
//! order; columns are positions in the input rows.  A constant has the column's type (a mistyped constant is
//! INVALID_ARGUMENT); string constants and IN lists are owned by the expression.
enum class EFilterOp {
    Compare = 1, CompareColumns = 2, In = 3, StartsWith = 4, IsNull = 5, IsNotNull = 6, And = 7, Or = 8, Not = 9, Contains = 10, Like = 11
};
struct TFilterConstant {
    EValueType Type = EValueType::Null;
    uint64_t Bits = 0;    // Int64 / Uint64 / Double bit pattern, Boolean 0 / 1
    std::string Bytes;    // String
    static TFilterConstant Of(const TUnversionedValue& v) {
        TFilterConstant c;
        c.Type = v.Type;
        if (v.Type == EValueType::String) c.Bytes.assign(v.Data.String, v.Length);
        else if (v.Type == EValueType::Boolean) c.Bits = v.Data.Boolean ? 1 : 0;
        else c.Bits = v.Data.Uint64;
        return c;
    }
};
struct TFilterNode {
    EFilterOp Op = EFilterOp::Compare;
    EBinaryOp Cmp = EBinaryOp::None;       // Compare, CompareColumns
    int Column = -1;                       // leaves
    int Column2 = -1;                      // CompareColumns
    TFilterConstant Constant;              // Compare; StartsWith / Contains / Like: the prefix, needle or pattern (a String)
    std::vector<TFilterConstant> List;     // In
    int Escape = -1;                       // Like: the escape byte 0..255, -1 for none
};
struct TFilterExpression {
    std::vector<TFilterNode> Nodes;
    TFilterExpression& Compare(int column, EBinaryOp cmp, const TUnversionedValue& v) {
        Nodes.push_back({EFilterOp::Compare, cmp, column, -1, TFilterConstant::Of(v), {}});
        return *this;
    }
    TFilterExpression& CompareColumns(int column, EBinaryOp cmp, int column2) {
        Nodes.push_back({EFilterOp::CompareColumns, cmp, column, column2, {}, {}});
        return *this;
    }
    TFilterExpression& In(int column, const std::vector<TUnversionedValue>& values) {
        TFilterNode n{EFilterOp::In, EBinaryOp::None, column, -1, {}, {}};
        for (const auto& v : values) n.List.push_back(TFilterConstant::Of(v));
        Nodes.push_back(std::move(n));
        return *this;
    }
    TFilterExpression& StartsWith(int column, const std::string& prefix) {
        TFilterConstant c;
        c.Type = EValueType::String;
        c.Bytes = prefix;
        Nodes.push_back({EFilterOp::StartsWith, EBinaryOp::None, column, -1, c, {}});
        return *this;
    }
    //! QL is_substr(needle, s) / ClickHouse position(s, needle) > 0.
    TFilterExpression& Contains(int column, const std::string& needle) {
        TFilterConstant c;
        c.Type = EValueType::String;
        c.Bytes = needle;
        Nodes.push_back({EFilterOp::Contains, EBinaryOp::None, column, -1, c, {}});
        return *this;
    }
    //! s LIKE pattern (% any bytes, _ one UTF-8 character, the escape byte quotes the next byte); NOT LIKE is Like(...).Not().
    TFilterExpression& Like(int column, const std::string& pattern, std::optional<unsigned char> escape = std::nullopt) {
        TFilterConstant c;
        c.Type = EValueType::String;
        c.Bytes = pattern;
        Nodes.push_back({EFilterOp::Like, EBinaryOp::None, column, -1, c, {}, escape ? (int)*escape : -1});
        return *this;
    }
    TFilterExpression& IsNull(int column) { Nodes.push_back({EFilterOp::IsNull, EBinaryOp::None, column, -1, {}, {}}); return *this; }
    TFilterExpression& IsNotNull(int column) { Nodes.push_back({EFilterOp::IsNotNull, EBinaryOp::None, column, -1, {}, {}}); return *this; }
    TFilterExpression& And() { Nodes.push_back({EFilterOp::And, EBinaryOp::None, -1, -1, {}, {}}); return *this; }
    TFilterExpression& Or() { Nodes.push_back({EFilterOp::Or, EBinaryOp::None, -1, -1, {}, {}}); return *this; }
    TFilterExpression& Not() { Nodes.push_back({EFilterOp::Not, EBinaryOp::None, -1, -1, {}, {}}); return *this; }
};

//! An arithmetic, bitwise, cast, if_null, concat, lower, upper, farm_hash or conditional (comparison, and / or / not,
//! is_null, if) expression, evaluated on the GPU into a computed column (ytgpu_evaluate_expression_strings: the semantics —
//! NULLs, wrap-around, division errors and the branches they follow, casts, ASCII case mapping, the fingerprint — are in
//! include/ytgpu.h).  Nodes are in postfix order; a Column leaf names a position (in the
//! input rows for TMultiGroupQuery::Computed, in the output row for Select).  Binary operands have one type: there is no
//! implicit widening, write Cast.  Select and Having take no string ops; of the predicates they take In over numbers; of
//! the timestamp functions they take the floors.
enum class EExpressionOp {
    Column = 1, Constant = 2, Add = 3, Sub = 4, Mul = 5, Div = 6, Mod = 7, Neg = 8, BitAnd = 9, BitOr = 10, BitXor = 11, BitNot = 12,
    Cast = 13, IfNull = 14, Concat = 15, Lower = 16, Upper = 17, FarmHash = 18,
    Compare = 19, And = 20, Or = 21, Not = 22, IsNull = 23, IsNotNull = 24, If = 25,
    In = 26, IsPrefix = 27, IsSubstr = 28, Like = 29,
    TimestampFloor = 30, FormatTimestamp = 31
};
//! A typed literal: an In list entry.
struct TExpressionLiteral {
    EValueType Type = EValueType::Null;
    uint64_t Bits = 0;                    // Int64 / Uint64 / Double bit pattern, Boolean 0 / 1
    std::string Bytes = {};               // a String's bytes
};
struct TExpressionNode {
    EExpressionOp Op = EExpressionOp::Column;
    int Column = -1;                      // Column; FarmHash: the operand count; Compare: the EBinaryOp; Like: the escape byte or -1;
                                          // TimestampFloor: the ytgpu_timestamp_unit
    EValueType Type = EValueType::Null;   // Constant: its type; Cast: the target type
    uint64_t Bits = 0;                    // Constant: Int64 / Uint64 / Double bit pattern, Boolean 0 / 1
    std::string Bytes = {};               // Constant: a String's bytes; IsPrefix / IsSubstr / Like: the prefix, needle or pattern;
                                          // FormatTimestamp: the format
    std::vector<TExpressionLiteral> List = {};  // In: the entries
};
struct TExpression {
    std::vector<TExpressionNode> Nodes;
    TExpression& Column(int position) { Nodes.push_back({EExpressionOp::Column, position, EValueType::Null, 0}); return *this; }
    TExpression& Constant(const TUnversionedValue& v) {
        if (v.Type == EValueType::String) {
            Nodes.push_back({EExpressionOp::Constant, -1, v.Type, 0, std::string(v.Data.String, v.Length)});
            return *this;
        }
        Nodes.push_back({EExpressionOp::Constant, -1, v.Type, v.Type == EValueType::Boolean ? (v.Data.Boolean ? 1u : 0u) : v.Data.Uint64});
        return *this;
    }
    TExpression& Add() { return Op(EExpressionOp::Add); }
    TExpression& Sub() { return Op(EExpressionOp::Sub); }
    TExpression& Mul() { return Op(EExpressionOp::Mul); }
    TExpression& Div() { return Op(EExpressionOp::Div); }
    TExpression& Mod() { return Op(EExpressionOp::Mod); }
    TExpression& Neg() { return Op(EExpressionOp::Neg); }
    TExpression& BitAnd() { return Op(EExpressionOp::BitAnd); }
    TExpression& BitOr() { return Op(EExpressionOp::BitOr); }
    TExpression& BitXor() { return Op(EExpressionOp::BitXor); }
    TExpression& BitNot() { return Op(EExpressionOp::BitNot); }
    TExpression& Cast(EValueType type) { Nodes.push_back({EExpressionOp::Cast, -1, type, 0}); return *this; }
    TExpression& IfNull() { return Op(EExpressionOp::IfNull); }
    //! concat(a, b) of two strings; lower / upper of a string (ASCII only: a byte >= 0x80 throws YTGPU_ERR_UNSUPPORTED).
    TExpression& Concat() { return Op(EExpressionOp::Concat); }
    TExpression& Lower() { return Op(EExpressionOp::Lower); }
    TExpression& Upper() { return Op(EExpressionOp::Upper); }
    //! farm_hash of the last `count` (1..16) values, of any type: a Uint64, never NULL.
    TExpression& FarmHash(int count) { Nodes.push_back({EExpressionOp::FarmHash, count, EValueType::Null, 0}); return *this; }
    //! a <cmp> b over two values of one type (strings included): a Boolean, NULL if either is NULL.  EBinaryOp Less .. NotEqual
    //! are ytgpu_cmp_op LT .. NE.
    TExpression& Compare(EBinaryOp cmp) { Nodes.push_back({EExpressionOp::Compare, (int)cmp, EValueType::Null, 0}); return *this; }
    //! Kleene and / or / not over Booleans; is_null / is_not_null of any value (never NULL).
    TExpression& And() { return Op(EExpressionOp::And); }
    TExpression& Or() { return Op(EExpressionOp::Or); }
    TExpression& Not() { return Op(EExpressionOp::Not); }
    TExpression& IsNull() { return Op(EExpressionOp::IsNull); }
    TExpression& IsNotNull() { return Op(EExpressionOp::IsNotNull); }
    //! if(c, a, b) over the last three values: a where c is true, b where it is false, NULL where c is NULL.  A division or
    //! case-mapping error in the branch not taken does not throw.
    TExpression& If() { return Op(EExpressionOp::If); }
    //! x in (list): a Boolean, NULL where x is NULL.  The entries have x's type (an all-NULL input column takes theirs) and
    //! none is NULL: a mistyped entry throws YTGPU_ERR_INVALID_ARGUMENT.  Equality is Compare's: NaN never matches, -0.0 = 0.0.
    TExpression& In(const std::vector<TUnversionedValue>& list) {
        TExpressionNode node{EExpressionOp::In, -1, EValueType::Null, 0};
        for (const auto& v : list) {
            TExpressionLiteral e{v.Type, 0, {}};
            if (v.Type == EValueType::String) e.Bytes.assign(v.Data.String, v.Length);
            else if (v.Type == EValueType::Boolean) e.Bits = v.Data.Boolean ? 1 : 0;
            else if (v.Type != EValueType::Null) e.Bits = v.Data.Uint64;
            node.List.push_back(std::move(e));
        }
        Nodes.push_back(std::move(node));
        return *this;
    }
    //! is_prefix(prefix, s), is_substr(needle, s) and s like pattern (% any bytes, _ one UTF-8 character, the escape byte
    //! quotes the next byte) over the string on top: a Boolean, NULL where s is NULL.  An all-NULL input column is a string.
    TExpression& IsPrefix(const std::string& prefix) { return Text(EExpressionOp::IsPrefix, prefix, -1); }
    TExpression& IsSubstr(const std::string& needle) { return Text(EExpressionOp::IsSubstr, needle, -1); }
    TExpression& Like(const std::string& pattern, std::optional<unsigned char> escape = std::nullopt) {
        return Text(EExpressionOp::Like, pattern, escape ? (int)*escape : -1);
    }
    //! timestamp_floor_hour / day / week (from Monday) / month / year of an Int64 or Uint64 of seconds since the epoch, UTC:
    //! the operand's type (an all-NULL input column is an Int64).  A value outside [0, 9999-12-31T23:59:59Z] that is
    //! evaluated, or a week floor before 1970-01-05, throws YTGPU_ERR_UNSUPPORTED.
    TExpression& TimestampFloorHour() { return Floor(0); }
    TExpression& TimestampFloorDay() { return Floor(1); }
    TExpression& TimestampFloorWeek() { return Floor(2); }
    TExpression& TimestampFloorMonth() { return Floor(3); }
    TExpression& TimestampFloorYear() { return Floor(4); }
    //! format_timestamp(t, format): a String, C-locale strftime of t in UTC (the conversions in include/ytgpu.h).  Computed
    //! columns only; the range rule of the floors applies.
    TExpression& FormatTimestamp(const std::string& format) { return Text(EExpressionOp::FormatTimestamp, format, -1); }

private:
    TExpression& Text(EExpressionOp op, const std::string& bytes, int column) {
        Nodes.push_back({op, column, EValueType::Null, 0, bytes});
        return *this;
    }
    TExpression& Op(EExpressionOp op) { Nodes.push_back({op, -1, EValueType::Null, 0}); return *this; }
    TExpression& Floor(int unit) { Nodes.push_back({EExpressionOp::TimestampFloor, unit, EValueType::Null, 0}); return *this; }
};

struct TMultiGroupQuery {
    std::vector<int> GroupColumns;               // positions of the group items in the input rows (1..8)
    std::vector<TAggregateItem> AggregateItems;
    int WhereColumn = -1;                        // position of the filtered column (must be an aggregate / by argument)
    EBinaryOp WhereOp = EBinaryOp::None;
    TUnversionedValue WhereConstant{};
    std::optional<TFilterExpression> Where;      // a general WHERE expression; not together with WhereOp
    //! Computed columns: expressions over positions of the input rows.  Computed column j is named by the position
    //! ComputedColumn(j) wherever an input position may stand: group items, aggregate Column / ByColumn, WhereColumn and the
    //! leaves of Where.  Each one that is named is evaluated once.
    std::vector<TExpression> Computed;
    static constexpr int ComputedColumn(int j) { return -2 - j; }
    static constexpr bool IsComputedColumn(int position) { return position <= -2; }
    //! The output row: expressions over its positions (group items first, then aggregates), e.g. sum(b) + x.  Without it
    //! the output row is the group items followed by the aggregates.
    std::optional<std::vector<TExpression>> Select;
    //! HAVING: a Boolean expression over the output row's positions, as Select's (e.g. sum(x) > 100).  Only the groups where
    //! it is true are written, and RowsWritten counts them.  Select is evaluated over those groups only (its selection), so a
    //! division by zero in a dropped group does not throw.  The program is checked whatever the data: a Having that is not
    //! a Boolean throws on an empty input too.  Without it every group is written.
    std::optional<TExpression> Having;
    //! JOIN (JoinOpHelper, cg_routines/registry.cpp): an inner or left equi-join of the reader's rows (the primary side)
    //! with Foreign's rows on SelfColumns[k] = ForeignColumns[k].  With Join set, every position above that names an input
    //! column names a column of the JOINED row: a primary position as without it, or ForeignColumn(j) for position j of the
    //! foreign rows.  Select and Having keep naming output positions.  A LEFT join's primary row without a match gets NULL
    //! in every foreign column.  Join keys compare as the GROUP BY keys do: NULL equals NULL, doubles by bit pattern.
    //! Join is the FIRST clause; NextJoins holds clauses 2..N (at most kMaxJoinClauses in all), applied left to right:
    //! clause c joins the joined rows of clauses 0..c-1 with its foreign rows, and ForeignColumn(c, j) names position j of
    //! clause c's foreign rows.  The joined rows are ordered by (primary row, foreign row of clause 0, of clause 1, ...).
    //! A key is a column or an expression (ON f.k % 1000 = d.id, ON cast(f.u as int64) = d.id, ON lower(f.host) = d.host):
    //! ComputedColumn(e) in SelfColumns / ForeignColumns names SelfExpressions[e] / ForeignExpressions[e].  A self key
    //! (column or expression leaf) reads primary positions and foreign positions of EARLIER clauses; a foreign expression
    //! reads positions of this clause's foreign rows (plain j).  No key reads a query.Computed position.  Each key
    //! expression is evaluated once over every row of its side, before its join and so before WHERE: a division by zero
    //! in any row throws, even in a row a later WHERE drops.  Keys keep one type per key pair (an all-NULL column takes the
    //! other side's type).  Because NULL equals NULL in every clause, a row that a LEFT clause left without a match, NULL
    //! in that clause's columns, matches a foreign NULL key of a later clause that keys on those columns.  That YT QL
    //! allows several clauses whose keys read the tables joined before, and expressions as join keys evaluated before
    //! WHERE, is recalled, not read.
    struct TJoinClause {
        ISchemalessMultiChunkReaderPtr Foreign;   // the foreign table's rows, in the order the reference fetches them
        std::vector<int> SelfColumns;             // join key positions in the (joined) primary rows (1..8)
        std::vector<int> ForeignColumns;          // the matching positions in the foreign rows
        bool IsLeft = false;
        std::vector<TExpression> SelfExpressions = {};     // the self keys that are expressions: ComputedColumn(e)
        std::vector<TExpression> ForeignExpressions = {};  // the foreign keys that are expressions: ComputedColumn(e)
    };
    std::optional<TJoinClause> Join;
    std::vector<TJoinClause> NextJoins;          // clauses 2..N, in order; they need Join
    static constexpr int kMaxJoinClauses = 8;
    static constexpr int kForeignColumnBase = 1 << 24;
    static constexpr int ForeignColumn(int j) { return kForeignColumnBase + j; }
    static constexpr int ForeignColumn(int clause, int j) { return (clause + 1) * kForeignColumnBase + j; }
    static constexpr bool IsForeignColumn(int position) { return position >= kForeignColumnBase; }
    static constexpr int ForeignClause(int position) { return position / kForeignColumnBase - 1; }
    static constexpr int ForeignIndex(int position) { return position % kForeignColumnBase; }
    //! A query WITHOUT GROUP BY: the output row is these positions of the (joined) input rows, input, computed (string
    //! results included) or foreign columns.  Non-empty exactly when GroupColumns and AggregateItems are empty.  Select then
    //! names positions of this output row, as it names group / aggregate positions otherwise; Having is refused.
    std::vector<int> Project;
    //! ORDER BY: expressions over output-row positions, as Having's, compared in turn.  A bare Column item may name a string
    //! position (a string group item, a string MIN / MAX, a projected string); any other item is a numeric expression.
    struct TOrderItem {
        TExpression Expression;
        bool Descending = false;
    };
    std::vector<TOrderItem> OrderBy;
    //! LIMIT and OFFSET: the rows written are positions [Offset, Offset + Limit) of the ordered rows.  OrderBy needs a Limit
    //! and a non-zero Offset needs OrderBy, as QL's query preparer requires.
    std::optional<int64_t> Limit;
    int64_t Offset = 0;
};

struct TQueryStatistics {
    int64_t RowsRead = 0;
    int64_t RowsWritten = 0;
};

//! IEvaluator::Run (engine_api/evaluator.h:17-31) for TGroupQuery: reads the schemaful rows, aggregates on the GPU and
//! writes one row per group — ids 0..n-1, cleared flags (cg_routines/registry.cpp:283-291), groups in FIRST-SEEN order
//! like InsertGroupRow (registry.cpp:1571-1655), sum = Null when the group has no non-null value (udf/sum.c:12-36).
struct IEvaluator {
    virtual ~IEvaluator() = default;
    virtual TQueryStatistics Run(const TGroupQuery& query, const ISchemalessMultiChunkReaderPtr& reader,
                                 const IUnversionedRowsetWriterPtr& writer) = 0;
    //! The same for TMultiGroupQuery: one ytgpu_scan_filter_groupby_multi_strings call over all rows the reader yields (at
    //! most 2^30 per query fragment).  Every column holds one type of Int64 / Uint64 / Double / Boolean / String (or Null);
    //! a string group item goes through ytgpu_string_value_ids, and min / max / first / count / argmin / argmax take string
    //! arguments.  sum / avg of a string column and a string WHERE column throw YTGPU_ERR_UNSUPPORTED.
    //! Computed columns are evaluated with ytgpu_evaluate_expression_strings, nothing on the host, in QL's order: first those the
    //! WHERE reads, over all rows; then the WHERE, once, as a filter pass (with computed columns the WhereOp form runs as a
    //! one-node COMPARE program, which selects the same rows); then the other computed columns over the selected rows only,
    //! so a division by zero in a row the WHERE drops does not throw.  Select items and Having are evaluated the same way over
    //! the result rows; a bare Column of a string result passes through, arithmetic on it throws YTGPU_ERR_UNSUPPORTED, as does
    //! a numeric op over a string input column.  A computed column may yield a string (concat, lower, upper, if_null): it is
    //! a string column to every consumer (group item, string aggregate argument, WHERE leaf); lower / upper of a non-ASCII
    //! value throws YTGPU_ERR_UNSUPPORTED.  Errors of the calls (a division by zero, a mistyped expression:
    //! YTGPU_ERR_INVALID_ARGUMENT) throw TErrorException.  A query without computed columns and Select runs as before.
    //! With Join, both sides are flattened, the join keys typed (an all-NULL key column takes the other side's type; any
    //! other mismatch, Int64 against Uint64 included, throws YTGPU_ERR_INVALID_ARGUMENT: the caller casts first; string keys
    //! go through one joint ytgpu_string_value_ids call per clause and key), ytgpu_hash_join makes the pairs (a count query,
    //! then the fill), and every column the query reads is gathered at the joined rows.  With several clauses each side is
    //! flattened once and one row map per table is kept: per clause only the self key inputs are gathered at the current
    //! joined rows, the key expressions of both sides are evaluated (ytgpu_evaluate_expression_strings), the clause joins,
    //! and the earlier maps are composed through the pairs' primary rows (ytgpu_gather_column); after the last clause every
    //! column is gathered once from its table.  The joined rows stay below 2^30 (checked after each clause's count query:
    //! YTGPU_ERR_UNSUPPORTED).  Everything above then runs unchanged over the joined rows: WHERE filters joined rows, the SQL
    //! meaning for both kinds.  So, beside the note on division errors: a computed column or WHERE is not evaluated over a
    //! primary row that an INNER join drops, while a join key expression is evaluated over every row of its side before its
    //! join, so its division by zero throws even in a row a later WHERE drops.  RowsRead counts primary rows.  A query
    //! without Join runs exactly as before.
    //! Evaluation order, as QL plans it: scan (+ JOIN) -> WHERE -> computed columns -> GROUP BY -> HAVING -> ORDER BY, OFFSET
    //! and LIMIT -> SELECT -> write.  ORDER BY items are evaluated over the rows WHERE keeps (a projection) or the groups
    //! HAVING keeps only; one ytgpu_order_rows call over those rows gives the window.  Without ORDER BY, LIMIT keeps the first
    //! rows WHERE keeps in input (joined) order, or the first groups HAVING keeps in first-seen order.  SELECT is evaluated
    //! over the window only: a projection's output columns are gathered at the window rows first, a grouped query's Select
    //! runs over the window's groups; so a division by zero outside the window does not throw.  RowsWritten counts the rows
    //! written.  A query that sets none of Project, OrderBy, Limit and Offset runs exactly as before.
    virtual TQueryStatistics Run(const TMultiGroupQuery& query, const ISchemalessMultiChunkReaderPtr& reader,
                                 const IUnversionedRowsetWriterPtr& writer) = 0;
};
using IEvaluatorPtr = std::shared_ptr<IEvaluator>;
IEvaluatorPtr CreateGpuEvaluator();

//! TTopCollector (engine_api/top_collector.h:10-47), the state of ORDER BY ... LIMIT k (OrderOpHelper,
//! cg_routines/registry.cpp:1948): keeps the `limit` smallest rows under the comparator.  The reference maintains a heap
//! row by row; here rows are buffered and the buffer is cut back to `limit` with one GPU sort whenever it has grown to a
//! multiple of the limit.  GetRows() returns the rows in order (ties: earlier rows first).
class TTopCollector {
public:
    TTopCollector(int64_t limit, TComparator comparator);
    void AddRow(TUnversionedRow row);
    std::vector<TUnversionedOwningRow> GetRows();

private:
    void Compact();
    int64_t Limit_;
    TComparator Comparator_;
    std::vector<TUnversionedOwningRow> Rows_;
    size_t CompactAt_;
};

}  // namespace NYT::NQueryClient

namespace NYT::NClickHouseServer {

using namespace NTableClient;

//! What ISource::generate returns here: the result columns of the aggregation as flat vectors (a DB::Chunk of
//! ColumnUInt64 / ColumnNullable(ColumnInt64|UInt64|Float64) / ColumnUInt64 in the real integration).
struct TAggregatedChunk {
    std::vector<uint64_t> Keys;
    std::vector<uint8_t> KeyNulls;      // YT optional key column -> Nullable(UInt64)
    std::vector<uint64_t> Sums;         // bit patterns in the value type
    std::vector<uint8_t> SumNulls;
    std::vector<uint64_t> Counts;       // COUNT(*) is UInt64
    std::vector<uint64_t> Mins, Maxs;   // min(value) / max(value) when requested; NULL where SumNulls is set
    size_t Rows() const { return Keys.size(); }
};

//! TSecondaryQuerySourceBase::generate (secondary_query_source.cpp:293-400) fused with the first stage of
//! DB::Aggregator (executeOnBlock, key64 + AggregateFunctionSum/Count): every columnar batch the reader yields is
//! decoded, PREWHERE-filtered and aggregated on the GPU; partial states of the batches are merged like
//! Aggregator::mergeBlocks.  generate() returns the aggregated chunk once (then an empty chunk = end of stream).
struct IAggregatingSource {
    virtual ~IAggregatingSource() = default;
    virtual TAggregatedChunk generate() = 0;
};
std::unique_ptr<IAggregatingSource> CreateGpuAggregatingSource(IColumnarReaderPtr reader, int keyColumnId, int valueColumnId,
                                                               NQueryClient::EBinaryOp prewhereOp, uint64_t prewhereConstant,
                                                               uint64_t groupCountHint, bool withMinMax = false);

}  // namespace NYT::NClickHouseServer

namespace NYql::NMiniKQL {

//! A fixed-width arrow::ArrayData as TArrowBlock hands it to an aggregator (buffers[0] validity, buffers[1] values), or
//! an Arrow binary / utf8 array (buffers[1] offsets, buffers[2] data): element i is then the bytes [Offsets[Offset + i],
//! Offsets[Offset + i + 1]) of Values.  That YQL's block String / Utf8 columns use these 32-bit offsets is recalled, not read.
struct TArrowColumn {
    const void* Values = nullptr;
    const uint8_t* Validity = nullptr;  // LSB bit order, 1 = valid; null = no nulls
    int64_t Offset = 0;
    int64_t Length = 0;
    uint8_t ValueType = 0;  // YTGPU_TYPE_INT64 / UINT64 / DOUBLE, or YTGPU_TYPE_STRING with Offsets
    const int32_t* Offsets = nullptr;  // STRING only: Offset + Length + 1 entries
};

//! BlockCombineHashed with one key column and the sum / count aggregators (mkql_block_agg.cpp:1234-1400 drives
//! IBlockAggregatorCombineKeys::InitKey / UpdateKey row by row, mkql_block_agg_factory.h:46-58): here a whole block is one
//! call, the per-key states of all blocks are merged at Finish (IAggColumnBuilder::Build).
struct IBlockCombineHashed {
    virtual ~IBlockCombineHashed() = default;
    virtual void AddBlock(const TArrowColumn& keys, const TArrowColumn& values) = 0;
    struct TResult {
        std::vector<uint64_t> Keys, Sums, Counts;
        std::vector<uint64_t> Mins, Maxs;         // the min / max aggregators' states (mkql_block_agg_minmax.cpp), when requested
        std::vector<uint8_t> KeyValid, SumValid;  // Optional<T> outputs: 1 = has a value (Mins / Maxs share SumValid)
    };
    virtual TResult Finish() = 0;
};
std::unique_ptr<IBlockCombineHashed> CreateGpuBlockCombineHashed(uint64_t groupCountHint, bool withMinMax = false);

//! BlockCombineHashed over a key TUPLE with a list of aggregates (mkql_block_agg.cpp:1234-1400), on one GPU GROUP BY table
//! (ytgpu_groupby_table_*) that stays on the device for the whole input.
//!   * Keys: INT64, UINT64, DOUBLE, and STRING as an Arrow binary / utf8 array with 32-bit Offsets; 1..8 columns.  The key
//!     tuple is the numeric keys in their order, then the string keys in theirs.  Values: INT64, UINT64 or DOUBLE columns,
//!     and STRING as an Arrow binary / utf8 array with 32-bit Offsets; TAggregateItem::Column / ByColumn index them.  A
//!     STRING value takes MIN, MAX, FIRST, COUNT, and ARGMIN / ARGMAX as the value, the bound or both (that YQL's block
//!     MIN / MAX take String / Utf8 arguments is recalled, not read).  Types and counts come from the first block; a later
//!     block that differs is INVALID_ARGUMENT, as are decreasing or negative offsets; any other type, and a STRING column
//!     without offsets, is UNSUPPORTED.  The checks run before a block is staged, so a refused block changes nothing.
//!   * NULL keys form one group (SQL GROUP BY); doubles group by bit pattern; strings by their bytes.  Groups come out in
//!     first-seen order, the aggregates with the semantics of ytgpu_scan_filter_groupby_multi (header).
//!   * Blocks are copied into pinned host staging and folded into the table once BlockCombineHashedKeysStageRows rows are
//!     staged, and at Finish: an update has fixed launch and synchronisation costs that small YQL blocks would pay each.
//!   * Result: Keys / KeyValid per numeric key, StringKeyBytes / StringKeyOffsets (Arrow layout, groups + 1 offsets) /
//!     StringKeyValid per string key, Values / ValueValid per aggregate (bit patterns of the result type; AVG a double).
//!     A string-valued aggregate (MIN / MAX / FIRST of a STRING value, ARGMIN / ARGMAX whose Column is one) has its global
//!     input row in Values and its bytes in StringValueBytes / StringValueOffsets / StringValueValid, one per such
//!     aggregate in aggregate order.
constexpr uint64_t BlockCombineHashedKeysStageRows = 1ull << 20;  // from bench_groupby_table.py's block-size legs (DESIGN.md 7)
struct IBlockCombineHashedKeys {
    virtual ~IBlockCombineHashedKeys() = default;
    virtual void AddBlock(const std::vector<TArrowColumn>& keys, const std::vector<TArrowColumn>& values) = 0;
    struct TResult {
        std::vector<std::vector<uint64_t>> Keys;
        std::vector<std::vector<uint8_t>> KeyValid;  // numeric keys: 1 = has a value
        std::vector<std::string> StringKeyBytes;
        std::vector<std::vector<int32_t>> StringKeyOffsets;
        std::vector<std::vector<uint8_t>> StringKeyValid;
        std::vector<std::vector<uint64_t>> Values;
        std::vector<std::vector<uint8_t>> ValueValid;
        std::vector<std::string> StringValueBytes;
        std::vector<std::vector<int32_t>> StringValueOffsets;
        std::vector<std::vector<uint8_t>> StringValueValid;
    };
    virtual TResult Finish() = 0;
};
std::unique_ptr<IBlockCombineHashedKeys> CreateGpuBlockCombineHashedKeys(std::vector<NYT::NQueryClient::TAggregateItem> aggregates, uint64_t groupCountHint);

//! BlockMapJoinCore (mkql_block_map_join.cpp, in the same comp_nodes directory): a map join of Arrow blocks, the right
//! (dimension) side held in a hash table, every left block probed against it.  The operator's name, its kinds and its
//! output order below are RECALLED, NOT READ: SURVEY.md read only the block-aggregate files of comp_nodes.
//!   * AddRightBlock adds a block of right key columns (as many blocks as needed, before the first probe).  The right
//!     side is built into one GPU join table (ytgpu_join_table_build) on the first ProbeBlock; every later probe reuses it.
//!   * ProbeBlock joins one left block.  LeftRows are rows of that block; RightRows index the right rows over all right
//!     blocks in the order they were added.  Inner / Left: the pairs in ascending (left, right) order, a Left miss as
//!     (l, YTGPU_JOIN_NO_ROW).  LeftSemi / LeftOnly: each left row with / without a match, once, ascending; RightRows empty.
//!   * NULLs follow SQL: a key tuple with a NULL component matches nothing (YTGPU_JOIN_NULLS_NEVER_MATCH), so a NULL left
//!     key is a Left miss and a LeftOnly row.  Doubles compare by bit pattern (-0.0 is not +0.0, a NaN matches only the
//!     same NaN bits): what YQL's map join does with such keys is not known here.
//!   * Key types INT64, UINT64, DOUBLE and STRING.  A STRING key is an Arrow binary / utf8 array with 32-bit Offsets;
//!     keys compare by their bytes (that YQL's map join compares string keys by bytes is recalled, not read).  The table
//!     keeps the right side's strings in its own dictionary (ytgpu_join_table_build_strings); a left block passes its bytes
//!     from Offsets[Offset] on, with starts and lengths made on the host.  A STRING key without Offsets (views, dictionary
//!     arrays, large_binary) and any other type throw UNSUPPORTED; a key count, a type that differs between the right
//!     blocks, a position that is a string key in one block and numeric in another, and decreasing offsets throw
//!     INVALID_ARGUMENT.
enum class EBlockJoinKind { Inner, Left, LeftSemi, LeftOnly };

struct IBlockMapJoin {
    virtual ~IBlockMapJoin() = default;
    virtual void AddRightBlock(const std::vector<TArrowColumn>& keys) = 0;
    struct TResult {
        std::vector<uint32_t> LeftRows, RightRows;
    };
    virtual TResult ProbeBlock(const std::vector<TArrowColumn>& leftKeys) = 0;
};
std::unique_ptr<IBlockMapJoin> CreateGpuBlockMapJoin(EBlockJoinKind kind, uint32_t keyCount);

}  // namespace NYql::NMiniKQL
