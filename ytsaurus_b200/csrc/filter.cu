// filter.cu — WHERE expressions over several columns: AND / OR / NOT of comparisons, IN lists, NULL tests, string
// prefix and substring tests and LIKE patterns, evaluated into a selection bitmap / bytemap / row list
// (ytgpu_evaluate_filter, semantics in ytgpu.h).
//
// One pass over the rows, separate from the aggregation: the result bitmap has the layout of a BOOLEAN column with
// bit_width 1, so ytgpu_scan_filter_groupby_multi[_strings] aggregates the selected rows through its existing {EQ, 1}
// predicate, and no aggregation kernel changes.  The kernel is an interpreter of a postfix program:
//   * one thread per row and 32 consecutive rows per warp, so direct columns load coalesced and the 32-row result is one
//     __ballot_sync word of the bitmap (whole words, no atomics);
//   * every lane runs the same node, so the interpreter loop does not diverge; the program, the referenced columns' views,
//     the head of the (sorted) IN lists and of the string constants are staged in shared memory once per CTA, the rest of
//     the lists and constants is read through __ldg;
//   * the truth stack is two bits per entry (bit 0 TRUE, bit 1 FALSE, neither NULL) in one 32-bit register: 16 entries,
//     Kleene AND / OR / NOT are two bit operations each, and nothing goes to local memory;
//   * an RLE column finds its run from a hint that lane 0 finds once per 32 rows (rle_pos_from, as groupby_multi);
//   * CONTAINS and LIKE run the bit-parallel matcher of strings.cuh over patterns compiled on the host and staged in
//     shared memory after the constants.  The kernel is a template on "the program has pattern nodes", chosen by the host
//     from the checked program, so programs without them run the same code as before.
// The column checks, compact column tables, staging and upload are program.cuh's, shared with expression.cu; the IN-list
// and pattern formats are strings.cuh's.  The IN search stays here: through a shared helper it compiled differently.
#include <algorithm>
#include <vector>

#include "program.cuh"
#include "scan.cuh"

using namespace ytgpu;

namespace {

constexpr int kFilterThreads = 256;
constexpr u32 kStagedConstBytes = 4096;   // bytes of string constants kept in shared memory per CTA
constexpr u32 kMaxFilterColumns = 2 * YTGPU_FILTER_MAX_NODES;  // distinct columns one program can reference

// T = 1, F = 2, NULL = 0 (bit 0: the value is TRUE, bit 1: it is FALSE)
constexpr u32 kTrue = 1, kFalse = 2, kNull = 0;

struct NodeDev {
    u8 op;
    u8 cmp;
    u8 is_string;  // the node's column(s) are string columns: col / col2 index the string table
    u8 pad;
    u16 col, col2;  // compact column tables (referenced columns only)
    u32 length;     // string constant bytes / IN entries
    u64 constant;   // scalar constant bits / string constant offset / first IN entry (in the sorted list)
};
static_assert(sizeof(NodeDev) == 24, "NodeDev layout");

struct FilterArgs {
    const NodeDev* nodes;
    u32 node_count;
    u32 scalar_count, string_count;
    const ColumnDev* scalars;
    const StringDev* strings;
    const u64* lists;  // sorted IN entries (scalars: minmax order words; strings: (offset << 32) | length)
    u32 list_count, staged_list;
    const u8* consts;
    u32 const_bytes, staged_const;
    const u8* patterns;   // compiled CONTAINS / LIKE patterns (strings.cuh), all staged in shared memory
    u32 pattern_bytes;
    u64 n;
    u32* bitmap;         // 2 * ceil(n / 64) words of 32 bits
    u8* bytemap;         // nullable
    u64* word_counts;    // nullable: popcount of every 32-bit bitmap word (for the row list)
    u32 bytemap_vec;     // the bytemap is 16-byte aligned: whole 32-row groups are written as two 16-byte stores
    unsigned long long* result;  // [0] selected count, [1] error bits
};

__device__ __forceinline__ u64 load_list(const FilterArgs& A, const u64* s_list, u64 k) {
    return k < A.staged_list ? s_list[k] : __ldg(A.lists + k);
}

// The constant bytes [off, off + len) as a (heap, value) pair: the shared-memory copy when it holds them.
__device__ __forceinline__ const u8* const_heap(const FilterArgs& A, const u8* s_const, u64 off, u32 len) {
    return off + len <= A.staged_const ? s_const : A.consts;
}

// The shared-memory offset of the compiled patterns: after the staged constants, 16-byte aligned.
__host__ __device__ __forceinline__ size_t pattern_smem_offset(size_t before) { return (before + 15) & ~(size_t)15; }

template <bool kPatterns>
__global__ void __launch_bounds__(kFilterThreads) filter_kernel(const FilterArgs A) {
    extern __shared__ __align__(16) unsigned char smem[];
    NodeDev* s_nodes = reinterpret_cast<NodeDev*>(smem);
    ColumnDev* s_scalars = reinterpret_cast<ColumnDev*>(s_nodes + A.node_count);
    StringDev* s_strings = reinterpret_cast<StringDev*>(s_scalars + A.scalar_count);
    u64* s_list = reinterpret_cast<u64*>(s_strings + A.string_count);
    u8* s_const = reinterpret_cast<u8*>(s_list + A.staged_list);
    u8* s_pat = nullptr;
    if constexpr (kPatterns) {
        s_pat = smem + pattern_smem_offset((size_t)(s_const + A.staged_const - smem));
        const uint4* src = reinterpret_cast<const uint4*>(A.patterns);
        uint4* dst = reinterpret_cast<uint4*>(s_pat);
        for (u32 k = threadIdx.x; k < A.pattern_bytes / 16; k += blockDim.x) dst[k] = src[k];
    }
    {
        const u32* src = reinterpret_cast<const u32*>(A.nodes);
        u32* dst = reinterpret_cast<u32*>(s_nodes);
        for (u32 k = threadIdx.x; k < A.node_count * (u32)(sizeof(NodeDev) / 4); k += blockDim.x) dst[k] = src[k];
        src = reinterpret_cast<const u32*>(A.scalars);
        dst = reinterpret_cast<u32*>(s_scalars);
        for (u32 k = threadIdx.x; k < A.scalar_count * (u32)(sizeof(ColumnDev) / 4); k += blockDim.x) dst[k] = src[k];
        src = reinterpret_cast<const u32*>(A.strings);
        dst = reinterpret_cast<u32*>(s_strings);
        for (u32 k = threadIdx.x; k < A.string_count * (u32)(sizeof(StringDev) / 4); k += blockDim.x) dst[k] = src[k];
        for (u32 k = threadIdx.x; k < A.staged_list; k += blockDim.x) s_list[k] = A.lists[k];
        for (u32 k = threadIdx.x; k < A.staged_const; k += blockDim.x) s_const[k] = A.consts[k];
    }
    __syncthreads();

    const u32 lane = threadIdx.x & 31;
    const u64 words = (A.n + 63) / 64 * 2;  // 32-row groups, the last 64-bit word of the bitmap included
    const u64 warps = (u64)gridDim.x * (blockDim.x >> 5);
    u32 bad = 0;
    u64 selected = 0;
    for (u64 w = (u64)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w < words; w += warps) {
        const u64 row0 = w * 32;
        const u64 i = row0 + lane;
        const bool live = i < A.n;
        u32 stack = 0;
#pragma unroll 1
        for (u32 k = 0; k < A.node_count; ++k) {
            const NodeDev nd = s_nodes[k];
            u32 r;
            if (nd.op == YTGPU_FILTER_AND || nd.op == YTGPU_FILTER_OR) {
                const u32 a = stack & 3, b = (stack >> 2) & 3;
                stack >>= 4;
                r = nd.op == YTGPU_FILTER_AND ? ((a & b & 1) | ((a | b) & 2)) : (((a | b) & 1) | (a & b & 2));
            } else if (nd.op == YTGPU_FILTER_NOT) {
                const u32 a = stack & 3;
                stack >>= 2;
                r = ((a & 1) << 1) | (a >> 1);
            } else if (nd.is_string) {
                const StringDev& sc = s_strings[nd.col];
                ytgpu_value v{};
                const bool have = live && string_at(sc, i, &v, &bad);
                if (nd.op == YTGPU_FILTER_IS_NULL) r = have || !live ? kFalse : kTrue;
                else if (nd.op == YTGPU_FILTER_IS_NOT_NULL) r = have ? kTrue : kFalse;
                else if (!have) r = kNull;
                else if (nd.op == YTGPU_FILTER_COMPARE_COLUMNS) {
                    const StringDev& sc2 = s_strings[nd.col2];
                    ytgpu_value v2{};
                    r = string_at(sc2, i, &v2, &bad) ? (cmp_holds(nd.cmp, string_compare2(sc.heap, v, sc2.heap, v2)) ? kTrue : kFalse)
                                                      : kNull;
                } else if (nd.op == YTGPU_FILTER_COMPARE) {
                    ytgpu_value c{};
                    c.type = YTGPU_TYPE_STRING;
                    c.length = nd.length;
                    c.data = nd.constant;
                    r = cmp_holds(nd.cmp, string_compare2(sc.heap, v, const_heap(A, s_const, nd.constant, nd.length), c)) ? kTrue : kFalse;
                } else if (kPatterns && (nd.op == YTGPU_FILTER_CONTAINS || nd.op == YTGPU_FILTER_LIKE)) {
                    r = pattern_match(s_pat + nd.constant, sc.heap + v.data, v.length) ? kTrue : kFalse;
                } else if (nd.op == YTGPU_FILTER_STARTS_WITH) {
                    bool ok = v.length >= nd.length;
                    const u8* p = const_heap(A, s_const, nd.constant, nd.length) + nd.constant;
                    const u8* s = sc.heap + v.data;
                    for (u32 b = 0; ok && b < nd.length; ++b) ok = s[b] == p[b];
                    r = ok ? kTrue : kFalse;
                } else {  // IN: binary search over the sorted entries
                    u64 lo = nd.constant, cnt = nd.length;
                    while (cnt > 0) {
                        const u64 half = cnt >> 1, mid = lo + half;
                        const u64 e = load_list(A, s_list, mid);
                        ytgpu_value c{};
                        c.type = YTGPU_TYPE_STRING;
                        c.length = (u32)e;
                        c.data = e >> 32;
                        if (string_compare2(sc.heap, v, const_heap(A, s_const, c.data, c.length), c) > 0) {
                            lo = mid + 1;
                            cnt -= half + 1;
                        } else {
                            cnt = half;
                        }
                    }
                    r = kFalse;
                    if (lo < nd.constant + nd.length) {
                        const u64 e = load_list(A, s_list, lo);
                        ytgpu_value c{};
                        c.type = YTGPU_TYPE_STRING;
                        c.length = (u32)e;
                        c.data = e >> 32;
                        if (string_compare2(sc.heap, v, const_heap(A, s_const, c.data, c.length), c) == 0) r = kTrue;
                    }
                }
            } else {
                const ColumnDev& c = s_scalars[nd.col];
                bool nul;
                const u64 v = scalar_value(c, i, row0, live, &nul);
                if (nd.op == YTGPU_FILTER_IS_NULL) r = nul && live ? kTrue : kFalse;
                else if (nd.op == YTGPU_FILTER_IS_NOT_NULL) r = nul ? kFalse : kTrue;
                else if (nd.op == YTGPU_FILTER_COMPARE_COLUMNS) {
                    bool nul2;
                    const u64 v2 = scalar_value(s_scalars[nd.col2], i, row0, live, &nul2);
                    r = nul || nul2 ? kNull : (passes(nd.cmp, c.value_type, v, v2) ? kTrue : kFalse);
                } else if (nul) r = kNull;
                else if (nd.op == YTGPU_FILTER_COMPARE) r = passes(nd.cmp, c.value_type, v, nd.constant) ? kTrue : kFalse;
                else {  // IN: lower bound of the value's order word, then the EQ rule on the entry found
                    const u64 key = in_key(c.value_type, v);
                    u64 lo = nd.constant, cnt = nd.length;
                    while (cnt > 0) {
                        const u64 half = cnt >> 1, mid = lo + half;
                        if (load_list(A, s_list, mid) < key) {
                            lo = mid + 1;
                            cnt -= half + 1;
                        } else {
                            cnt = half;
                        }
                    }
                    r = lo < nd.constant + nd.length &&
                                passes(YTGPU_CMP_EQ, c.value_type, v, minmax_decode(c.value_type, load_list(A, s_list, lo)))
                            ? kTrue : kFalse;
                }
            }
            stack = (stack << 2) | r;
        }
        const bool sel = live && (stack & 3) == kTrue;
        const u32 m = __ballot_sync(0xffffffffu, sel);
        if (lane == 0) {
            A.bitmap[w] = m;
            if (A.word_counts) A.word_counts[w] = (u64)__popc(m);
        }
        selected += (u64)__popc(m);
        if (A.bytemap) {
            if (A.bytemap_vec && row0 + 32 <= A.n) {
                if (lane < 2) {  // 16 rows per lane: bit b of the ballot becomes byte b
                    u32 q[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const u32 b = (m >> (16 * lane + 4 * j)) & 0xF;
                        q[j] = (b & 1) | ((b & 2) << 7) | ((b & 4) << 14) | ((b & 8) << 21);
                    }
                    *reinterpret_cast<uint4*>(A.bytemap + row0 + 16 * lane) = make_uint4(q[0], q[1], q[2], q[3]);
                }
            } else if (live) {
                A.bytemap[i] = sel ? 1 : 0;
            }
        }
    }
    if (lane == 0 && selected) atomicAdd(&A.result[0], (unsigned long long)selected);
    if (bad) atomicOr(&A.result[1], (unsigned long long)DE_STRING_OUT_OF_HEAP);
}

// out_rows[scan[w] + rank of the bit] = row, for every set bit of bitmap word w.
__global__ void __launch_bounds__(kFilterThreads) filter_rows_kernel(const u32* __restrict__ bitmap, const u64* __restrict__ offsets,
                                                                     u64 words, u32* out_rows) {
    const u32 lane = threadIdx.x & 31;
    const u64 warps = (u64)gridDim.x * (blockDim.x >> 5);
    for (u64 w = (u64)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w < words; w += warps) {
        const u32 m = bitmap[w];
        if ((m >> lane) & 1) out_rows[offsets[w] + __popc(m & lanemask_lt())] = (u32)(w * 32 + lane);
    }
}

// ---- host ----
struct Checked {
    std::vector<NodeDev> nodes;
    std::vector<u64> lists;   // sorted entries of every IN node, node by node
    std::vector<u8> patterns; // compiled CONTAINS / LIKE patterns, node by node (strings.cuh)
    SlotMap scalars, strings;  // the referenced columns' compact tables
};

Status check_program(const ytgpu_column_view* columns, u32 column_count, u32 string_count, const ytgpu_filter_node* program,
                     u32 node_count, const u64* list_values, u64 list_value_count, const u8* consts, u64 const_bytes,
                     Checked* out) {
    if (node_count == 0 || node_count > (u32)YTGPU_FILTER_MAX_NODES)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "a filter program has 1 .. %d nodes", YTGPU_FILTER_MAX_NODES);
    if (!program) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null program");
    if (const_bytes > (u64)YTGPU_FILTER_MAX_STRING_CONSTANT_BYTES)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "at most %u bytes of string constants", YTGPU_FILTER_MAX_STRING_CONSTANT_BYTES);
    if (const_bytes && !consts) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null string_constants");
    if (list_value_count && !list_values) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null list_values");
    const u64 total = (u64)column_count + string_count;
    auto slot = [&](u32 c) { return c < column_count ? out->scalars.slot(c) : out->strings.slot(c - column_count); };
    auto string_range_ok = [&](u64 off, u64 len) { return off <= const_bytes && len <= const_bytes - off; };
    u64 in_entries = 0;
    int depth = 0;
    for (u32 k = 0; k < node_count; ++k) {
        const ytgpu_filter_node& N = program[k];
        NodeDev d{};
        d.op = (u8)N.op;
        const bool leaf = (N.op >= YTGPU_FILTER_COMPARE && N.op <= YTGPU_FILTER_IS_NOT_NULL) || N.op == YTGPU_FILTER_CONTAINS ||
                          N.op == YTGPU_FILTER_LIKE;
        if (!leaf && N.op != YTGPU_FILTER_AND && N.op != YTGPU_FILTER_OR && N.op != YTGPU_FILTER_NOT)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: unknown op %d", k, N.op);
        if (!leaf) {
            const int pops = N.op == YTGPU_FILTER_NOT ? 1 : 2;
            if (depth < pops) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: stack underflow", k);
            depth -= pops - 1;
            out->nodes.push_back(d);
            continue;
        }
        if (N.column < 0 || (u64)N.column >= total) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: column %d out of range", k, N.column);
        const bool str = (u32)N.column >= column_count;
        const u8 vtype = str ? (u8)YTGPU_TYPE_STRING : columns[N.column].value_type;
        if (!str && !is_scalar_type(vtype))
            return make_status(YTGPU_ERR_UNSUPPORTED, "node %u: column %d has value type 0x%x (INT64, UINT64, DOUBLE or BOOLEAN)", k,
                               N.column, vtype);
        d.is_string = str;
        d.col = slot((u32)N.column);
        if (N.op == YTGPU_FILTER_COMPARE || N.op == YTGPU_FILTER_COMPARE_COLUMNS) {
            if (N.cmp < YTGPU_CMP_LT || N.cmp > YTGPU_CMP_NE) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: unknown cmp %d", k, N.cmp);
            d.cmp = (u8)N.cmp;
        }
        switch (N.op) {
            case YTGPU_FILTER_COMPARE:
                if (str && !string_range_ok(N.constant, N.length))
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: string constant outside string_constants", k);
                if (!str && N.length) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: a string constant on a scalar column", k);
                d.constant = N.constant;
                d.length = N.length;
                break;
            case YTGPU_FILTER_STARTS_WITH:
                if (!str) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: STARTS_WITH on a scalar column", k);
                if (!string_range_ok(N.constant, N.length))
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: prefix outside string_constants", k);
                d.constant = N.constant;
                d.length = N.length;
                break;
            case YTGPU_FILTER_CONTAINS:
            case YTGPU_FILTER_LIKE: {
                const bool like = N.op == YTGPU_FILTER_LIKE;
                if (!str) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: %s on a scalar column", k, like ? "LIKE" : "CONTAINS");
                if (!string_range_ok(N.constant, N.length))
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: %s outside string_constants", k, like ? "pattern" : "needle");
                d.constant = out->patterns.size();
                YTGPU_TRY(add_pattern(k, consts + N.constant, N.length, like, like ? N.column2 : -1, &out->patterns));
                break;
            }
            case YTGPU_FILTER_COMPARE_COLUMNS: {
                if (N.column2 < 0 || (u64)N.column2 >= total)
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: column2 %d out of range", k, N.column2);
                const bool str2 = (u32)N.column2 >= column_count;
                if (str != str2 || (!str && columns[N.column2].value_type != vtype))
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: COMPARE_COLUMNS over different types", k);
                d.col2 = slot((u32)N.column2);
                break;
            }
            case YTGPU_FILTER_IN: {
                if (N.constant > list_value_count || (u64)N.length > list_value_count - N.constant)
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: IN list outside list_values", k);
                d.constant = out->lists.size();
                YTGPU_TRY(add_in_list(k, vtype, list_values + N.constant, N.length, consts, const_bytes, &in_entries, &out->lists));
                d.length = (u32)(out->lists.size() - d.constant);
                break;
            }
            default:  // IS_NULL / IS_NOT_NULL
                break;
        }
        if (++depth > YTGPU_FILTER_MAX_DEPTH)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: stack deeper than %d", k, YTGPU_FILTER_MAX_DEPTH);
        out->nodes.push_back(d);
    }
    if (depth != 1) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "the program leaves %d values on the stack, not 1", depth);
    return Status{};
}

Status evaluate_filter_impl(Context* ctx, const ytgpu_column_view* columns, u32 column_count, const ytgpu_string_column* string_columns,
                            u32 string_count, const ytgpu_filter_node* program, u32 node_count, const u64* list_values,
                            u64 list_value_count, const u8* consts, u64 const_bytes, u8* out_bitmap, u8* out_bytemap, u32* out_rows,
                            u64 rows_capacity, u64* out_selected, int out_mem) {
    u64 n;
    YTGPU_TRY(check_program_columns(columns, column_count, string_columns, string_count, out_mem, &n));
    Checked P;
    YTGPU_TRY(check_program(columns, column_count, string_count, program, node_count, list_values, list_value_count, consts, const_bytes, &P));
    if (P.scalars.cols.size() + P.strings.cols.size() > kMaxFilterColumns)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "too many columns");  // unreachable: 64 nodes reference at most 128
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    if (out_selected) *out_selected = 0;
    if (n == 0) return Status{};

    StagedProgramColumns cols;
    YTGPU_TRY(cols.stage(ctx, columns, P.scalars, string_columns, P.strings));
    // one upload: nodes | scalar views | string views | sorted lists | string constants | compiled patterns
    ProgramBlob blob;
    const size_t o_nodes = blob.add(P.nodes.data(), P.nodes.size() * sizeof(NodeDev));
    const size_t o_scal = blob.add(cols.scalars.data(), cols.scalars.size() * sizeof(ColumnDev));
    const size_t o_str = blob.add(cols.strings.data(), cols.strings.size() * sizeof(StringDev));
    const size_t o_list = blob.add(P.lists.data(), P.lists.size() * 8);
    const size_t o_const = blob.add(consts, const_bytes);
    const size_t o_pat = blob.add(P.patterns.data(), P.patterns.size());
    YTGPU_TRY(blob.upload(ctx));

    const u64 words = (n + 63) / 64 * 2;  // 32-bit bitmap words
    const bool host = out_mem == YTGPU_MEM_HOST;
    DevBuf<u32> tbitmap;
    DevBuf<u64> word_counts, scan_sums, scan_total;
    DevBuf<unsigned long long> result;
    u32* dbitmap = reinterpret_cast<u32*>(out_bitmap);
    if (!out_bitmap || host) {  // the kernel writes the bitmap even when the caller asks for none
        YTGPU_TRY(tbitmap.allocate(ctx, words));
        dbitmap = tbitmap.p;
    }
    OutBuf<u8> bytemap;
    YTGPU_TRY(bytemap.prepare(ctx, out_bytemap, n, out_mem));
    if (out_rows) YTGPU_TRY(word_counts.allocate(ctx, words));
    YTGPU_TRY(result.allocate(ctx, 2));
    YTGPU_CUDA_TRY(cudaMemsetAsync(result.p, 0, 16, ctx->stream));

    FilterArgs A{};
    A.nodes = blob.at<NodeDev>(o_nodes);
    A.node_count = (u32)P.nodes.size();
    A.scalars = blob.at<ColumnDev>(o_scal);
    A.scalar_count = (u32)cols.scalars.size();
    A.strings = blob.at<StringDev>(o_str);
    A.string_count = (u32)cols.strings.size();
    A.lists = blob.at<u64>(o_list);
    A.list_count = (u32)P.lists.size();
    A.staged_list = std::min<u32>(A.list_count, kStagedListEntries);
    A.consts = blob.at<u8>(o_const);
    A.const_bytes = (u32)const_bytes;
    A.staged_const = std::min<u32>(A.const_bytes, kStagedConstBytes);
    A.patterns = blob.at<u8>(o_pat);
    A.pattern_bytes = (u32)((P.patterns.size() + 15) & ~(size_t)15);  // staged in 16-byte units, as the blob pads them
    A.n = n;
    A.bitmap = dbitmap;
    A.bytemap = bytemap.p;
    A.word_counts = out_rows ? word_counts.p : nullptr;
    A.bytemap_vec = bytemap.p && (reinterpret_cast<uintptr_t>(bytemap.p) & 15) == 0;
    A.result = result.p;
    // shared memory in the kernel's order; every part is a multiple of 8 bytes (NodeDev 24, ColumnDev / StringDev 8-aligned)
    const bool patterns = !P.patterns.empty();
    size_t smem = P.nodes.size() * sizeof(NodeDev) + A.scalar_count * sizeof(ColumnDev) + A.string_count * sizeof(StringDev) +
                  (size_t)A.staged_list * 8 + A.staged_const;
    if (patterns) smem = pattern_smem_offset(smem) + A.pattern_bytes;
    static_assert(sizeof(ColumnDev) % 8 == 0 && sizeof(StringDev) % 8 == 0, "shared-memory layout");
    if (patterns)  // up to 32 KiB of patterns may take the stage past the 48 KB default
        YTGPU_CUDA_TRY(cudaFuncSetAttribute(filter_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const u32 blocks = blocks_for(words * 32, kFilterThreads, 8);  // a warp per 32-row group
    {
        KernelTimer t(ctx, KC_DECODE);
        if (patterns) filter_kernel<true><<<blocks, kFilterThreads, smem, ctx->stream>>>(A);
        else filter_kernel<false><<<blocks, kFilterThreads, smem, ctx->stream>>>(A);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    unsigned long long res[2] = {0, 0};  // the one host read: selected count and error bits
    YTGPU_CUDA_TRY(cudaMemcpyAsync(res, result.p, 16, cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (res[1] & DE_STRING_OUT_OF_HEAP)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "a string value of a filter column leaves its heap");
    const u64 selected = res[0];
    if (out_selected) *out_selected = selected;
    if (out_rows && selected > rows_capacity)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "%llu rows selected, rows_capacity is %llu", (unsigned long long)selected,
                           (unsigned long long)rows_capacity);

    OutBuf<u32> rows;
    if (out_rows && selected) {
        YTGPU_TRY(rows.prepare(ctx, out_rows, selected, out_mem));
        YTGPU_TRY(scan_sums.allocate(ctx, scan_block_count(words)));
        YTGPU_TRY(scan_total.allocate(ctx, 1));
        {
            KernelTimer t(ctx, KC_DECODE, 4);
            exclusive_scan_u64(ctx->stream, word_counts.p, words, scan_sums.p, scan_total.p);
            filter_rows_kernel<<<blocks, kFilterThreads, 0, ctx->stream>>>(dbitmap, word_counts.p, words, rows.p);
            YTGPU_CUDA_TRY(cudaGetLastError());
        }
        YTGPU_TRY(rows.download(ctx, selected));
    }
    if (host && out_bitmap) YTGPU_TRY(copy_out(ctx, out_bitmap, dbitmap, words * 4, YTGPU_MEM_HOST));
    YTGPU_TRY(bytemap.download(ctx, n));
    if (host) YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return Status{};
}

}  // namespace

extern "C" {

int ytgpu_evaluate_filter(ytgpu_context* h, const ytgpu_column_view* columns, uint32_t column_count,
                          const ytgpu_string_column* string_columns, uint32_t string_count, const ytgpu_filter_node* program,
                          uint32_t node_count, const uint64_t* list_values, uint64_t list_value_count,
                          const uint8_t* string_constants, uint64_t string_constant_bytes, uint8_t* out_bitmap,
                          uint8_t* out_bytemap, uint32_t* out_rows, uint64_t rows_capacity, uint64_t* out_selected, int out_mem,
                          ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, evaluate_filter_impl(as_context(h), columns, column_count, string_columns, string_count, program, node_count,
                                                list_values, list_value_count, string_constants, string_constant_bytes, out_bitmap,
                                                out_bytemap, out_rows, rows_capacity, out_selected, out_mem));
}

}  // extern "C"
