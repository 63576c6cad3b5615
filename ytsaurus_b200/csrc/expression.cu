// expression.cu — computed columns: arithmetic, bitwise, cast and if_null expressions over several columns, evaluated into a
// 64-bit value vector plus a null bitmap (ytgpu_evaluate_expression, semantics in ytgpu.h).
//
// A separate pass, like the filter: its output is a plain 64-bit column with a null bitmap, which every GROUP BY, filter and
// decode call already takes, so no aggregation or filter kernel changes.  The kernel is an interpreter of a typed postfix
// program, laid out like filter_kernel:
//   * one thread per row and 32 consecutive rows per warp: direct columns load coalesced, each lane stores its 8-byte
//     result, and the 32 NULL flags of a warp are one __ballot_sync word of the null bitmap;
//   * every lane runs the same node, so the interpreter loop does not diverge; the program and the referenced columns'
//     views are staged in shared memory once per CTA; an RLE column finds its run from a hint lane 0 finds once per 32 rows;
//   * the top of the value stack is a register, the entries below it live in shared memory as [depth][threadIdx.x] u64
//     (conflict-free, sized by the program's depth: nothing when it is at most 1 deep, 30 KB at 16); the NULL flags are
//     a bit stack in one register.  The depth at every node is the same in all lanes, so nothing goes to local memory;
//   * a 32-row group without a selected row skips the program;
//   * the NULL count and the division-error bits are reduced per warp, one atomic each.
//
// String expressions (ytgpu_evaluate_expression_strings) run the instantiation expression_kernel<true, true>.  A STRING stack
// entry is a list of pieces (pointer, length, case map): a leaf makes one piece, CONCAT appends the lists, LOWER / UPPER
// set the case map of every piece (on ASCII lower(upper(x)) = lower(x), so the outermost wins) and IF_NULL keeps one of
// them.  The pieces form a second stack in shared memory, [piece][threadIdx.x] (pointer u64, length u32); the value
// stack holds a string entry's piece count, 0 when it is NULL, and the case maps are 2 bits per piece in one register.
// So no piece is ever moved: CONCAT's operands are adjacent already and IF_NULL's NULL first operand has no pieces.  The
// piece count is bounded at check time (YTGPU_EXPR_MAX_PIECES).  A STRING result takes two passes of the same program:
//   1. kModeSize writes each row's length, NULL byte and (as the scan input) its length into starts, and checks the
//      bytes under LOWER / UPPER are ASCII;
//   2. an exclusive scan (scan.cuh) turns the lengths into starts, its total is the heap size;
//   3. kModeFill evaluates the program again and copies the pieces with their case maps, row-centric as
//      string_to_ch.cu's copy: a warp whose 32 values are short assembles them in shared memory and writes the stretch
//      with 16-byte stores; a long value is copied by the whole warp, 4 bytes per lane when aligned.
// FARM_HASH hashes its operands with farmhash.cuh's value and row combiners; a string operand is one piece.
//
// Conditional ops (COMPARE, AND, OR, NOT, IS_NULL, IS_NOT_NULL, IF) run in both instantiations.  A BOOLEAN entry holds 0 / 1
// (0 when NULL), so Kleene AND / OR are a & b / a | b plus a NULL rule.  A STRING COMPARE walks both piece lists byte by
// byte under their case maps and drops both; a STRING IF keeps a's pieces, or moves b's (at most 16) down over them.
// Errors follow the data: each entry carries its error kinds in a bit stack in registers (kEW bits per entry), every op
// ORs its operands' bits, IF takes the condition's and the taken branch's, FALSE AND x / TRUE OR x drop x's, and only the
// result's bits reach the error word.  So a program without IF / AND / OR fails on the rows it always failed on.
//
// Predicates inside expressions (IN, STARTS_WITH, CONTAINS, LIKE) run in instantiations of their own, chosen by the host
// from the checked program: expression_kernel<false, true, true> for a numeric IN without strings, <true, true, true> for
// the rest.  Programs without them launch the other three exactly as before.  The sorted IN lists (strings.cuh
// prepare_in_list, shared with the filter) and the compiled patterns (compile_pattern) travel in the one upload; the
// patterns and the head of the lists are staged in shared memory after everything else.  A STRING operand is consumed
// where its pieces lie: a single piece without a case map is matched as contiguous bytes, as the filter does, a longer
// list through PieceBytes, which walks the pieces under their case maps for the same matcher; a string IN searches
// with pieces_compare against the constant bytes.  The column checks, compact column tables, staging and upload are
// program.cuh's, shared with filter.cu; the kernel's prologue and IN search stay here, as shared helpers changed its code.
//
// TIMESTAMP_FLOOR and FORMAT_TIMESTAMP run in expression_time_kernel<false> / <true>, which also carry the conditional ops
// and the predicates: their range error takes one more error bit per entry.  FORMAT_TIMESTAMP writes its value into a
// 64-byte scratch line per thread and node, and its piece points there; lines written by this kernel must not be read
// through the read-only path, so the time instantiations read every piece with plain loads.  Their body,
// expression_time_body, and its readers are copies of the ones above rather than template parameters of them: every such
// parameter changed the code of expression_kernel<true, true>.
#include <algorithm>
#include <cstring>
#include <type_traits>
#include <vector>

#include "farmhash.cuh"
#include "program.cuh"
#include "scan.cuh"

using namespace ytgpu;

namespace {

constexpr int kExprThreads = 256;
// Errors that follow the data: a bit stack per kind beside the NULL stack, 2 bits per entry in expression_kernel<false, true>,
// 3 in expression_kernel<true, true>; only the result's bits fail the call.  expression_kernel<false, false> runs programs
// without conditional ops, where every error reaches the result, so it raises them at once.  The others are input
// checks, raised at once.
constexpr u32 kErrDivZero = 1, kErrIntMinByMinusOne = 2, kErrNonAscii = 4;
constexpr u32 kErrOutOfHeap = 8, kErrTooLong = 16;
constexpr u32 kErrMatchTooLong = 32;  // CONTAINS / LIKE over 2^32 bytes or more: the matcher counts in 32 bits
constexpr u32 kErrTimeRange = 64;     // a timestamp outside [0, 9999-12-31T23:59:59Z], or a week floor before the epoch
constexpr u32 kModeValues = 0, kModeSize = 1, kModeFill = 2;  // a 64-bit result; a STRING result's two passes
constexpr u32 kCaseLower = 1, kCaseUpper = 2;
constexpr u32 kShortValue = 48;                                        // longer values are copied by the whole warp
constexpr u32 kStageBytes = 32 * kShortValue + 16;                     // a warp's short values and the 16-byte skew

struct ExprNodeDev {
    u8 op;
    u8 type;  // the node's result type
    u8 from;  // CAST, COMPARE, IS_NULL, IS_NOT_NULL, IN: the operand's type
    u8 pad;
    u16 col;  // COLUMN: compact column table (referenced columns only; a STRING leaf: the compact string table);
              // FARM_HASH: its operand count; COMPARE: the ytgpu_cmp_op
    u16 pad2;
    u64 constant;  // CONSTANT: the bit pattern, a STRING one (offset << 32) | length; FARM_HASH: bit j = operand j is a STRING;
                   // IN: (first entry in lists << 32) | entries; STARTS_WITH: the prefix as a STRING CONSTANT;
                   // CONTAINS, LIKE: the compiled pattern's offset in patterns
};
static_assert(sizeof(ExprNodeDev) == 16, "ExprNodeDev layout");

struct ExprArgs {
    const ExprNodeDev* nodes;
    u32 node_count;
    u32 column_count;
    const ColumnDev* columns;
    const u32* selection;  // nullable: 2 * ceil(n / 64) words of 32 bits
    u64 n;
    u64* values;
    u32* nulls;                   // 2 * ceil(n / 64) words of 32 bits
    unsigned long long* result;   // [0] NULL rows, [1] error bits, [2] (STRING result) heap bytes
    // expression_kernel<true, true> only
    const StringDev* strings;
    u32 string_count;
    u32 mode;
    u32 max_depth;                // stack entries below the top: max_depth - 1
    u32 max_pieces;
    const u8* consts;             // the string constants
    u64* starts;                  // kModeSize: the lengths (the scan's input); kModeFill: the starts
    u32* lengths;
    u8* null_bytes;
    u8* heap;
};

// expression_pred_kernel only.  A parameter of its own: ExprArgs grown past 128 bytes changed how the compiler reads it,
// and with that the code of the other kernels.
struct PredArgs {
    const u64* lists;             // the sorted IN entries (strings.cuh prepare_in_list), node by node
    const u8* patterns;           // the compiled CONTAINS / LIKE patterns, node by node
    u32 staged_list;              // entries of lists staged in shared memory
    u32 pattern_bytes;            // a multiple of 16, all staged
    u32 pred_smem;                // the shared-memory offset (16-aligned) of the staged patterns, then the staged entries
};

__device__ __forceinline__ double as_double(u64 x) { return __longlong_as_double((long long)x); }
__device__ __forceinline__ u64 double_bits(double x) { return (u64)__double_as_longlong(x); }

// Both operands are non-NULL and have the node's type.
__device__ __forceinline__ u64 binary_op(u32 op, u32 type, u64 a, u64 b, u32* err) {
    const bool dbl = type == YTGPU_TYPE_DOUBLE;
    switch (op) {
        case YTGPU_EXPR_ADD: return dbl ? double_bits(__dadd_rn(as_double(a), as_double(b))) : a + b;
        case YTGPU_EXPR_SUB: return dbl ? double_bits(__dsub_rn(as_double(a), as_double(b))) : a - b;
        case YTGPU_EXPR_MUL: return dbl ? double_bits(__dmul_rn(as_double(a), as_double(b))) : a * b;
        case YTGPU_EXPR_DIV:
        case YTGPU_EXPR_MOD: {
            if (dbl) return double_bits(__ddiv_rn(as_double(a), as_double(b)));  // MOD takes no doubles
            if (b == 0) {
                *err |= kErrDivZero;
                return 0;
            }
            if (type == YTGPU_TYPE_INT64) {
                if (a == 0x8000000000000000ull && b == ~0ull) {
                    *err |= kErrIntMinByMinusOne;
                    return 0;
                }
                return op == YTGPU_EXPR_DIV ? (u64)((i64)a / (i64)b) : (u64)((i64)a % (i64)b);
            }
            return op == YTGPU_EXPR_DIV ? a / b : a % b;
        }
        case YTGPU_EXPR_BIT_AND: return a & b;
        case YTGPU_EXPR_BIT_OR: return a | b;
        default: return a ^ b;  // BIT_XOR
    }
}

// The operand is non-NULL.  BOOLEAN values are 0 / 1 already.
__device__ __forceinline__ u64 unary_op(u32 op, u32 type, u32 from, u64 a) {
    if (op == YTGPU_EXPR_NEG) return type == YTGPU_TYPE_DOUBLE ? a ^ 0x8000000000000000ull : 0 - a;
    if (op == YTGPU_EXPR_BIT_NOT) return ~a;
    if (from == type) return a;  // CAST
    if (type == YTGPU_TYPE_DOUBLE) {
        if (from == YTGPU_TYPE_INT64) return double_bits(__ll2double_rn((long long)a));
        if (from == YTGPU_TYPE_UINT64) return double_bits(__ull2double_rn(a));
        return double_bits(a ? 1.0 : 0.0);
    }
    if (from == YTGPU_TYPE_DOUBLE) {  // cvt.rzi: truncation, saturating; NaN -> 0 (cvt.rzi.s64.f64 gives INT64_MIN for it)
        const double x = as_double(a);
        if (x != x) return 0;
        return type == YTGPU_TYPE_INT64 ? (u64)__double2ll_rz(x) : (u64)__double2ull_rz(x);
    }
    return a;  // INT64 <-> UINT64, BOOLEAN -> integer
}

// A byte under a case map; ASCII letters only (a mapped piece holds ASCII bytes, checked in kModeSize).
__device__ __forceinline__ u32 case_byte(u32 b, u32 cm) {
    if (cm == kCaseLower) return b - 'A' < 26u ? b + 32 : b;
    if (cm == kCaseUpper) return b - 'a' < 26u ? b - 32 : b;
    return b;
}

// Four ASCII bytes at once: bit 7 of a byte of (w + 0x3f..) is set iff the byte is >= 'A', of (w + 0x25..) iff > 'Z'; no
// carry crosses a byte while every byte is below 0x80.
__device__ __forceinline__ u32 case_word(u32 w, u32 cm) {
    if (cm == kCaseLower) return w ^ ((((w + 0x3f3f3f3fu) & ~(w + 0x25252525u)) & 0x80808080u) >> 2);
    if (cm == kCaseUpper) return w ^ ((((w + 0x1f1f1f1fu) & ~(w + 0x05050505u)) & 0x80808080u) >> 2);
    return w;
}

__device__ __forceinline__ bool ascii_only(const u8* p, u32 len) {
    const u32 head = min(len, (u32)((8 - (reinterpret_cast<uintptr_t>(p) & 7)) & 7));
    u32 acc = 0, j = 0;
    for (; j < head; ++j) acc |= __ldg(p + j);
    for (; j + 8 <= len; j += 8)
        if (__ldg(reinterpret_cast<const unsigned long long*>(p + j)) & 0x8080808080808080ull) return false;
    for (; j < len; ++j) acc |= __ldg(p + j);
    return (acc & 0x80) == 0;
}

// The whole warp copies len bytes: bytes up to the destination's 4-byte boundary, then 4 bytes per lane when the source
// is aligned there too (else 1), then the tail — string_to_ch.cu's long-value copy, with the case map applied.
__device__ __forceinline__ void warp_copy(u8* dst, const u8* src, u64 len, u32 cm, u32 lane) {
    const u32 head = (u32)min(len, (u64)((4 - (reinterpret_cast<uintptr_t>(dst) & 3)) & 3));
    for (u32 j = lane; j < head; j += 32) dst[j] = (u8)case_byte(__ldg(src + j), cm);
    const u64 body = (len - head) & ~3ull;
    if (((reinterpret_cast<uintptr_t>(src) + head) & 3) == 0) {
        const u32* s4 = reinterpret_cast<const u32*>(src + head);
        u32* d4 = reinterpret_cast<u32*>(dst + head);
        for (u64 w = lane; w < body / 4; w += 32) d4[w] = case_word(__ldg(s4 + w), cm);
    } else {
        for (u64 j = lane; j < body; j += 32) dst[head + j] = (u8)case_byte(__ldg(src + head + j), cm);
    }
    for (u64 j = head + body + lane; j < len; j += 32) dst[j] = (u8)case_byte(__ldg(src + j), cm);
}

// A STRING COMPARE: the pieces [a, a + na) against [b, b + nb) of this thread's piece stack (pptr / plen: its entry 0,
// stride kExprThreads), byte by byte under their case maps: unsigned bytes, then the shorter value first.  With nb = 0 the
// right-hand side is the lb contiguous bytes at pb instead (a constant).
__device__ __forceinline__ int pieces_compare(const u64* pptr, const u32* plen, u32 cases, u32 a, u32 na, u32 b, u32 nb,
                                              const u8* pb = nullptr, u32 lb = 0) {
    const u32 ea = a + na, eb = b + nb;
    const u8* pa = nullptr;
    u32 la = 0, ca = 0, cb = 0;  // bytes left in the current pieces (lb: on the right), their case maps
    for (;;) {
        while (la == 0 && a < ea) {
            pa = reinterpret_cast<const u8*>(pptr[a * kExprThreads]);
            la = plen[a * kExprThreads];
            ca = (cases >> (2 * a)) & 3;
            ++a;
        }
        while (lb == 0 && b < eb) {
            pb = reinterpret_cast<const u8*>(pptr[b * kExprThreads]);
            lb = plen[b * kExprThreads];
            cb = (cases >> (2 * b)) & 3;
            ++b;
        }
        if (la == 0 || lb == 0) return (la != 0) - (lb != 0);
        const u32 x = case_byte(__ldg(pa), ca), y = case_byte(__ldg(pb), cb);
        if (x != y) return x < y ? -1 : 1;
        ++pa, ++pb, --la, --lb;
    }
}

// The bytes of the pieces p, p + 1, ... of this thread's piece stack under their case maps, in order: pattern_match's byte
// source.  The caller asks for no more bytes than the pieces hold.
struct PieceBytes {
    const u64* pptr;
    const u32* plen;
    u32 cases;
    u32 p;
    const u8* cur = nullptr;
    u32 left = 0, cm = 0;
    __device__ __forceinline__ u32 operator()(u32) {
        while (left == 0) {
            cur = reinterpret_cast<const u8*>(pptr[p * kExprThreads]);
            left = plen[p * kExprThreads];
            cm = (cases >> (2 * p)) & 3;
            ++p;
        }
        --left;
        return case_byte(__ldg(cur++), cm);
    }
};

// kCond: the program may hold COMPARE, AND, OR, NOT, IS_NULL, IS_NOT_NULL or IF.  Without them the scalar instantiation
// keeps the dispatch and the error handling of a program of arithmetic only (the conditional ops cost the old programs
// 6-14 % in bench_expressions.py when compiled in); the string one always takes them.  kPred: the program may hold IN,
// STARTS_WITH, CONTAINS or LIKE (the string ones with kStrings only), so the other instantiations do not carry them.
template <bool kStrings, bool kCond, bool kPred>
__device__ __forceinline__ void expression_body(const ExprArgs& A, const PredArgs& Q) {
    static_assert(kCond || !kStrings, "expression_kernel<true, false> is not instantiated");
    static_assert(kCond || !kPred, "the predicates are conditional ops");
    // the error bit stacks: kEW bits per entry, entry d from the top at bit kEW * d (a 16-deep stack fills 32 / 48 bits)
    using ErrStack = typename std::conditional<kStrings, u64, u32>::type;
    constexpr u32 kEW = kStrings ? 3 : 2;
    constexpr ErrStack kEM = (ErrStack)((1u << kEW) - 1);
    extern __shared__ __align__(16) unsigned char smem[];
    ExprNodeDev* s_nodes = reinterpret_cast<ExprNodeDev*>(smem);
    ColumnDev* s_cols = reinterpret_cast<ColumnDev*>(s_nodes + A.node_count);
    StringDev* s_strs = reinterpret_cast<StringDev*>(s_cols + A.column_count);
    u64* s_stack = reinterpret_cast<u64*>(s_strs + (kStrings ? A.string_count : 0)) + threadIdx.x;  // entry d: [d * kExprThreads]
    // expression_kernel<true, true>: the piece stack [p * kExprThreads], then a short-value stage per warp
    u64* s_pptr = s_stack + (kStrings ? (size_t)(A.max_depth - 1) * kExprThreads : 0);
    u32* s_plen = reinterpret_cast<u32*>(s_pptr - threadIdx.x + (size_t)A.max_pieces * kExprThreads) + threadIdx.x;
    u8* s_stage = reinterpret_cast<u8*>((reinterpret_cast<uintptr_t>(s_plen - threadIdx.x + (size_t)A.max_pieces * kExprThreads) + 15) & ~(uintptr_t)15) +
                  (threadIdx.x >> 5) * kStageBytes;
    {
        const u32* src = reinterpret_cast<const u32*>(A.nodes);
        u32* dst = reinterpret_cast<u32*>(s_nodes);
        for (u32 k = threadIdx.x; k < A.node_count * (u32)(sizeof(ExprNodeDev) / 4); k += blockDim.x) dst[k] = src[k];
        src = reinterpret_cast<const u32*>(A.columns);
        dst = reinterpret_cast<u32*>(s_cols);
        for (u32 k = threadIdx.x; k < A.column_count * (u32)(sizeof(ColumnDev) / 4); k += blockDim.x) dst[k] = src[k];
        if constexpr (kStrings) {
            src = reinterpret_cast<const u32*>(A.strings);
            dst = reinterpret_cast<u32*>(s_strs);
            for (u32 k = threadIdx.x; k < A.string_count * (u32)(sizeof(StringDev) / 4); k += blockDim.x) dst[k] = src[k];
        }
    }
    const u8* s_pat = nullptr;
    const u64* s_list = nullptr;
    if constexpr (kPred) {
        uint4* pat = reinterpret_cast<uint4*>(smem + Q.pred_smem);
        const uint4* psrc = reinterpret_cast<const uint4*>(Q.patterns);
        for (u32 k = threadIdx.x; k < Q.pattern_bytes / 16; k += blockDim.x) pat[k] = psrc[k];
        u64* list = reinterpret_cast<u64*>(smem + Q.pred_smem + Q.pattern_bytes);
        for (u32 k = threadIdx.x; k < Q.staged_list; k += blockDim.x) list[k] = Q.lists[k];
        s_pat = smem + Q.pred_smem;
        s_list = list;
    }
    __syncthreads();

    const u32 lane = threadIdx.x & 31;
    const u64 words = (A.n + 63) / 64 * 2;  // 32-row groups, the last 64-bit word of the bitmap included
    const u64 warps = (u64)gridDim.x * (blockDim.x >> 5);
    u32 err = 0;
    u64 null_rows = 0;
    for (u64 w = (u64)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w < words; w += warps) {
        const u64 row0 = w * 32;
        const u64 i = row0 + lane;
        const u32 sel = A.selection ? A.selection[w] : ~0u;
        const bool live = i < A.n && ((sel >> lane) & 1);
        u64 top = 0;
        u32 nul_stack = 1;  // bit d: entry d from the top is NULL
        u32 np = 0;         // pieces on the piece stack
        u32 cases = 0;      // 2 bits per piece: its case map
        ErrStack es = 0;    // the entries' error bits
        if (sel != 0) {
            u32 depth = 0;  // entries below the top, in s_stack
#pragma unroll 1
            for (u32 k = 0; k < A.node_count; ++k) {
                const ExprNodeDev nd = s_nodes[k];
                if (nd.op == YTGPU_EXPR_COLUMN || nd.op == YTGPU_EXPR_CONSTANT) {
                    bool nul = !live;
                    u64 v = nd.constant;
                    if (kStrings && nd.type == YTGPU_TYPE_STRING) {
                        const u8* p = A.consts + (nd.constant >> 32);
                        u32 len = (u32)nd.constant;
                        if (nd.op == YTGPU_EXPR_COLUMN && !nul) {
                            const StringDev& sc = s_strs[nd.col];
                            ytgpu_value sv;
                            u32 bad = 0;
                            nul = !string_at(sc, i, &sv, &bad);
                            if (bad) err |= kErrOutOfHeap;
                            p = sc.heap + sv.data;
                            len = sv.length;
                        }
                        v = 0;
                        if (!nul) {  // one piece
                            s_pptr[np * kExprThreads] = reinterpret_cast<u64>(p);
                            s_plen[np * kExprThreads] = len;
                            cases &= ~(3u << (2 * np));
                            ++np;
                            v = 1;
                        }
                    } else if (nd.op == YTGPU_EXPR_COLUMN) {
                        const ColumnDev& c = s_cols[nd.col];
                        v = scalar_value(c, i, row0, live, &nul);
                        if (c.value_type == YTGPU_TYPE_BOOLEAN) v = v != 0;
                    }
                    if (k) s_stack[depth++ * kExprThreads] = top;
                    top = nul ? 0 : v;
                    nul_stack = (nul_stack << 1) | (nul ? 1u : 0u);
                    if (kCond) es <<= kEW;
                } else if (nd.op == YTGPU_EXPR_NEG || nd.op == YTGPU_EXPR_BIT_NOT || nd.op == YTGPU_EXPR_CAST) {
                    if (!(nul_stack & 1)) top = unary_op(nd.op, nd.type, nd.from, top);
                } else if (kCond && nd.op == YTGPU_EXPR_NOT) {
                    top ^= (nul_stack & 1) ^ 1;  // a NULL entry holds 0 and stays NULL
                } else if (kCond && (nd.op == YTGPU_EXPR_IS_NULL || nd.op == YTGPU_EXPR_IS_NOT_NULL)) {
                    if (kStrings && nd.from == YTGPU_TYPE_STRING) np -= (u32)top;  // a NULL string has no pieces
                    top = (nul_stack & 1) ^ (nd.op == YTGPU_EXPR_IS_NULL ? 0u : 1u);
                    nul_stack &= ~1u;
                } else if (kPred && nd.op == YTGPU_EXPR_IN) {
                    // lower bound over the sorted entries, then equality on the entry found (a number: the EQ rule)
                    const u32 first = (u32)(nd.constant >> 32), end = first + (u32)nd.constant;
                    const bool str = kStrings && nd.from == YTGPU_TYPE_STRING;
                    const u32 p0 = np - (str ? (u32)top : 0u);
                    bool r = false;
                    if (!(nul_stack & 1)) {
                        const u64 key = str ? 0 : in_key(nd.from, top);
                        u32 lo = first, cnt = end - first;
                        int c = 1;
                        while (cnt > 0) {
                            const u32 half = cnt >> 1, mid = lo + half;
                            const u64 e = mid < Q.staged_list ? s_list[mid] : __ldg(Q.lists + mid);
                            const bool below = str ? pieces_compare(s_pptr, s_plen, cases, p0, (u32)top, 0, 0, A.consts + (e >> 32), (u32)e) > 0
                                                   : e < key;
                            if (below) {
                                lo = mid + 1;
                                cnt -= half + 1;
                            } else {
                                cnt = half;
                            }
                        }
                        if (lo < end) {
                            const u64 e = lo < Q.staged_list ? s_list[lo] : __ldg(Q.lists + lo);
                            if (str) c = pieces_compare(s_pptr, s_plen, cases, p0, (u32)top, 0, 0, A.consts + (e >> 32), (u32)e);
                            r = str ? c == 0 : passes(YTGPU_CMP_EQ, nd.from, top, minmax_decode(nd.from, e));
                        }
                    }
                    np = p0;  // a STRING operand's pieces are dropped
                    top = r ? 1 : 0;
                } else if (kStrings && kPred && (nd.op == YTGPU_EXPR_STARTS_WITH || nd.op == YTGPU_EXPR_CONTAINS || nd.op == YTGPU_EXPR_LIKE)) {
                    const u32 p0 = np - (u32)top;
                    bool r = false;
                    if (!(nul_stack & 1)) {
                        u64 len = 0;
                        for (u32 p = p0; p < np; ++p) len += s_plen[p * kExprThreads];
                        PieceBytes src{s_pptr, s_plen, cases, p0};
                        if (nd.op == YTGPU_EXPR_STARTS_WITH) {
                            const u8* q = A.consts + (nd.constant >> 32);
                            const u32 ql = (u32)nd.constant;
                            r = len >= ql;
                            for (u32 j = 0; r && j < ql; ++j) r = src(j) == __ldg(q + j);
                        } else if (len > 0xffffffffull) {
                            err |= kErrMatchTooLong;
                        } else if (top == 1 && ((cases >> (2 * p0)) & 3) == 0) {  // one piece as it is: the filter's contiguous scan
                            r = pattern_match(s_pat + nd.constant, reinterpret_cast<const u8*>(s_pptr[p0 * kExprThreads]), (u32)len);
                        } else {
                            r = pattern_match(s_pat + nd.constant, src, (u32)len);
                        }
                    }
                    np = p0;
                    top = r ? 1 : 0;
                } else if (kStrings && (nd.op == YTGPU_EXPR_LOWER || nd.op == YTGPU_EXPR_UPPER)) {
                    if (!(nul_stack & 1)) {
                        const u32 first = np - (u32)top;
                        if (A.mode != kModeFill)  // the fill pass runs only once the size pass found no error
                            for (u32 p = first; p < np; ++p)
                                if (!ascii_only(reinterpret_cast<const u8*>(s_pptr[p * kExprThreads]), s_plen[p * kExprThreads]))
                                    es |= kErrNonAscii;
                        const u32 mask = (u32)(((1ull << (2 * np)) - 1) & ~((1ull << (2 * first)) - 1));
                        cases = (cases & ~mask) | ((nd.op == YTGPU_EXPR_LOWER ? 0x55555555u : 0xaaaaaaaau) & mask);
                    }
                } else if (kStrings && nd.op == YTGPU_EXPR_FARM_HASH) {
                    // GetFarmFingerprint over the operands, deepest first; a NULL operand (a numeric one holds 0) hashes as
                    // fingerprint_u64(0), a string one is a single piece
                    const u32 count = nd.col, strs = (u32)nd.constant, below = depth - (count - 1);
                    u32 sp = 0;
                    for (u32 j = 0; j < count; ++j)
                        if ((strs >> j) & 1) sp += (u32)(j + 1 == count ? top : s_stack[(below + j) * kExprThreads]);
                    u32 p = np - sp;
                    u64 h = 0xdeadc0deULL;
                    for (u32 j = 0; j < count; ++j) {
                        const u64 v = j + 1 == count ? top : s_stack[(below + j) * kExprThreads];
                        u64 f;
                        if (((strs >> j) & 1) && v) {
                            f = fh::fingerprint_bytes(reinterpret_cast<const u8*>(s_pptr[p * kExprThreads]), s_plen[p * kExprThreads]);
                            ++p;
                        } else {
                            f = fh::fingerprint_u64((strs >> j) & 1 ? 0 : v);
                        }
                        h = fh::fingerprint_u128(h, f);
                    }
                    np -= sp;
                    depth = below;
                    top = h ^ (u64)count;
                    nul_stack = (nul_stack >> count) << 1;
                    ErrStack er = 0;
                    for (u32 j = 0; j < count; ++j) er |= (es >> (kEW * j)) & kEM;
                    es = ((es >> (kEW * count)) << kEW) | er;
                } else if (kCond && nd.op == YTGPU_EXPR_IF) {
                    // c a b IF: the value, NULL flag and error bits of the branch c takes; a NULL c takes neither
                    const u64 b = top, a = s_stack[(depth - 1) * kExprThreads], c = s_stack[(depth - 2) * kExprThreads];
                    depth -= 2;
                    const u32 nb = nul_stack & 1, na = (nul_stack >> 1) & 1, nc = (nul_stack >> 2) & 1;
                    if (kStrings && nd.type == YTGPU_TYPE_STRING) {  // a's pieces, then b's, on top of the piece stack
                        const u32 first = np - (u32)(a + b);
                        if (nc) {
                            np = first;
                        } else if (c) {
                            np -= (u32)b;
                        } else {  // b's pieces move down over a's, at most YTGPU_EXPR_MAX_PIECES of them
                            for (u32 p = 0; p < (u32)b; ++p) {
                                s_pptr[(first + p) * kExprThreads] = s_pptr[(first + (u32)a + p) * kExprThreads];
                                s_plen[(first + p) * kExprThreads] = s_plen[(first + (u32)a + p) * kExprThreads];
                            }
                            const u64 bc = ((u64)cases >> (2 * (first + (u32)a))) & ((1ull << (2 * (u32)b)) - 1);
                            cases = (u32)(((u64)cases & ((1ull << (2 * first)) - 1)) | (bc << (2 * first)));
                            np = first + (u32)b;
                        }
                    }
                    top = c ? a : b;  // a NULL c holds 0: b, which nc makes NULL below
                    const u32 nr = nc | (c ? na : nb);
                    top = nr ? 0 : top;
                    nul_stack = ((nul_stack >> 3) << 1) | nr;
                    const ErrStack er = ((es >> (2 * kEW)) & kEM) | (nc ? 0 : (es >> (c ? kEW : 0)) & kEM);
                    es = ((es >> (3 * kEW)) << kEW) | er;
                } else {
                    const u64 a = s_stack[--depth * kExprThreads], b = top;
                    const u32 nb = nul_stack & 1, na = (nul_stack >> 1) & 1;
                    ErrStack er = (es | (es >> kEW)) & kEM;  // both operands' bits
                    u32 nr;
                    if (nd.op == YTGPU_EXPR_IF_NULL) {
                        top = na ? b : a;
                        nr = na & nb;
                        if (kStrings && nd.type == YTGPU_TYPE_STRING && !na) np -= (u32)b;  // a NULL first operand has no pieces
                    } else if (kStrings && nd.op == YTGPU_EXPR_CONCAT) {
                        nr = na | nb;
                        np -= nr ? (u32)(a + b) : 0;
                        top = nr ? 0 : a + b;
                    } else if (kCond && nd.op == YTGPU_EXPR_COMPARE) {
                        nr = na | nb;
                        bool r;
                        if (kStrings && nd.from == YTGPU_TYPE_STRING) {  // both operands' pieces are dropped
                            np -= (u32)(a + b);
                            r = !nr && cmp_holds(nd.col, pieces_compare(s_pptr, s_plen, cases, np, (u32)a, np + (u32)a, (u32)b));
                        } else {
                            r = !nr && passes(nd.col, nd.from, a, b);
                        }
                        top = r ? 1 : 0;
                    } else if (kCond && (nd.op == YTGPU_EXPR_AND || nd.op == YTGPU_EXPR_OR)) {
                        // Kleene over 0 / 1 entries (a NULL one holds 0): F AND x = F, T OR x = T, else NULL with a NULL
                        // operand.  A deciding left operand drops the right one's error bits.
                        const bool is_and = nd.op == YTGPU_EXPR_AND;
                        const bool left_decides = is_and ? (!na && !a) : (a != 0);
                        const bool decided = left_decides || (is_and ? (!nb && !b) : (b != 0));
                        top = is_and ? (a & b) : (a | b);
                        nr = !decided && (na | nb);
                        if (left_decides) er = (es >> kEW) & kEM;
                    } else {
                        nr = na | nb;
                        u32 e = 0;
                        top = nr ? 0 : binary_op(nd.op, nd.type, a, b, kCond ? &e : &err);
                        if (kCond) er |= e;
                    }
                    nul_stack = ((nul_stack >> 2) << 1) | nr;
                    if (kCond) es = ((es >> (2 * kEW)) << kEW) | er;
                }
            }
        }
        if (kCond) err |= (u32)(es & kEM);  // the result's error bits
        const bool nul = !live || (nul_stack & 1);
        if (!kStrings || A.mode == kModeValues) {
            const u32 m = __ballot_sync(0xffffffffu, nul && i < A.n);
            if (i < A.n) A.values[i] = nul ? 0 : top;
            if (lane == 0) {
                A.nulls[w] = m;
                null_rows += (u64)__popc(m);
            }
            continue;
        }
        if constexpr (kStrings) {
            u64 len = 0;
            if (!nul)
                for (u32 p = 0; p < np; ++p) len += s_plen[p * kExprThreads];
            if (A.mode == kModeSize) {
                if (len > 0xffffffffull) {
                    err |= kErrTooLong;
                    len = 0;
                }
                const u32 m = __ballot_sync(0xffffffffu, nul && i < A.n);
                if (i < A.n) {
                    A.starts[i] = len;
                    A.lengths[i] = (u32)len;
                    A.null_bytes[i] = nul ? 1 : 0;
                }
                if (lane == 0) null_rows += (u64)__popc(m);
                continue;
            }
            // kModeFill
            if (row0 >= A.n) continue;  // a group past the last row (the bitmap's last word); warp-uniform
            const u64 pos = i < A.n ? A.starts[i] : 0;
            const bool is_long = len > kShortValue;
            u32 todo = __ballot_sync(0xffffffffu, is_long);
            if (todo == 0) {
                // every value of the group is short: the group's output [p0, p1) is one stretch, assembled in the warp's stage
                // from its 16-byte boundary below heap + p0 and written out with 16-byte stores
                const u64 p0 = __shfl_sync(0xffffffffu, pos, 0);
                u64 p1 = i < A.n ? pos + len : p0;
#pragma unroll
                for (int d = 16; d > 0; d >>= 1) p1 = max(p1, __shfl_xor_sync(0xffffffffu, p1, d));
                const u32 skew = (u32)(reinterpret_cast<uintptr_t>(A.heap + p0) & 15);
                u8* dst = s_stage + skew + (u32)(pos - p0);
                if (len)
                    for (u32 p = 0; p < np; ++p) {
                        const u8* src = reinterpret_cast<const u8*>(s_pptr[p * kExprThreads]);
                        const u32 l = s_plen[p * kExprThreads], cm = (cases >> (2 * p)) & 3;
                        for (u32 j = 0; j < l; ++j) dst[j] = (u8)case_byte(__ldg(src + j), cm);
                        dst += l;
                    }
                __syncwarp();
                const u32 begin = skew, end = skew + (u32)(p1 - p0);
                u8* gbase = A.heap + p0 - skew;  // 16-byte aligned
                for (u32 q = lane; q * 16 < end; q += 32) {
                    const u32 lo = q * 16, hi = lo + 16;
                    if (lo >= begin && hi <= end) {
                        reinterpret_cast<uint4*>(gbase)[q] = reinterpret_cast<const uint4*>(s_stage)[q];
                    } else {
                        for (u32 b = max(lo, begin); b < min(hi, end); ++b) gbase[b] = s_stage[b];
                    }
                }
                __syncwarp();  // the stage is reused by the next group
                continue;
            }
            if (!is_long && len) {
                u8* dst = A.heap + pos;
                for (u32 p = 0; p < np; ++p) {
                    const u8* src = reinterpret_cast<const u8*>(s_pptr[p * kExprThreads]);
                    const u32 l = s_plen[p * kExprThreads], cm = (cases >> (2 * p)) & 3;
                    for (u32 j = 0; j < l; ++j) dst[j] = (u8)case_byte(__ldg(src + j), cm);
                    dst += l;
                }
            }
            __syncwarp();  // the owners' piece stacks, written while the program ran, are read by the whole warp
            while (todo) {  // long values, one at a time by the whole warp, piece by piece from the owner's piece stack
                const int l = __ffs(todo) - 1;
                todo &= todo - 1;
                const u32 owner = (threadIdx.x & ~31u) + (u32)l;
                const u32 lnp = __shfl_sync(0xffffffffu, np, l), lcases = __shfl_sync(0xffffffffu, cases, l);
                u8* dst = A.heap + __shfl_sync(0xffffffffu, pos, l);
                for (u32 p = 0; p < lnp; ++p) {
                    const u8* src = reinterpret_cast<const u8*>(s_pptr[p * kExprThreads - threadIdx.x + owner]);
                    const u32 pl = s_plen[p * kExprThreads - threadIdx.x + owner];
                    warp_copy(dst, src, pl, (lcases >> (2 * p)) & 3, lane);
                    dst += pl;
                }
            }
            __syncwarp();  // ... and are overwritten by the next group's program
        }
    }
    err = __reduce_or_sync(0xffffffffu, err);
    if (lane == 0) {
        if (null_rows) atomicAdd(&A.result[0], (unsigned long long)null_rows);
        if (err) atomicOr(&A.result[1], (unsigned long long)err);
    }
}

template <bool kStrings, bool kCond>
__global__ void __launch_bounds__(kExprThreads) expression_kernel(const ExprArgs A) {
    expression_body<kStrings, kCond, false>(A, PredArgs{});
}

// Programs with IN, STARTS_WITH, CONTAINS or LIKE.  Left to itself ptxas keeps this kernel at the others' 32 / 64 registers
// and spills; with this budget it has no stack frame and no spills.
template <bool kStrings>
__global__ void __launch_bounds__(kExprThreads) __maxnreg__(kStrings ? 80 : 40) expression_pred_kernel(const ExprArgs A, const PredArgs Q) {
    expression_body<kStrings, true, true>(A, Q);
}

// The piece readers above with plain loads, for expression_time_body: a piece may point at a line FORMAT_TIMESTAMP wrote
// in the same kernel, which the non-coherent read-only path must not read.
__device__ __forceinline__ bool ascii_only_plain(const u8* p, u32 len) {
    const u32 head = min(len, (u32)((8 - (reinterpret_cast<uintptr_t>(p) & 7)) & 7));
    u32 acc = 0, j = 0;
    for (; j < head; ++j) acc |= *(p + j);
    for (; j + 8 <= len; j += 8)
        if (*(reinterpret_cast<const unsigned long long*>(p + j)) & 0x8080808080808080ull) return false;
    for (; j < len; ++j) acc |= *(p + j);
    return (acc & 0x80) == 0;
}

__device__ __forceinline__ void warp_copy_plain(u8* dst, const u8* src, u64 len, u32 cm, u32 lane) {
    const u32 head = (u32)min(len, (u64)((4 - (reinterpret_cast<uintptr_t>(dst) & 3)) & 3));
    for (u32 j = lane; j < head; j += 32) dst[j] = (u8)case_byte(*(src + j), cm);
    const u64 body = (len - head) & ~3ull;
    if (((reinterpret_cast<uintptr_t>(src) + head) & 3) == 0) {
        const u32* s4 = reinterpret_cast<const u32*>(src + head);
        u32* d4 = reinterpret_cast<u32*>(dst + head);
        for (u64 w = lane; w < body / 4; w += 32) d4[w] = case_word(*(s4 + w), cm);
    } else {
        for (u64 j = lane; j < body; j += 32) dst[head + j] = (u8)case_byte(*(src + head + j), cm);
    }
    for (u64 j = head + body + lane; j < len; j += 32) dst[j] = (u8)case_byte(*(src + j), cm);
}

__device__ __forceinline__ int pieces_compare_plain(const u64* pptr, const u32* plen, u32 cases, u32 a, u32 na, u32 b, u32 nb,
                                              const u8* pb = nullptr, u32 lb = 0) {
    const u32 ea = a + na, eb = b + nb;
    const u8* pa = nullptr;
    u32 la = 0, ca = 0, cb = 0;  // bytes left in the current pieces (lb: on the right), their case maps
    for (;;) {
        while (la == 0 && a < ea) {
            pa = reinterpret_cast<const u8*>(pptr[a * kExprThreads]);
            la = plen[a * kExprThreads];
            ca = (cases >> (2 * a)) & 3;
            ++a;
        }
        while (lb == 0 && b < eb) {
            pb = reinterpret_cast<const u8*>(pptr[b * kExprThreads]);
            lb = plen[b * kExprThreads];
            cb = (cases >> (2 * b)) & 3;
            ++b;
        }
        if (la == 0 || lb == 0) return (la != 0) - (lb != 0);
        const u32 x = case_byte(*(pa), ca), y = case_byte(*(pb), cb);
        if (x != y) return x < y ? -1 : 1;
        ++pa, ++pb, --la, --lb;
    }
}

struct PieceBytesPlain {
    const u64* pptr;
    const u32* plen;
    u32 cases;
    u32 p;
    const u8* cur = nullptr;
    u32 left = 0, cm = 0;
    __device__ __forceinline__ u32 operator()(u32) {
        while (left == 0) {
            cur = reinterpret_cast<const u8*>(pptr[p * kExprThreads]);
            left = plen[p * kExprThreads];
            cm = (cases >> (2 * p)) & 3;
            ++p;
        }
        --left;
        return case_byte(*(cur++), cm);
    }
};

// ---- TIMESTAMP_FLOOR and FORMAT_TIMESTAMP (semantics in ytgpu.h) ----
constexpr u64 kMaxTimestamp = 253402300799ull;  // 9999-12-31T23:59:59Z
constexpr u32 kFormatLine = YTGPU_EXPR_MAX_FORMATTED_BYTES;  // a FORMAT_TIMESTAMP value's scratch line per thread

// The proleptic Gregorian date of day z since 1970-01-01 (z <= 2932896, the last day of 9999): Hinnant's days-to-civil
// with an unsigned era, every division by a constant.  yday counts from January 1 (0-based).
struct Civil {
    u32 y, m, d, yday;
};
__host__ __device__ __forceinline__ Civil civil_from_days(u32 z) {
    z += 719468;
    const u32 era = z / 146097, doe = z - era * 146097;
    const u32 yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
    const u32 doy = doe - (365 * yoe + yoe / 4 - yoe / 100);  // from March 1
    const u32 mp = (5 * doy + 2) / 153;
    Civil c;
    c.d = doy - (153 * mp + 2) / 5 + 1;
    c.m = mp < 10 ? mp + 3 : mp - 9;
    c.y = yoe + era * 400 + (c.m <= 2);
    const u32 leap = (c.y % 4 == 0 && c.y % 100 != 0) || c.y % 400 == 0;
    c.yday = mp < 10 ? doy + 59 + leap : doy - 306;
    return c;
}

// unit 0..4: hour, day, week (from Monday), month, year.  *bad: t outside [0, kMaxTimestamp] as unsigned, or a week
// before 1970-01-05 (its Monday is before the epoch).
__device__ __forceinline__ u64 timestamp_floor(u32 unit, u64 t, bool* bad) {
    if (t > kMaxTimestamp) {
        *bad = true;
        return 0;
    }
    if (unit == 0) return t - t % 3600;
    const u32 z = (u32)(t / 86400);
    u32 first;  // the first day of the bucket
    if (unit == 1) {
        first = z;
    } else if (unit == 2) {
        if (z < 4) *bad = true;
        first = z - (z + 3) % 7;
    } else {
        const Civil c = civil_from_days(z);
        first = z - (unit == 3 ? c.d - 1 : c.yday);
    }
    return (u64)first * 86400;
}

// The C locale's names, 10 bytes per entry: the weekdays from Sunday, then the months.  %a / %b are the first three.
__device__ const char kTimeNames[19][10] = {"Sunday", "Monday", "Tuesday", "Wednesday", "Thursday", "Friday", "Saturday",
                                            "January", "February", "March", "April", "May", "June", "July", "August",
                                            "September", "October", "November", "December"};
__device__ const u8 kTimeNameLength[19] = {6, 6, 7, 9, 8, 6, 8, 7, 8, 5, 5, 3, 4, 4, 6, 9, 7, 8, 8};

// glibc strftime's iso_week_days: the days since the Monday of ISO week 1 of yday's year (negative: an earlier year's).
__device__ __forceinline__ int iso_week_days(int yday, int wday) { return yday - (yday - wday + 4 + 378) % 7 + 3; }

// Writes one value into a 64-byte line, 8 bytes per store.
struct LineWriter {
    u64* line;
    u64 acc = 0;
    u32 len = 0;
    __device__ __forceinline__ void put(u32 b) {
        acc |= (u64)b << (8 * (len & 7));
        if ((++len & 7) == 0) {
            line[(len >> 3) - 1] = acc;
            acc = 0;
        }
    }
    __device__ __forceinline__ void num(u32 v, u32 digits) {  // zero-padded to digits (1..4)
        if (digits >= 4) put('0' + v / 1000 % 10);
        if (digits >= 3) put('0' + v / 100 % 10);
        if (digits >= 2) put('0' + v / 10 % 10);
        put('0' + v % 10);
    }
    __device__ __forceinline__ void name(u32 k, u32 abbreviated) {
        const u32 n = abbreviated ? 3 : kTimeNameLength[k];
        for (u32 j = 0; j < n; ++j) put((u8)kTimeNames[k][j]);
    }
    __device__ __forceinline__ u32 finish() {
        if (len & 7) line[len >> 3] = acc;
        return len;
    }
};

// C-locale strftime(fmt, gmtime(t)) for t in [0, kMaxTimestamp] from the format's tokens (compile_format: a conversion
// byte and a literal byte each), written to line; -> its length.
__device__ __forceinline__ u32 format_timestamp(const u8* tok, u32 count, u64 t, u8* line) {
    const u32 z = (u32)(t / 86400), s = (u32)(t - (u64)z * 86400);
    const Civil c = civil_from_days(z);
    const u32 wday = (z + 4) % 7, hour = s / 3600, minute = s / 60 % 60;
    LineWriter w{reinterpret_cast<u64*>(line)};
#pragma unroll 1
    for (u32 k = 0; k < count; ++k) {
        const u32 conv = tok[2 * k];
        switch (conv) {
            case 0: w.put(tok[2 * k + 1]); break;
            case 'a': case 'A': w.name(wday, conv == 'a'); break;
            case 'b': case 'B': w.name(6 + c.m, conv == 'b'); break;
            case 'p': w.put(hour < 12 ? 'A' : 'P'); w.put('M'); break;
            case 'C': w.num(c.y / 100, 2); break;
            case 'd': w.num(c.d, 2); break;
            case 'e': w.put(c.d < 10 ? ' ' : '0' + c.d / 10); w.put('0' + c.d % 10); break;
            case 'H': w.num(hour, 2); break;
            case 'I': w.num(hour % 12 ? hour % 12 : 12, 2); break;
            case 'j': w.num(c.yday + 1, 3); break;
            case 'm': w.num(c.m, 2); break;
            case 'M': w.num(minute, 2); break;
            case 'S': w.num(s % 60, 2); break;
            case 'u': w.num(wday ? wday : 7, 1); break;
            case 'w': w.num(wday, 1); break;
            case 'y': w.num(c.y % 100, 2); break;
            case 'Y': w.num(c.y, 4); break;
            case 'U': w.num((c.yday + 7 - wday) / 7, 2); break;
            case 'W': w.num((c.yday + 7 - (wday + 6) % 7) / 7, 2); break;
            default: {  // G, g, V
                int year = (int)c.y, days = iso_week_days((int)c.yday, (int)wday);
                const int leap = (year % 4 == 0 && year % 100 != 0) || year % 400 == 0;
                if (days < 0) {
                    --year;
                    const int pleap = (year % 4 == 0 && year % 100 != 0) || year % 400 == 0;
                    days = iso_week_days((int)c.yday + 365 + pleap, (int)wday);
                } else {
                    const int d = iso_week_days((int)c.yday - (365 + leap), (int)wday);
                    if (d >= 0) {
                        ++year;
                        days = d;
                    }
                }
                if (conv == 'V') w.num((u32)days / 7 + 1, 2);
                else if (conv == 'G') w.num((u32)year, 4);
                else w.num((u32)year % 100, 2);
            }
        }
    }
    return w.finish();
}

// expression_body with the time ops: a copy kept line for line beside it (kCond, kPred and kTime fixed), so that
// expression_body, its readers and the five kernels built from it compile exactly as before.  A change to one body
// belongs in the other.
template <bool kStrings>
__device__ __forceinline__ void expression_time_body(const ExprArgs& A, const PredArgs& Q, u8* scratch) {
    constexpr bool kCond = true, kPred = true, kTime = true;
    // the error bit stacks: kEW bits per entry, entry d from the top at bit kEW * d (a 16-deep stack fills 32 / 48 bits;
    // with kTime 48 / 64); the range error is the entry's top bit, kEsTime, and kErrTimeRange in the error word
    using ErrStack = typename std::conditional<kStrings || kTime, u64, u32>::type;
    constexpr u32 kEW = (kStrings ? 3 : 2) + (kTime ? 1 : 0);
    constexpr ErrStack kEM = (ErrStack)((1u << kEW) - 1);
    constexpr u32 kEsTime = 1u << (kEW - 1);
    extern __shared__ __align__(16) unsigned char smem[];
    ExprNodeDev* s_nodes = reinterpret_cast<ExprNodeDev*>(smem);
    ColumnDev* s_cols = reinterpret_cast<ColumnDev*>(s_nodes + A.node_count);
    StringDev* s_strs = reinterpret_cast<StringDev*>(s_cols + A.column_count);
    u64* s_stack = reinterpret_cast<u64*>(s_strs + (kStrings ? A.string_count : 0)) + threadIdx.x;  // entry d: [d * kExprThreads]
    // expression_kernel<true, true>: the piece stack [p * kExprThreads], then a short-value stage per warp
    u64* s_pptr = s_stack + (kStrings ? (size_t)(A.max_depth - 1) * kExprThreads : 0);
    u32* s_plen = reinterpret_cast<u32*>(s_pptr - threadIdx.x + (size_t)A.max_pieces * kExprThreads) + threadIdx.x;
    u8* s_stage = reinterpret_cast<u8*>((reinterpret_cast<uintptr_t>(s_plen - threadIdx.x + (size_t)A.max_pieces * kExprThreads) + 15) & ~(uintptr_t)15) +
                  (threadIdx.x >> 5) * kStageBytes;
    {
        const u32* src = reinterpret_cast<const u32*>(A.nodes);
        u32* dst = reinterpret_cast<u32*>(s_nodes);
        for (u32 k = threadIdx.x; k < A.node_count * (u32)(sizeof(ExprNodeDev) / 4); k += blockDim.x) dst[k] = src[k];
        src = reinterpret_cast<const u32*>(A.columns);
        dst = reinterpret_cast<u32*>(s_cols);
        for (u32 k = threadIdx.x; k < A.column_count * (u32)(sizeof(ColumnDev) / 4); k += blockDim.x) dst[k] = src[k];
        if constexpr (kStrings) {
            src = reinterpret_cast<const u32*>(A.strings);
            dst = reinterpret_cast<u32*>(s_strs);
            for (u32 k = threadIdx.x; k < A.string_count * (u32)(sizeof(StringDev) / 4); k += blockDim.x) dst[k] = src[k];
        }
    }
    const u8* s_pat = nullptr;
    const u64* s_list = nullptr;
    if constexpr (kPred) {
        uint4* pat = reinterpret_cast<uint4*>(smem + Q.pred_smem);
        const uint4* psrc = reinterpret_cast<const uint4*>(Q.patterns);
        for (u32 k = threadIdx.x; k < Q.pattern_bytes / 16; k += blockDim.x) pat[k] = psrc[k];
        u64* list = reinterpret_cast<u64*>(smem + Q.pred_smem + Q.pattern_bytes);
        for (u32 k = threadIdx.x; k < Q.staged_list; k += blockDim.x) list[k] = Q.lists[k];
        s_pat = smem + Q.pred_smem;
        s_list = list;
    }
    __syncthreads();

    const u32 lane = threadIdx.x & 31;
    const u64 words = (A.n + 63) / 64 * 2;  // 32-row groups, the last 64-bit word of the bitmap included
    const u64 warps = (u64)gridDim.x * (blockDim.x >> 5);
    u32 err = 0;
    u64 null_rows = 0;
    for (u64 w = (u64)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); w < words; w += warps) {
        const u64 row0 = w * 32;
        const u64 i = row0 + lane;
        const u32 sel = A.selection ? A.selection[w] : ~0u;
        const bool live = i < A.n && ((sel >> lane) & 1);
        u64 top = 0;
        u32 nul_stack = 1;  // bit d: entry d from the top is NULL
        u32 np = 0;         // pieces on the piece stack
        u32 cases = 0;      // 2 bits per piece: its case map
        ErrStack es = 0;    // the entries' error bits
        if (sel != 0) {
            u32 depth = 0;  // entries below the top, in s_stack
#pragma unroll 1
            for (u32 k = 0; k < A.node_count; ++k) {
                const ExprNodeDev nd = s_nodes[k];
                {
                    if (nd.op == YTGPU_EXPR_TIMESTAMP_FLOOR) {
                        if (!(nul_stack & 1)) {
                            bool bad = false;
                            top = timestamp_floor(nd.col, top, &bad);
                            if (bad) es |= kEsTime;
                        }
                        continue;
                    }
                    if (kStrings && nd.op == YTGPU_EXPR_FORMAT_TIMESTAMP) {
                        // one piece: the value formatted into this thread's line of the node (nd.col: its FORMAT ordinal)
                        if (!(nul_stack & 1)) {
                            if (top > kMaxTimestamp) {
                                es |= kEsTime;
                                nul_stack |= 1;
                                top = 0;
                            } else {
                                u8* line = scratch + ((size_t)nd.col * gridDim.x * blockDim.x + (size_t)blockIdx.x * blockDim.x + threadIdx.x) *
                                                         kFormatLine;
                                const u32 len = format_timestamp(s_pat + (nd.constant >> 32), (u32)nd.constant, top, line);
                                s_pptr[np * kExprThreads] = reinterpret_cast<u64>(line);
                                s_plen[np * kExprThreads] = len;
                                cases &= ~(3u << (2 * np));
                                ++np;
                                top = 1;
                            }
                        }
                        continue;
                    }
                }
                if (nd.op == YTGPU_EXPR_COLUMN || nd.op == YTGPU_EXPR_CONSTANT) {
                    bool nul = !live;
                    u64 v = nd.constant;
                    if (kStrings && nd.type == YTGPU_TYPE_STRING) {
                        const u8* p = A.consts + (nd.constant >> 32);
                        u32 len = (u32)nd.constant;
                        if (nd.op == YTGPU_EXPR_COLUMN && !nul) {
                            const StringDev& sc = s_strs[nd.col];
                            ytgpu_value sv;
                            u32 bad = 0;
                            nul = !string_at(sc, i, &sv, &bad);
                            if (bad) err |= kErrOutOfHeap;
                            p = sc.heap + sv.data;
                            len = sv.length;
                        }
                        v = 0;
                        if (!nul) {  // one piece
                            s_pptr[np * kExprThreads] = reinterpret_cast<u64>(p);
                            s_plen[np * kExprThreads] = len;
                            cases &= ~(3u << (2 * np));
                            ++np;
                            v = 1;
                        }
                    } else if (nd.op == YTGPU_EXPR_COLUMN) {
                        const ColumnDev& c = s_cols[nd.col];
                        v = scalar_value(c, i, row0, live, &nul);
                        if (c.value_type == YTGPU_TYPE_BOOLEAN) v = v != 0;
                    }
                    if (k) s_stack[depth++ * kExprThreads] = top;
                    top = nul ? 0 : v;
                    nul_stack = (nul_stack << 1) | (nul ? 1u : 0u);
                    if (kCond) es <<= kEW;
                } else if (nd.op == YTGPU_EXPR_NEG || nd.op == YTGPU_EXPR_BIT_NOT || nd.op == YTGPU_EXPR_CAST) {
                    if (!(nul_stack & 1)) top = unary_op(nd.op, nd.type, nd.from, top);
                } else if (kCond && nd.op == YTGPU_EXPR_NOT) {
                    top ^= (nul_stack & 1) ^ 1;  // a NULL entry holds 0 and stays NULL
                } else if (kCond && (nd.op == YTGPU_EXPR_IS_NULL || nd.op == YTGPU_EXPR_IS_NOT_NULL)) {
                    if (kStrings && nd.from == YTGPU_TYPE_STRING) np -= (u32)top;  // a NULL string has no pieces
                    top = (nul_stack & 1) ^ (nd.op == YTGPU_EXPR_IS_NULL ? 0u : 1u);
                    nul_stack &= ~1u;
                } else if (kPred && nd.op == YTGPU_EXPR_IN) {
                    // lower bound over the sorted entries, then equality on the entry found (a number: the EQ rule)
                    const u32 first = (u32)(nd.constant >> 32), end = first + (u32)nd.constant;
                    const bool str = kStrings && nd.from == YTGPU_TYPE_STRING;
                    const u32 p0 = np - (str ? (u32)top : 0u);
                    bool r = false;
                    if (!(nul_stack & 1)) {
                        const u64 key = str ? 0 : in_key(nd.from, top);
                        u32 lo = first, cnt = end - first;
                        int c = 1;
                        while (cnt > 0) {
                            const u32 half = cnt >> 1, mid = lo + half;
                            const u64 e = mid < Q.staged_list ? s_list[mid] : __ldg(Q.lists + mid);
                            const bool below = str ? pieces_compare_plain(s_pptr, s_plen, cases, p0, (u32)top, 0, 0, A.consts + (e >> 32), (u32)e) > 0
                                                   : e < key;
                            if (below) {
                                lo = mid + 1;
                                cnt -= half + 1;
                            } else {
                                cnt = half;
                            }
                        }
                        if (lo < end) {
                            const u64 e = lo < Q.staged_list ? s_list[lo] : __ldg(Q.lists + lo);
                            if (str) c = pieces_compare_plain(s_pptr, s_plen, cases, p0, (u32)top, 0, 0, A.consts + (e >> 32), (u32)e);
                            r = str ? c == 0 : passes(YTGPU_CMP_EQ, nd.from, top, minmax_decode(nd.from, e));
                        }
                    }
                    np = p0;  // a STRING operand's pieces are dropped
                    top = r ? 1 : 0;
                } else if (kStrings && kPred && (nd.op == YTGPU_EXPR_STARTS_WITH || nd.op == YTGPU_EXPR_CONTAINS || nd.op == YTGPU_EXPR_LIKE)) {
                    const u32 p0 = np - (u32)top;
                    bool r = false;
                    if (!(nul_stack & 1)) {
                        u64 len = 0;
                        for (u32 p = p0; p < np; ++p) len += s_plen[p * kExprThreads];
                        PieceBytesPlain src{s_pptr, s_plen, cases, p0};
                        if (nd.op == YTGPU_EXPR_STARTS_WITH) {
                            const u8* q = A.consts + (nd.constant >> 32);
                            const u32 ql = (u32)nd.constant;
                            r = len >= ql;
                            for (u32 j = 0; r && j < ql; ++j) r = src(j) == __ldg(q + j);
                        } else if (len > 0xffffffffull) {
                            err |= kErrMatchTooLong;
                        } else {  // PieceBytesPlain even for one piece: the filter's contiguous scan reads through __ldg
                            r = pattern_match(s_pat + nd.constant, src, (u32)len);
                        }
                    }
                    np = p0;
                    top = r ? 1 : 0;
                } else if (kStrings && (nd.op == YTGPU_EXPR_LOWER || nd.op == YTGPU_EXPR_UPPER)) {
                    if (!(nul_stack & 1)) {
                        const u32 first = np - (u32)top;
                        if (A.mode != kModeFill)  // the fill pass runs only once the size pass found no error
                            for (u32 p = first; p < np; ++p)
                                if (!ascii_only_plain(reinterpret_cast<const u8*>(s_pptr[p * kExprThreads]), s_plen[p * kExprThreads]))
                                    es |= kErrNonAscii;
                        const u32 mask = (u32)(((1ull << (2 * np)) - 1) & ~((1ull << (2 * first)) - 1));
                        cases = (cases & ~mask) | ((nd.op == YTGPU_EXPR_LOWER ? 0x55555555u : 0xaaaaaaaau) & mask);
                    }
                } else if (kStrings && nd.op == YTGPU_EXPR_FARM_HASH) {
                    // GetFarmFingerprint over the operands, deepest first; a NULL operand (a numeric one holds 0) hashes as
                    // fingerprint_u64(0), a string one is a single piece
                    const u32 count = nd.col, strs = (u32)nd.constant, below = depth - (count - 1);
                    u32 sp = 0;
                    for (u32 j = 0; j < count; ++j)
                        if ((strs >> j) & 1) sp += (u32)(j + 1 == count ? top : s_stack[(below + j) * kExprThreads]);
                    u32 p = np - sp;
                    u64 h = 0xdeadc0deULL;
                    for (u32 j = 0; j < count; ++j) {
                        const u64 v = j + 1 == count ? top : s_stack[(below + j) * kExprThreads];
                        u64 f;
                        if (((strs >> j) & 1) && v) {
                            f = fh::fingerprint_bytes(reinterpret_cast<const u8*>(s_pptr[p * kExprThreads]), s_plen[p * kExprThreads]);
                            ++p;
                        } else {
                            f = fh::fingerprint_u64((strs >> j) & 1 ? 0 : v);
                        }
                        h = fh::fingerprint_u128(h, f);
                    }
                    np -= sp;
                    depth = below;
                    top = h ^ (u64)count;
                    nul_stack = (nul_stack >> count) << 1;
                    ErrStack er = 0;
                    for (u32 j = 0; j < count; ++j) er |= (es >> (kEW * j)) & kEM;
                    es = ((es >> (kEW * count)) << kEW) | er;
                } else if (kCond && nd.op == YTGPU_EXPR_IF) {
                    // c a b IF: the value, NULL flag and error bits of the branch c takes; a NULL c takes neither
                    const u64 b = top, a = s_stack[(depth - 1) * kExprThreads], c = s_stack[(depth - 2) * kExprThreads];
                    depth -= 2;
                    const u32 nb = nul_stack & 1, na = (nul_stack >> 1) & 1, nc = (nul_stack >> 2) & 1;
                    if (kStrings && nd.type == YTGPU_TYPE_STRING) {  // a's pieces, then b's, on top of the piece stack
                        const u32 first = np - (u32)(a + b);
                        if (nc) {
                            np = first;
                        } else if (c) {
                            np -= (u32)b;
                        } else {  // b's pieces move down over a's, at most YTGPU_EXPR_MAX_PIECES of them
                            for (u32 p = 0; p < (u32)b; ++p) {
                                s_pptr[(first + p) * kExprThreads] = s_pptr[(first + (u32)a + p) * kExprThreads];
                                s_plen[(first + p) * kExprThreads] = s_plen[(first + (u32)a + p) * kExprThreads];
                            }
                            const u64 bc = ((u64)cases >> (2 * (first + (u32)a))) & ((1ull << (2 * (u32)b)) - 1);
                            cases = (u32)(((u64)cases & ((1ull << (2 * first)) - 1)) | (bc << (2 * first)));
                            np = first + (u32)b;
                        }
                    }
                    top = c ? a : b;  // a NULL c holds 0: b, which nc makes NULL below
                    const u32 nr = nc | (c ? na : nb);
                    top = nr ? 0 : top;
                    nul_stack = ((nul_stack >> 3) << 1) | nr;
                    const ErrStack er = ((es >> (2 * kEW)) & kEM) | (nc ? 0 : (es >> (c ? kEW : 0)) & kEM);
                    es = ((es >> (3 * kEW)) << kEW) | er;
                } else {
                    const u64 a = s_stack[--depth * kExprThreads], b = top;
                    const u32 nb = nul_stack & 1, na = (nul_stack >> 1) & 1;
                    ErrStack er = (es | (es >> kEW)) & kEM;  // both operands' bits
                    u32 nr;
                    if (nd.op == YTGPU_EXPR_IF_NULL) {
                        top = na ? b : a;
                        nr = na & nb;
                        if (kStrings && nd.type == YTGPU_TYPE_STRING && !na) np -= (u32)b;  // a NULL first operand has no pieces
                    } else if (kStrings && nd.op == YTGPU_EXPR_CONCAT) {
                        nr = na | nb;
                        np -= nr ? (u32)(a + b) : 0;
                        top = nr ? 0 : a + b;
                    } else if (kCond && nd.op == YTGPU_EXPR_COMPARE) {
                        nr = na | nb;
                        bool r;
                        if (kStrings && nd.from == YTGPU_TYPE_STRING) {  // both operands' pieces are dropped
                            np -= (u32)(a + b);
                            r = !nr && cmp_holds(nd.col, pieces_compare_plain(s_pptr, s_plen, cases, np, (u32)a, np + (u32)a, (u32)b));
                        } else {
                            r = !nr && passes(nd.col, nd.from, a, b);
                        }
                        top = r ? 1 : 0;
                    } else if (kCond && (nd.op == YTGPU_EXPR_AND || nd.op == YTGPU_EXPR_OR)) {
                        // Kleene over 0 / 1 entries (a NULL one holds 0): F AND x = F, T OR x = T, else NULL with a NULL
                        // operand.  A deciding left operand drops the right one's error bits.
                        const bool is_and = nd.op == YTGPU_EXPR_AND;
                        const bool left_decides = is_and ? (!na && !a) : (a != 0);
                        const bool decided = left_decides || (is_and ? (!nb && !b) : (b != 0));
                        top = is_and ? (a & b) : (a | b);
                        nr = !decided && (na | nb);
                        if (left_decides) er = (es >> kEW) & kEM;
                    } else {
                        nr = na | nb;
                        u32 e = 0;
                        top = nr ? 0 : binary_op(nd.op, nd.type, a, b, kCond ? &e : &err);
                        if (kCond) er |= e;
                    }
                    nul_stack = ((nul_stack >> 2) << 1) | nr;
                    if (kCond) es = ((es >> (2 * kEW)) << kEW) | er;
                }
            }
        }
        {  // the result's error bits, the range error as kErrTimeRange
            const u32 r = (u32)(es & kEM);
            err |= (r & (kEsTime - 1)) | (r & kEsTime ? kErrTimeRange : 0u);
        }
        const bool nul = !live || (nul_stack & 1);
        if (!kStrings || A.mode == kModeValues) {
            const u32 m = __ballot_sync(0xffffffffu, nul && i < A.n);
            if (i < A.n) A.values[i] = nul ? 0 : top;
            if (lane == 0) {
                A.nulls[w] = m;
                null_rows += (u64)__popc(m);
            }
            continue;
        }
        if constexpr (kStrings) {
            u64 len = 0;
            if (!nul)
                for (u32 p = 0; p < np; ++p) len += s_plen[p * kExprThreads];
            if (A.mode == kModeSize) {
                if (len > 0xffffffffull) {
                    err |= kErrTooLong;
                    len = 0;
                }
                const u32 m = __ballot_sync(0xffffffffu, nul && i < A.n);
                if (i < A.n) {
                    A.starts[i] = len;
                    A.lengths[i] = (u32)len;
                    A.null_bytes[i] = nul ? 1 : 0;
                }
                if (lane == 0) null_rows += (u64)__popc(m);
                continue;
            }
            // kModeFill
            if (row0 >= A.n) continue;  // a group past the last row (the bitmap's last word); warp-uniform
            const u64 pos = i < A.n ? A.starts[i] : 0;
            const bool is_long = len > kShortValue;
            u32 todo = __ballot_sync(0xffffffffu, is_long);
            if (todo == 0) {
                // every value of the group is short: the group's output [p0, p1) is one stretch, assembled in the warp's stage
                // from its 16-byte boundary below heap + p0 and written out with 16-byte stores
                const u64 p0 = __shfl_sync(0xffffffffu, pos, 0);
                u64 p1 = i < A.n ? pos + len : p0;
#pragma unroll
                for (int d = 16; d > 0; d >>= 1) p1 = max(p1, __shfl_xor_sync(0xffffffffu, p1, d));
                const u32 skew = (u32)(reinterpret_cast<uintptr_t>(A.heap + p0) & 15);
                u8* dst = s_stage + skew + (u32)(pos - p0);
                if (len)
                    for (u32 p = 0; p < np; ++p) {
                        const u8* src = reinterpret_cast<const u8*>(s_pptr[p * kExprThreads]);
                        const u32 l = s_plen[p * kExprThreads], cm = (cases >> (2 * p)) & 3;
                        for (u32 j = 0; j < l; ++j) dst[j] = (u8)case_byte(src[j], cm);
                        dst += l;
                    }
                __syncwarp();
                const u32 begin = skew, end = skew + (u32)(p1 - p0);
                u8* gbase = A.heap + p0 - skew;  // 16-byte aligned
                for (u32 q = lane; q * 16 < end; q += 32) {
                    const u32 lo = q * 16, hi = lo + 16;
                    if (lo >= begin && hi <= end) {
                        reinterpret_cast<uint4*>(gbase)[q] = reinterpret_cast<const uint4*>(s_stage)[q];
                    } else {
                        for (u32 b = max(lo, begin); b < min(hi, end); ++b) gbase[b] = s_stage[b];
                    }
                }
                __syncwarp();  // the stage is reused by the next group
                continue;
            }
            if (!is_long && len) {
                u8* dst = A.heap + pos;
                for (u32 p = 0; p < np; ++p) {
                    const u8* src = reinterpret_cast<const u8*>(s_pptr[p * kExprThreads]);
                    const u32 l = s_plen[p * kExprThreads], cm = (cases >> (2 * p)) & 3;
                    for (u32 j = 0; j < l; ++j) dst[j] = (u8)case_byte(src[j], cm);
                    dst += l;
                }
            }
            __syncwarp();  // the owners' piece stacks and FORMAT_TIMESTAMP lines, written while the program ran, are read by the whole warp
            while (todo) {  // long values, one at a time by the whole warp, piece by piece from the owner's piece stack
                const int l = __ffs(todo) - 1;
                todo &= todo - 1;
                const u32 owner = (threadIdx.x & ~31u) + (u32)l;
                const u32 lnp = __shfl_sync(0xffffffffu, np, l), lcases = __shfl_sync(0xffffffffu, cases, l);
                u8* dst = A.heap + __shfl_sync(0xffffffffu, pos, l);
                for (u32 p = 0; p < lnp; ++p) {
                    const u8* src = reinterpret_cast<const u8*>(s_pptr[p * kExprThreads - threadIdx.x + owner]);
                    const u32 pl = s_plen[p * kExprThreads - threadIdx.x + owner];
                    warp_copy_plain(dst, src, pl, (lcases >> (2 * p)) & 3, lane);
                    dst += pl;
                }
            }
            __syncwarp();  // ... and are overwritten by the next group's program
        }
    }
    err = __reduce_or_sync(0xffffffffu, err);
    if (lane == 0) {
        if (null_rows) atomicAdd(&A.result[0], (unsigned long long)null_rows);
        if (err) atomicOr(&A.result[1], (unsigned long long)err);
    }
}

// Programs with TIMESTAMP_FLOOR or FORMAT_TIMESTAMP (and any other op): scratch holds 64 bytes per thread of the grid and
// FORMAT_TIMESTAMP node.
template <bool kStrings>
__global__ void __launch_bounds__(kExprThreads) __maxnreg__(kStrings ? 96 : 40)
    expression_time_kernel(const ExprArgs A, const PredArgs Q, u8* scratch) {
    expression_time_body<kStrings>(A, Q, scratch);
}

// ---- host ----
struct CheckedExpr {
    std::vector<ExprNodeDev> nodes;
    SlotMap cols, strings;  // the referenced columns' compact tables
    u32 max_depth = 0;
    u32 max_pieces = 0;
    bool strings_kernel = false;  // a STRING node or FARM_HASH: expression_kernel<true, true>
    bool conditional = false;     // a conditional op: expression_kernel<false, true> for a scalar program
    bool predicates = false;      // IN, STARTS_WITH, CONTAINS or LIKE: expression_pred_kernel
    bool time = false;            // TIMESTAMP_FLOOR or FORMAT_TIMESTAMP: expression_time_kernel
    u32 formats = 0;              // FORMAT_TIMESTAMP nodes: scratch lines per thread
    std::vector<u64> lists;       // the sorted IN entries, node by node
    std::vector<u8> patterns;     // the compiled CONTAINS / LIKE patterns and FORMAT_TIMESTAMP formats, node by node
    u8 type = 0;  // the result type
};

bool is_number_type(u32 t) { return t == YTGPU_TYPE_INT64 || t == YTGPU_TYPE_UINT64 || t == YTGPU_TYPE_DOUBLE; }
bool is_integer_type(u32 t) { return t == YTGPU_TYPE_INT64 || t == YTGPU_TYPE_UINT64; }

// A FORMAT_TIMESTAMP format compiled into tokens of two bytes, (conversion, 0) or (0, literal byte), appended to *out at
// an 8-byte boundary (the patterns beside them are read in 8-byte words).  %D %F %R %T expand to their conversions, %h is
// %b, %n %t %% are literals.  -> nullptr, or the reason the format is refused (YTGPU_ERR_UNSUPPORTED).
const char* compile_format(const u8* f, u32 len, std::vector<u8>* out, u32* tokens) {
    static const char kOne[] = "aAbBpCdeHIjmMSuwyYUWGgV";
    static const u8 kWidth[] = {3, 9, 3, 9, 2, 2, 2, 2, 2, 2, 3, 2, 2, 2, 1, 1, 2, 4, 2, 2, 4, 2, 2};  // the widest output
    std::vector<u8> t;
    u32 bytes = 0;
    auto conv = [&](char c) {
        t.push_back((u8)c);
        t.push_back(0);
        bytes += kWidth[strchr(kOne, c) - kOne];
    };
    auto lit = [&](u8 b) {
        t.push_back(0);
        t.push_back(b);
        ++bytes;
    };
    for (u32 j = 0; j < len; ++j) {
        if (f[j] != '%') {
            lit(f[j]);
            continue;
        }
        if (++j == len) return "a lone % ends the format";
        const char c = (char)f[j];
        if (c != 0 && strchr(kOne, c)) conv(c);
        else if (c == 'h') conv('b');
        else if (c == 'D') for (char x : {'m', '/', 'd', '/', 'y'}) x == '/' ? lit('/') : conv(x);
        else if (c == 'F') for (char x : {'Y', '-', 'm', '-', 'd'}) x == '-' ? lit('-') : conv(x);
        else if (c == 'R') for (char x : {'H', ':', 'M'}) x == ':' ? lit(':') : conv(x);
        else if (c == 'T') for (char x : {'H', ':', 'M', ':', 'S'}) x == ':' ? lit(':') : conv(x);
        else if (c == 'n') lit('\n');
        else if (c == 't') lit('\t');
        else if (c == '%') lit('%');
        else return "a conversion, modifier, flag or width outside the supported set";
    }
    if (bytes > (u32)YTGPU_EXPR_MAX_FORMATTED_BYTES) return "its longest output exceeds YTGPU_EXPR_MAX_FORMATTED_BYTES";
    *tokens = (u32)(t.size() / 2);
    out->insert(out->end(), t.begin(), t.end());
    out->resize((out->size() + 7) & ~(size_t)7);
    return nullptr;
}

// `strings`: the program comes through ytgpu_evaluate_expression_strings, which takes string leaves and the string ops.
Status check_expression(const ytgpu_column_view* columns, u32 column_count, bool strings, u32 string_count, const u8* consts,
                        u64 const_bytes, const ytgpu_expr_node* program, u32 node_count, CheckedExpr* out) {
    if (node_count == 0 || node_count > (u32)YTGPU_EXPR_MAX_NODES)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "an expression program has 1 .. %d nodes", YTGPU_EXPR_MAX_NODES);
    if (!program) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null program");
    struct Entry {
        u8 type;
        u8 plain;     // STRING: one piece without a case map at most (a leaf, a constant or IF_NULL of those)
        u32 pieces;   // STRING: the most pieces it may have
    };
    std::vector<Entry> stack;
    u32 pieces = 0;  // on the whole stack
    u64 in_entries = 0;
    for (u32 k = 0; k < node_count; ++k) {
        const ytgpu_expr_node& N = program[k];
        ExprNodeDev d{};
        d.op = (u8)N.op;
        const bool string_op = N.op == YTGPU_EXPR_CONCAT || N.op == YTGPU_EXPR_LOWER || N.op == YTGPU_EXPR_UPPER || N.op == YTGPU_EXPR_FARM_HASH ||
                               (N.op >= YTGPU_EXPR_IN && N.op <= YTGPU_EXPR_LIKE) || N.op == YTGPU_EXPR_FORMAT_TIMESTAMP;
        if (string_op && !strings) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: unknown op %d", k, N.op);
        switch (N.op) {
            case YTGPU_EXPR_COLUMN: {
                if (N.column < 0 || (u64)N.column >= (u64)column_count + (strings ? string_count : 0))
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: column %d out of range", k, N.column);
                if ((u32)N.column >= column_count) {  // string_columns[column - column_count]
                    d.col = out->strings.slot((u32)N.column - column_count);
                    d.type = YTGPU_TYPE_STRING;
                    stack.push_back({YTGPU_TYPE_STRING, 1, 1});
                    ++pieces;
                    break;
                }
                const u8 t = columns[N.column].value_type;
                if (!is_scalar_type(t))
                    return make_status(YTGPU_ERR_UNSUPPORTED, "node %u: column %d has value type 0x%x (INT64, UINT64, DOUBLE or BOOLEAN)", k,
                                       N.column, t);
                d.col = out->cols.slot((u32)N.column);
                d.type = t;
                stack.push_back({t, 0, 0});
                break;
            }
            case YTGPU_EXPR_CONSTANT:
                if (strings && N.type == YTGPU_TYPE_STRING) {
                    const u64 off = N.constant >> 32, len = N.constant & 0xffffffffull;
                    if (off + len > const_bytes)
                        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: string constant outside string_constants", k);
                    d.type = N.type;
                    d.constant = N.constant;
                    stack.push_back({YTGPU_TYPE_STRING, 1, 1});
                    ++pieces;
                    break;
                }
                if (!is_scalar_type(N.type)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: unknown constant type 0x%x", k, N.type);
                if (N.type == YTGPU_TYPE_BOOLEAN && N.constant > 1)
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: a BOOLEAN constant is 0 or 1", k);
                d.type = N.type;
                d.constant = N.constant;
                stack.push_back({N.type, 0, 0});
                break;
            case YTGPU_EXPR_NEG:
            case YTGPU_EXPR_BIT_NOT:
            case YTGPU_EXPR_CAST: {
                if (stack.empty()) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: stack underflow", k);
                const u8 t = stack.back().type;
                if (t == YTGPU_TYPE_STRING) return make_status(YTGPU_ERR_UNSUPPORTED, "node %u: op %d does not take strings", k, N.op);
                if (N.op == YTGPU_EXPR_CAST) {
                    if (!is_number_type(N.type))
                        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: CAST to type 0x%x (INT64, UINT64 or DOUBLE)", k, N.type);
                    d.from = t;
                    d.type = N.type;
                } else {
                    if (N.op == YTGPU_EXPR_NEG ? !is_number_type(t) : !is_integer_type(t))
                        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: op %d does not take type 0x%x", k, N.op, t);
                    d.type = t;
                }
                stack.back().type = d.type;
                break;
            }
            case YTGPU_EXPR_LOWER:
            case YTGPU_EXPR_UPPER:
                if (stack.empty()) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: stack underflow", k);
                if (stack.back().type != YTGPU_TYPE_STRING)
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: op %d takes a STRING, not type 0x%x", k, N.op, stack.back().type);
                d.type = YTGPU_TYPE_STRING;
                stack.back().plain = 0;
                break;
            case YTGPU_EXPR_FARM_HASH: {
                if (N.column < 1 || N.column > YTGPU_EXPR_MAX_HASH_OPERANDS)
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: FARM_HASH of %d operands (1 .. %d)", k, N.column,
                                       YTGPU_EXPR_MAX_HASH_OPERANDS);
                const u32 count = (u32)N.column;
                if (stack.size() < count) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: stack underflow", k);
                u64 strs = 0;
                for (u32 j = 0; j < count; ++j) {
                    const Entry& e = stack[stack.size() - count + j];
                    if (e.type != YTGPU_TYPE_STRING) continue;
                    if (!e.plain)
                        return make_status(YTGPU_ERR_UNSUPPORTED, "node %u: FARM_HASH of a CONCAT, LOWER, UPPER or FORMAT_TIMESTAMP result", k);
                    strs |= 1ull << j;
                    pieces -= e.pieces;
                }
                stack.resize(stack.size() - count);
                d.col = (u16)count;
                d.constant = strs;
                d.type = YTGPU_TYPE_UINT64;
                stack.push_back({YTGPU_TYPE_UINT64, 0, 0});
                break;
            }
            case YTGPU_EXPR_NOT:
            case YTGPU_EXPR_IS_NULL:
            case YTGPU_EXPR_IS_NOT_NULL: {
                if (stack.empty()) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: stack underflow", k);
                const Entry e = stack.back();
                if (N.op == YTGPU_EXPR_NOT && e.type != YTGPU_TYPE_BOOLEAN)
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: NOT takes a BOOLEAN, not type 0x%x", k, e.type);
                pieces -= e.pieces;
                d.from = e.type;
                d.type = YTGPU_TYPE_BOOLEAN;
                stack.back() = {YTGPU_TYPE_BOOLEAN, 0, 0};
                break;
            }
            case YTGPU_EXPR_IF: {
                if (stack.size() < 3) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: stack underflow", k);
                const Entry eb = stack.back();
                stack.pop_back();
                const Entry ea = stack.back();
                stack.pop_back();
                if (stack.back().type != YTGPU_TYPE_BOOLEAN)
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: IF's condition has type 0x%x, not BOOLEAN", k, stack.back().type);
                if (ea.type != eb.type)
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: IF branches of types 0x%x and 0x%x (CAST one of them)", k, ea.type,
                                       eb.type);
                d.type = ea.type;
                stack.back() = {ea.type, (u8)(ea.plain & eb.plain), std::max(ea.pieces, eb.pieces)};  // keeps one branch's pieces
                pieces -= std::min(ea.pieces, eb.pieces);
                break;
            }
            case YTGPU_EXPR_COMPARE:
            case YTGPU_EXPR_AND:
            case YTGPU_EXPR_OR: {
                if (stack.size() < 2) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: stack underflow", k);
                const Entry eb = stack.back();
                stack.pop_back();
                const Entry ea = stack.back();
                if (ea.type != eb.type)
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: operands of types 0x%x and 0x%x (CAST one of them)", k, ea.type, eb.type);
                if (N.op == YTGPU_EXPR_COMPARE) {
                    if (N.column < YTGPU_CMP_LT || N.column > YTGPU_CMP_NE)
                        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: COMPARE with cmp %d (LT .. NE)", k, N.column);
                    d.col = (u16)N.column;
                    pieces -= ea.pieces + eb.pieces;
                } else if (ea.type != YTGPU_TYPE_BOOLEAN) {
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: op %d takes BOOLEANs, not type 0x%x", k, N.op, ea.type);
                }
                d.from = ea.type;
                d.type = YTGPU_TYPE_BOOLEAN;
                stack.back() = {YTGPU_TYPE_BOOLEAN, 0, 0};
                break;
            }
            case YTGPU_EXPR_IN: {
                if (stack.empty()) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: stack underflow", k);
                const Entry e = stack.back();
                const u64 off = N.constant >> 32, count = N.constant & 0xffffffffull;
                if ((off & 7) || off > const_bytes || count * 8 > const_bytes - off)
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: IN list outside string_constants or not 8-byte aligned", k);
                std::vector<u64> entries(count);
                if (count) memcpy(entries.data(), consts + off, count * 8);
                const u64 first = out->lists.size();
                YTGPU_TRY(add_in_list(k, e.type, entries.data(), (u32)count, consts, const_bytes, &in_entries, &out->lists));
                if (e.type == YTGPU_TYPE_BOOLEAN)  // after add_in_list: its entry limit is checked first, and it takes any bits
                    for (u64 j = 0; j < count; ++j)
                        if (entries[j] > 1)
                            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: IN entry %u of a BOOLEAN list is not 0 or 1", k, (u32)j);
                pieces -= e.pieces;
                d.from = e.type;
                d.type = YTGPU_TYPE_BOOLEAN;
                d.constant = (first << 32) | (out->lists.size() - first);
                stack.back() = {YTGPU_TYPE_BOOLEAN, 0, 0};
                break;
            }
            case YTGPU_EXPR_STARTS_WITH:
            case YTGPU_EXPR_CONTAINS:
            case YTGPU_EXPR_LIKE: {
                if (stack.empty()) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: stack underflow", k);
                const Entry e = stack.back();
                if (e.type != YTGPU_TYPE_STRING)
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: op %d takes a STRING, not type 0x%x", k, N.op, e.type);
                const u64 off = N.constant >> 32, len = N.constant & 0xffffffffull;
                const bool like = N.op == YTGPU_EXPR_LIKE;
                if (off > const_bytes || len > const_bytes - off)
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: %s outside string_constants", k,
                                       like ? "pattern" : (N.op == YTGPU_EXPR_CONTAINS ? "needle" : "prefix"));
                d.constant = N.constant;
                if (N.op != YTGPU_EXPR_STARTS_WITH) {
                    d.constant = out->patterns.size();
                    YTGPU_TRY(add_pattern(k, consts + off, (u32)len, like, like ? N.column : -1, &out->patterns));
                }
                pieces -= e.pieces;
                d.from = YTGPU_TYPE_STRING;
                d.type = YTGPU_TYPE_BOOLEAN;
                stack.back() = {YTGPU_TYPE_BOOLEAN, 0, 0};
                break;
            }
            case YTGPU_EXPR_TIMESTAMP_FLOOR:
            case YTGPU_EXPR_FORMAT_TIMESTAMP: {
                if (stack.empty()) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: stack underflow", k);
                const u8 t = stack.back().type;
                if (!is_integer_type(t))
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: op %d takes an INT64 or UINT64, not type 0x%x", k, N.op, t);
                d.from = t;
                if (N.op == YTGPU_EXPR_TIMESTAMP_FLOOR) {
                    if (N.column < YTGPU_TIMESTAMP_HOUR || N.column > YTGPU_TIMESTAMP_YEAR)
                        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: TIMESTAMP_FLOOR with unit %d (0 .. 4)", k, N.column);
                    d.col = (u16)N.column;
                    d.type = t;
                    break;
                }
                const u64 off = N.constant >> 32, len = N.constant & 0xffffffffull;
                if (off > const_bytes || len > const_bytes - off)
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: format outside string_constants", k);
                const u64 at = out->patterns.size();
                u32 tokens = 0;
                if (const char* why = compile_format(consts + off, (u32)len, &out->patterns, &tokens))
                    return make_status(YTGPU_ERR_UNSUPPORTED, "node %u: FORMAT_TIMESTAMP format: %s", k, why);
                d.col = (u16)out->formats++;
                d.constant = (at << 32) | tokens;
                d.type = YTGPU_TYPE_STRING;
                stack.back() = {YTGPU_TYPE_STRING, 0, 1};
                ++pieces;
                break;
            }
            case YTGPU_EXPR_ADD:
            case YTGPU_EXPR_SUB:
            case YTGPU_EXPR_MUL:
            case YTGPU_EXPR_DIV:
            case YTGPU_EXPR_MOD:
            case YTGPU_EXPR_BIT_AND:
            case YTGPU_EXPR_BIT_OR:
            case YTGPU_EXPR_BIT_XOR:
            case YTGPU_EXPR_IF_NULL:
            case YTGPU_EXPR_CONCAT: {
                if (stack.size() < 2) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: stack underflow", k);
                const Entry eb = stack.back();
                stack.pop_back();
                const Entry ea = stack.back();
                const u8 a = ea.type, b = eb.type;
                if (N.op == YTGPU_EXPR_CONCAT) {
                    if (a != YTGPU_TYPE_STRING || b != YTGPU_TYPE_STRING)
                        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: CONCAT of types 0x%x and 0x%x (two STRINGs)", k, a, b);
                    stack.back() = {YTGPU_TYPE_STRING, 0, ea.pieces + eb.pieces};
                    d.type = YTGPU_TYPE_STRING;
                    break;
                }
                if (N.op != YTGPU_EXPR_IF_NULL && (a == YTGPU_TYPE_STRING || b == YTGPU_TYPE_STRING))
                    return make_status(YTGPU_ERR_UNSUPPORTED, "node %u: op %d does not take strings", k, N.op);
                if (a != b) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: operands of types 0x%x and 0x%x (CAST one of them)", k, a, b);
                const bool ok = N.op == YTGPU_EXPR_IF_NULL ? true
                              : (N.op <= YTGPU_EXPR_DIV ? is_number_type(a) : is_integer_type(a));
                if (!ok) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: op %d does not take type 0x%x", k, N.op, a);
                d.type = a;
                if (a == YTGPU_TYPE_STRING) {  // IF_NULL keeps one operand's pieces
                    stack.back() = {YTGPU_TYPE_STRING, (u8)(ea.plain & eb.plain), std::max(ea.pieces, eb.pieces)};
                    pieces -= std::min(ea.pieces, eb.pieces);
                }
                break;
            }
            default:
                return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: unknown op %d", k, N.op);
        }
        if (stack.size() > (size_t)YTGPU_EXPR_MAX_DEPTH)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: stack deeper than %d", k, YTGPU_EXPR_MAX_DEPTH);
        if (pieces > (u32)YTGPU_EXPR_MAX_PIECES)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: more than %d string pieces on the stack", k, YTGPU_EXPR_MAX_PIECES);
        out->max_depth = std::max(out->max_depth, (u32)stack.size());
        out->max_pieces = std::max(out->max_pieces, pieces);
        out->strings_kernel |= d.type == YTGPU_TYPE_STRING || N.op == YTGPU_EXPR_FARM_HASH;
        out->conditional |= N.op >= YTGPU_EXPR_COMPARE && N.op <= YTGPU_EXPR_LIKE;
        out->predicates |= N.op >= YTGPU_EXPR_IN && N.op <= YTGPU_EXPR_LIKE;
        out->time |= N.op == YTGPU_EXPR_TIMESTAMP_FLOOR || N.op == YTGPU_EXPR_FORMAT_TIMESTAMP;
        out->nodes.push_back(d);
    }
    if (stack.size() != 1)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "the program leaves %d values on the stack, not 1", (int)stack.size());
    out->type = stack[0].type;
    return Status{};
}

// The outputs of a STRING result (ytgpu_evaluate_expression_strings).
struct StringResult {
    u8* heap;
    u64 capacity;
    u64* starts;
    u32* lengths;
    u8* null_bytemap;
    u64* heap_bytes;
};

Status evaluate_expression_impl(Context* ctx, const ytgpu_column_view* columns, u32 column_count, const ytgpu_string_column* string_columns,
                                u32 string_count, const u8* consts, u64 const_bytes, const StringResult* sr,
                                const ytgpu_expr_node* program, u32 node_count, const u8* selection, u64* out_values, u8* out_null_bitmap,
                                u8* out_value_type, u64* out_null_count, int out_mem) {
    const bool strings = sr != nullptr;  // the string entry point
    u64 n;
    YTGPU_TRY(check_program_columns(columns, column_count, string_columns, string_count, out_mem, &n));
    if (const_bytes > YTGPU_EXPR_MAX_STRING_CONSTANT_BYTES)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "more than %u bytes of string_constants", (unsigned)YTGPU_EXPR_MAX_STRING_CONSTANT_BYTES);
    if (const_bytes && !consts) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null string_constants");
    CheckedExpr P;
    YTGPU_TRY(check_expression(columns, column_count, strings, string_count, consts, const_bytes, program, node_count, &P));
    if (out_value_type) *out_value_type = P.type;
    if (out_null_count) *out_null_count = 0;
    const bool string_result = P.type == YTGPU_TYPE_STRING;
    if (string_result) {
        if (!sr->heap_bytes) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null out_heap_bytes");
        *sr->heap_bytes = 0;
        if (n && sr->heap && (!sr->starts || !sr->lengths || !sr->null_bytemap))
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null out_starts, out_lengths or out_null_bytemap");
    } else if (n && (!out_values || !out_null_bitmap)) {
        if (strings && !sr->heap && !out_values && !out_null_bitmap) return Status{};  // a type query: nothing is evaluated
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null out_values or out_null_bitmap");
    }
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    if (n == 0) return Status{};

    StagedProgramColumns cols;
    YTGPU_TRY(cols.stage(ctx, columns, P.cols, string_columns, P.strings));
    // one upload: nodes | column views | string views | string constants | sorted IN entries | compiled patterns
    ProgramBlob blob;
    const size_t o_nodes = blob.add(P.nodes.data(), P.nodes.size() * sizeof(ExprNodeDev));
    const size_t o_cols = blob.add(cols.scalars.data(), cols.scalars.size() * sizeof(ColumnDev));
    const size_t o_strs = blob.add(cols.strings.data(), cols.strings.size() * sizeof(StringDev));
    const size_t o_const = blob.add(consts, const_bytes);
    const size_t o_list = blob.add(P.lists.data(), P.lists.size() * 8);
    const size_t o_pat = blob.add(P.patterns.data(), P.patterns.size());
    YTGPU_TRY(blob.upload(ctx));

    const u64 words = (n + 63) / 64 * 2;  // 32-bit bitmap words
    const bool host = out_mem == YTGPU_MEM_HOST;
    DevBuf<u64> tstarts, scan_sums;
    DevBuf<u32> tlengths;
    DevBuf<u8> tnull_bytes, theap;
    DevBuf<unsigned long long> result;
    InBuf<u32> dselection;
    OutBuf<u64> values;
    OutBuf<u32> nulls;
    u64* dvalues = out_values;
    u32* dnulls = reinterpret_cast<u32*>(out_null_bitmap);
    YTGPU_TRY(dselection.stage(ctx, reinterpret_cast<const u32*>(selection), words, out_mem));
    u64* dstarts = nullptr;
    u32* dlengths = nullptr;
    u8* dnull_bytes = nullptr;
    // A string result is sized in one pass and filled in a second, so its scratch depends on more than out_mem.
    if (string_result) {  // the size pass writes the caller's DEVICE outputs only when they are filled too
        const bool direct = !host && sr->heap;
        dstarts = direct ? sr->starts : nullptr;
        dlengths = direct ? sr->lengths : nullptr;
        dnull_bytes = direct ? sr->null_bytemap : nullptr;
        if (!direct) {
            YTGPU_TRY(tstarts.allocate(ctx, n));
            YTGPU_TRY(tlengths.allocate(ctx, n));
            YTGPU_TRY(tnull_bytes.allocate(ctx, n));
            dstarts = tstarts.p;
            dlengths = tlengths.p;
            dnull_bytes = tnull_bytes.p;
        }
        YTGPU_TRY(scan_sums.allocate(ctx, scan_block_count(n)));
    } else {
        YTGPU_TRY(values.prepare(ctx, out_values, n, out_mem));
        YTGPU_TRY(nulls.prepare(ctx, dnulls, words, out_mem));
        dvalues = values.p;
        dnulls = nulls.p;
    }
    YTGPU_TRY(result.allocate(ctx, 3));
    YTGPU_CUDA_TRY(cudaMemsetAsync(result.p, 0, 24, ctx->stream));

    ExprArgs A{};
    A.nodes = blob.at<ExprNodeDev>(o_nodes);
    A.node_count = (u32)P.nodes.size();
    A.columns = blob.at<ColumnDev>(o_cols);
    A.column_count = (u32)cols.scalars.size();
    A.selection = dselection.p;
    A.n = n;
    A.values = dvalues;
    A.nulls = dnulls;
    A.result = result.p;
    A.strings = blob.at<StringDev>(o_strs);
    A.string_count = (u32)cols.strings.size();
    A.mode = string_result ? kModeSize : kModeValues;
    A.max_depth = P.max_depth;
    A.max_pieces = P.max_pieces;
    A.consts = blob.at<u8>(o_const);
    A.starts = dstarts;
    A.lengths = dlengths;
    A.null_bytes = dnull_bytes;
    PredArgs Q{};
    Q.lists = blob.at<u64>(o_list);
    Q.patterns = blob.at<u8>(o_pat);
    Q.staged_list = std::min<u32>((u32)P.lists.size(), kStagedListEntries);
    Q.pattern_bytes = (u32)((P.patterns.size() + 15) & ~(size_t)15);  // staged in 16-byte units, as the blob pads them
    // shared memory in the kernel's order: nodes (16 B each), column views, string views (8-byte multiples), the stack
    // below the top; expression_kernel<true, true>: the piece stack and, 16-byte aligned, a short-value stage per warp
    static_assert(sizeof(ColumnDev) % 8 == 0 && sizeof(StringDev) % 8 == 0, "shared-memory layout");
    const size_t nodes_b = P.nodes.size() * sizeof(ExprNodeDev), cols_b = cols.scalars.size() * sizeof(ColumnDev),
                 strs_b = cols.strings.size() * sizeof(StringDev);
    const size_t stack_b = (size_t)(P.max_depth - 1) * kExprThreads * sizeof(u64);
    const u32 blocks = blocks_for(words * 32, kExprThreads, 8);  // a warp per 32-row group
    // with predicates, after everything else at a 16-byte boundary: the compiled patterns, then the head of the IN entries
    size_t smem = P.strings_kernel ? nodes_b + cols_b + strs_b + stack_b + (size_t)P.max_pieces * kExprThreads * 12 + 16 +
                                         (size_t)(kExprThreads / 32) * kStageBytes
                                   : nodes_b + cols_b + stack_b;
    if (P.predicates || P.time) {
        Q.pred_smem = (u32)((smem + 15) & ~(size_t)15);
        smem = Q.pred_smem + Q.pattern_bytes + (size_t)Q.staged_list * 8;
    }
    // the kernel of the checked program; up to 16 pieces, a 16-deep stack and the predicates' stage exceed the 48 KB default
    void (*kernel)(ExprArgs) = P.strings_kernel ? expression_kernel<true, true> : (P.conditional ? expression_kernel<false, true> : expression_kernel<false, false>);
    void (*pred_kernel)(ExprArgs, PredArgs) = P.strings_kernel ? expression_pred_kernel<true> : expression_pred_kernel<false>;
    void (*time_kernel)(ExprArgs, PredArgs, u8*) = P.strings_kernel ? expression_time_kernel<true> : expression_time_kernel<false>;
    DevBuf<u8> scratch;  // FORMAT_TIMESTAMP: a line per thread of the grid and node
    if (P.formats) YTGPU_TRY(scratch.allocate(ctx, (size_t)P.formats * blocks * kExprThreads * kFormatLine));
    auto launch = [&] {
        if (P.time) time_kernel<<<blocks, kExprThreads, smem, ctx->stream>>>(A, Q, scratch.p);
        else if (P.predicates) pred_kernel<<<blocks, kExprThreads, smem, ctx->stream>>>(A, Q);
        else kernel<<<blocks, kExprThreads, smem, ctx->stream>>>(A);
    };
    if (P.time) YTGPU_CUDA_TRY(cudaFuncSetAttribute(time_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    else if (P.predicates) YTGPU_CUDA_TRY(cudaFuncSetAttribute(pred_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    else if (P.strings_kernel) YTGPU_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    {
        KernelTimer t(ctx, KC_DECODE, string_result ? 4 : 1);
        launch();
        if (string_result)  // starts = exclusive scan of the lengths, the total into result[2]
            exclusive_scan_u64(ctx->stream, dstarts, n, scan_sums.p, reinterpret_cast<u64*>(result.p + 2));
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    unsigned long long res[3] = {0, 0, 0};  // the one host read: NULL count, error bits and the heap size
    YTGPU_CUDA_TRY(cudaMemcpyAsync(res, result.p, string_result ? 24 : 16, cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_TRY(values.download(ctx, n));
    YTGPU_TRY(nulls.download(ctx, words));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (res[1] & kErrOutOfHeap) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "a string value of an expression column leaves its heap");
    if (res[1] & kErrNonAscii)
        return make_status(YTGPU_ERR_UNSUPPORTED, "lower / upper of a value with a byte >= 0x80: Unicode case mapping is not on the GPU path");
    if (res[1] & kErrTooLong) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "a string result is longer than 2^32 - 1 bytes");
    if (res[1] & kErrMatchTooLong)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "CONTAINS / LIKE over a value of 2^32 bytes or more");
    if (res[1] & kErrTimeRange)
        return make_status(YTGPU_ERR_UNSUPPORTED, "a timestamp outside [0, 253402300799] (9999-12-31T23:59:59Z), or a week floor before "
                                                  "1970-01-05: not on the GPU path");
    if (res[1] & kErrDivZero) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "Division by zero");
    if (res[1] & kErrIntMinByMinusOne) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "Division INT_MIN by -1");
    if (out_null_count) *out_null_count = res[0];
    if (!string_result) return Status{};

    const u64 total = res[2];
    *sr->heap_bytes = total;
    if (!sr->heap) return Status{};
    if (sr->capacity < total)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "out_heap holds %llu bytes, %llu are needed", (unsigned long long)sr->capacity,
                           (unsigned long long)total);
    u8* dheap = sr->heap;
    if (host) {
        YTGPU_TRY(theap.allocate(ctx, total));
        dheap = theap.p;
    }
    A.mode = kModeFill;
    A.heap = dheap;
    {
        KernelTimer t(ctx, KC_GATHER);
        launch();
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    if (host) {
        YTGPU_TRY(copy_out(ctx, sr->heap, dheap, total, YTGPU_MEM_HOST));
        YTGPU_TRY(copy_out(ctx, sr->starts, dstarts, n * 8, YTGPU_MEM_HOST));
        YTGPU_TRY(copy_out(ctx, sr->lengths, dlengths, n * 4, YTGPU_MEM_HOST));
        YTGPU_TRY(copy_out(ctx, sr->null_bytemap, dnull_bytes, n, YTGPU_MEM_HOST));
        YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    }
    return Status{};
}

}  // namespace

extern "C" {

int ytgpu_evaluate_expression(ytgpu_context* h, const ytgpu_column_view* columns, uint32_t column_count,
                              const ytgpu_expr_node* program, uint32_t node_count, const uint8_t* selection, uint64_t* out_values,
                              uint8_t* out_null_bitmap, uint8_t* out_value_type, uint64_t* out_null_count, int out_mem,
                              ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, evaluate_expression_impl(as_context(h), columns, column_count, nullptr, 0, nullptr, 0, nullptr, program, node_count,
                                                    selection, out_values, out_null_bitmap, out_value_type, out_null_count, out_mem));
}

int ytgpu_evaluate_expression_strings(ytgpu_context* h, const ytgpu_column_view* columns, uint32_t column_count,
                                      const ytgpu_string_column* string_columns, uint32_t string_count,
                                      const uint8_t* string_constants, uint64_t string_constant_bytes, const ytgpu_expr_node* program,
                                      uint32_t node_count, const uint8_t* selection, uint64_t* out_values, uint8_t* out_null_bitmap,
                                      uint8_t* out_heap, uint64_t out_heap_capacity, uint64_t* out_starts, uint32_t* out_lengths,
                                      uint8_t* out_null_bytemap, uint64_t* out_heap_bytes, uint8_t* out_value_type,
                                      uint64_t* out_null_count, int out_mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    const StringResult sr{out_heap, out_heap_capacity, out_starts, out_lengths, out_null_bytemap, out_heap_bytes};
    return fill_error(err, evaluate_expression_impl(as_context(h), columns, column_count, string_columns, string_count, string_constants,
                                                    string_constant_bytes, &sr, program, node_count, selection, out_values,
                                                    out_null_bitmap, out_value_type, out_null_count, out_mem));
}

}  // extern "C"
