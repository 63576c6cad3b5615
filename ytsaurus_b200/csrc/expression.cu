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
#include <algorithm>
#include <cstring>
#include <vector>

#include "columnar.cuh"
#include "context.cuh"

using namespace ytgpu;

namespace {

constexpr int kExprThreads = 256;
constexpr u32 kErrDivZero = 1, kErrIntMinByMinusOne = 2;

struct ExprNodeDev {
    u8 op;
    u8 type;  // the node's result type
    u8 from;  // CAST: the operand's type
    u8 pad;
    u16 col;  // COLUMN: compact column table (referenced columns only)
    u16 pad2;
    u64 constant;
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
    unsigned long long* result;   // [0] NULL rows, [1] error bits
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

__global__ void __launch_bounds__(kExprThreads) expression_kernel(const ExprArgs A) {
    extern __shared__ __align__(16) unsigned char smem[];
    ExprNodeDev* s_nodes = reinterpret_cast<ExprNodeDev*>(smem);
    ColumnDev* s_cols = reinterpret_cast<ColumnDev*>(s_nodes + A.node_count);
    u64* s_stack = reinterpret_cast<u64*>(s_cols + A.column_count) + threadIdx.x;  // entry d of this thread: [d * kExprThreads]
    {
        const u32* src = reinterpret_cast<const u32*>(A.nodes);
        u32* dst = reinterpret_cast<u32*>(s_nodes);
        for (u32 k = threadIdx.x; k < A.node_count * (u32)(sizeof(ExprNodeDev) / 4); k += blockDim.x) dst[k] = src[k];
        src = reinterpret_cast<const u32*>(A.columns);
        dst = reinterpret_cast<u32*>(s_cols);
        for (u32 k = threadIdx.x; k < A.column_count * (u32)(sizeof(ColumnDev) / 4); k += blockDim.x) dst[k] = src[k];
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
        if (sel != 0) {
            u32 depth = 0;  // entries below the top, in s_stack
#pragma unroll 1
            for (u32 k = 0; k < A.node_count; ++k) {
                const ExprNodeDev nd = s_nodes[k];
                if (nd.op == YTGPU_EXPR_COLUMN || nd.op == YTGPU_EXPR_CONSTANT) {
                    bool nul = !live;
                    u64 v = nd.constant;
                    if (nd.op == YTGPU_EXPR_COLUMN) {
                        const ColumnDev& c = s_cols[nd.col];
                        v = scalar_value(c, i, row0, live, &nul);
                        if (c.value_type == YTGPU_TYPE_BOOLEAN) v = v != 0;
                    }
                    if (k) s_stack[depth++ * kExprThreads] = top;
                    top = nul ? 0 : v;
                    nul_stack = (nul_stack << 1) | (nul ? 1u : 0u);
                } else if (nd.op == YTGPU_EXPR_NEG || nd.op == YTGPU_EXPR_BIT_NOT || nd.op == YTGPU_EXPR_CAST) {
                    if (!(nul_stack & 1)) top = unary_op(nd.op, nd.type, nd.from, top);
                } else {
                    const u64 a = s_stack[--depth * kExprThreads], b = top;
                    const u32 nb = nul_stack & 1, na = (nul_stack >> 1) & 1;
                    u32 nr;
                    if (nd.op == YTGPU_EXPR_IF_NULL) {
                        top = na ? b : a;
                        nr = na & nb;
                    } else {
                        nr = na | nb;
                        top = nr ? 0 : binary_op(nd.op, nd.type, a, b, &err);
                    }
                    nul_stack = ((nul_stack >> 2) << 1) | nr;
                }
            }
        }
        const bool nul = !live || (nul_stack & 1);
        const u32 m = __ballot_sync(0xffffffffu, nul && i < A.n);
        if (i < A.n) A.values[i] = nul ? 0 : top;
        if (lane == 0) {
            A.nulls[w] = m;
            null_rows += (u64)__popc(m);
        }
    }
    err = __reduce_or_sync(0xffffffffu, err);
    if (lane == 0) {
        if (null_rows) atomicAdd(&A.result[0], (unsigned long long)null_rows);
        if (err) atomicOr(&A.result[1], (unsigned long long)err);
    }
}

// ---- host ----
struct CheckedExpr {
    std::vector<ExprNodeDev> nodes;
    std::vector<u32> cols;  // compact slot -> caller column
    u32 max_depth = 0;
    u8 type = 0;  // the result type
};

bool is_expr_type(u32 t) {
    return t == YTGPU_TYPE_INT64 || t == YTGPU_TYPE_UINT64 || t == YTGPU_TYPE_DOUBLE || t == YTGPU_TYPE_BOOLEAN;
}
bool is_number_type(u32 t) { return t == YTGPU_TYPE_INT64 || t == YTGPU_TYPE_UINT64 || t == YTGPU_TYPE_DOUBLE; }
bool is_integer_type(u32 t) { return t == YTGPU_TYPE_INT64 || t == YTGPU_TYPE_UINT64; }

Status check_expression(const ytgpu_column_view* columns, u32 column_count, const ytgpu_expr_node* program, u32 node_count,
                        CheckedExpr* out) {
    if (node_count == 0 || node_count > (u32)YTGPU_EXPR_MAX_NODES)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "an expression program has 1 .. %d nodes", YTGPU_EXPR_MAX_NODES);
    if (!program) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null program");
    std::vector<int> slot_of(column_count, -1);
    std::vector<u8> types;  // the type stack
    for (u32 k = 0; k < node_count; ++k) {
        const ytgpu_expr_node& N = program[k];
        ExprNodeDev d{};
        d.op = (u8)N.op;
        switch (N.op) {
            case YTGPU_EXPR_COLUMN: {
                if (N.column < 0 || (u32)N.column >= column_count)
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: column %d out of range", k, N.column);
                const u8 t = columns[N.column].value_type;
                if (!is_expr_type(t))
                    return make_status(YTGPU_ERR_UNSUPPORTED, "node %u: column %d has value type 0x%x (INT64, UINT64, DOUBLE or BOOLEAN)", k,
                                       N.column, t);
                if (slot_of[N.column] < 0) {
                    slot_of[N.column] = (int)out->cols.size();
                    out->cols.push_back((u32)N.column);
                }
                d.col = (u16)slot_of[N.column];
                d.type = t;
                types.push_back(t);
                break;
            }
            case YTGPU_EXPR_CONSTANT:
                if (!is_expr_type(N.type)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: unknown constant type 0x%x", k, N.type);
                if (N.type == YTGPU_TYPE_BOOLEAN && N.constant > 1)
                    return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: a BOOLEAN constant is 0 or 1", k);
                d.type = N.type;
                d.constant = N.constant;
                types.push_back(N.type);
                break;
            case YTGPU_EXPR_NEG:
            case YTGPU_EXPR_BIT_NOT:
            case YTGPU_EXPR_CAST: {
                if (types.empty()) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: stack underflow", k);
                const u8 t = types.back();
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
                types.back() = d.type;
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
            case YTGPU_EXPR_IF_NULL: {
                if (types.size() < 2) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: stack underflow", k);
                const u8 b = types.back();
                types.pop_back();
                const u8 a = types.back();
                if (a != b) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: operands of types 0x%x and 0x%x (CAST one of them)", k, a, b);
                const bool ok = N.op == YTGPU_EXPR_IF_NULL ? true
                              : (N.op <= YTGPU_EXPR_DIV ? is_number_type(a) : is_integer_type(a));
                if (!ok) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: op %d does not take type 0x%x", k, N.op, a);
                d.type = a;
                break;
            }
            default:
                return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: unknown op %d", k, N.op);
        }
        if (types.size() > (size_t)YTGPU_EXPR_MAX_DEPTH)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: stack deeper than %d", k, YTGPU_EXPR_MAX_DEPTH);
        out->max_depth = std::max(out->max_depth, (u32)types.size());
        out->nodes.push_back(d);
    }
    if (types.size() != 1)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "the program leaves %d values on the stack, not 1", (int)types.size());
    out->type = types[0];
    return Status{};
}

Status evaluate_expression_impl(Context* ctx, const ytgpu_column_view* columns, u32 column_count, const ytgpu_expr_node* program,
                                u32 node_count, const u8* selection, u64* out_values, u8* out_null_bitmap, u8* out_value_type,
                                u64* out_null_count, int out_mem) {
    if (column_count && !columns) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null columns");
    if (column_count == 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "no columns");
    if (out_mem != YTGPU_MEM_DEVICE && out_mem != YTGPU_MEM_HOST)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "out_mem must be YTGPU_MEM_DEVICE or YTGPU_MEM_HOST");
    const u64 n = (u64)columns[0].value_count;
    for (u32 c = 0; c < column_count; ++c)
        if (columns[c].value_count < 0 || (u64)columns[c].value_count != n)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "column %u differs in length", c);
    if (n >= (1ull << 32)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "fewer than 2^32 rows per call");
    CheckedExpr P;
    YTGPU_TRY(check_expression(columns, column_count, program, node_count, &P));
    if (out_value_type) *out_value_type = P.type;
    if (out_null_count) *out_null_count = 0;
    if (n && (!out_values || !out_null_bitmap)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null out_values or out_null_bitmap");
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    if (n == 0) return Status{};

    std::vector<StagedColumn> sc(P.cols.size());
    std::vector<ColumnDev> hc(P.cols.size());
    for (size_t k = 0; k < sc.size(); ++k) {
        YTGPU_TRY(stage_column(ctx, &columns[P.cols[k]], &sc[k]));
        hc[k] = sc[k].dev;
    }
    // one upload: nodes | column views
    const size_t nodes_b = P.nodes.size() * sizeof(ExprNodeDev), cols_b = hc.size() * sizeof(ColumnDev);
    std::vector<u8> blob(nodes_b + cols_b);
    memcpy(blob.data(), P.nodes.data(), nodes_b);
    if (cols_b) memcpy(blob.data() + nodes_b, hc.data(), cols_b);
    DevBuf<u8> dblob;
    YTGPU_TRY(dblob.allocate(ctx, blob.size()));
    YTGPU_CUDA_TRY(cudaMemcpyAsync(dblob.p, blob.data(), blob.size(), cudaMemcpyHostToDevice, ctx->stream));

    const u64 words = (n + 63) / 64 * 2;  // 32-bit bitmap words
    const bool host = out_mem == YTGPU_MEM_HOST;
    DevBuf<u64> tvalues;
    DevBuf<u32> tnulls, tselection;
    DevBuf<unsigned long long> result;
    u64* dvalues = out_values;
    u32* dnulls = reinterpret_cast<u32*>(out_null_bitmap);
    const u32* dselection = reinterpret_cast<const u32*>(selection);
    if (host) {
        YTGPU_TRY(tvalues.allocate(ctx, n));
        YTGPU_TRY(tnulls.allocate(ctx, words));
        dvalues = tvalues.p;
        dnulls = tnulls.p;
        if (selection) {
            YTGPU_TRY(tselection.allocate(ctx, words));
            YTGPU_TRY(copy_in(ctx, tselection.p, selection, words * 4, YTGPU_MEM_HOST));
            dselection = tselection.p;
        }
    }
    YTGPU_TRY(result.allocate(ctx, 2));
    YTGPU_CUDA_TRY(cudaMemsetAsync(result.p, 0, 16, ctx->stream));

    ExprArgs A{};
    A.nodes = reinterpret_cast<const ExprNodeDev*>(dblob.p);
    A.node_count = (u32)P.nodes.size();
    A.columns = reinterpret_cast<const ColumnDev*>(dblob.p + nodes_b);
    A.column_count = (u32)hc.size();
    A.selection = dselection;
    A.n = n;
    A.values = dvalues;
    A.nulls = dnulls;
    A.result = result.p;
    // shared memory in the kernel's order: nodes (16 B each), column views (8-byte multiple), the stack below the top
    static_assert(sizeof(ColumnDev) % 8 == 0, "shared-memory layout");
    const size_t smem = nodes_b + cols_b + (size_t)(P.max_depth - 1) * kExprThreads * sizeof(u64);
    const u32 blocks = (u32)std::max<u64>(1, std::min<u64>((words * 32 + kExprThreads - 1) / kExprThreads, (u64)kNumSms * 8));
    {
        KernelTimer t(ctx, KC_DECODE);
        expression_kernel<<<blocks, kExprThreads, smem, ctx->stream>>>(A);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    unsigned long long res[2] = {0, 0};  // the one host read: NULL count and error bits
    YTGPU_CUDA_TRY(cudaMemcpyAsync(res, result.p, 16, cudaMemcpyDeviceToHost, ctx->stream));
    if (host) {
        YTGPU_TRY(copy_out(ctx, out_values, dvalues, n * 8, YTGPU_MEM_HOST));
        YTGPU_TRY(copy_out(ctx, out_null_bitmap, dnulls, words * 4, YTGPU_MEM_HOST));
    }
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (res[1] & kErrDivZero) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "Division by zero");
    if (res[1] & kErrIntMinByMinusOne) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "Division INT_MIN by -1");
    if (out_null_count) *out_null_count = res[0];
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
    return fill_error(err, evaluate_expression_impl(as_context(h), columns, column_count, program, node_count, selection, out_values,
                                                    out_null_bitmap, out_value_type, out_null_count, out_mem));
}

}  // extern "C"
