// program.cuh — what the two postfix-program evaluators, WHERE programs (filter.cu) and computed columns (expression.cu),
// do alike around their interpreters: the checks on their input columns, the compact tables of the columns a program
// references, staging those columns on the device, the one upload of a call's program and tables, and the comparison
// rule.  The IN-list and pattern formats are in strings.cuh.  TU-local (anonymous namespace), like strings.cuh.
#pragma once

#include <cstring>
#include <vector>

#include "columnar.cuh"
#include "context.cuh"
#include "strings.cuh"

namespace {

using namespace ytgpu;

// Whether c, a three-way comparison's result, satisfies the ytgpu_cmp_op op.
__device__ __forceinline__ bool cmp_holds(u32 op, int c) {
    switch (op) {
        case YTGPU_CMP_LT: return c < 0;
        case YTGPU_CMP_LE: return c <= 0;
        case YTGPU_CMP_GT: return c > 0;
        case YTGPU_CMP_GE: return c >= 0;
        case YTGPU_CMP_EQ: return c == 0;
        default: return c != 0;
    }
}

// The value types a scalar column of a program may have.
inline bool is_scalar_type(u32 t) {
    return t == YTGPU_TYPE_INT64 || t == YTGPU_TYPE_UINT64 || t == YTGPU_TYPE_DOUBLE || t == YTGPU_TYPE_BOOLEAN;
}

// The input columns of an evaluator call: non-null arrays, at least one column, one row count for all of them (*n),
// readable string columns, a known out_mem and fewer than 2^32 rows.  An empty string column may have null starts and
// lengths: nothing reads them.
Status check_program_columns(const ytgpu_column_view* columns, u32 column_count, const ytgpu_string_column* string_columns,
                             u32 string_count, int out_mem, u64* n) {
    if ((column_count && !columns) || (string_count && !string_columns)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null columns");
    if (column_count + (u64)string_count == 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "no columns");
    if (out_mem != YTGPU_MEM_DEVICE && out_mem != YTGPU_MEM_HOST)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "out_mem must be YTGPU_MEM_DEVICE or YTGPU_MEM_HOST");
    *n = column_count ? (u64)columns[0].value_count : string_columns[0].row_count;
    for (u32 c = 0; c < column_count; ++c)
        if (columns[c].value_count < 0 || (u64)columns[c].value_count != *n)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "column %u differs in length", c);
    for (u32 s = 0; s < string_count; ++s) {
        const ytgpu_string_column& S = string_columns[s];
        if (S.row_count != *n) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string column %u differs in length", s);
        if ((S.heap_bytes && !S.heap) || (*n && (!S.starts || !S.lengths)))
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string column %u: null heap, starts or lengths", s);
        if (S.mem != YTGPU_MEM_DEVICE && S.mem != YTGPU_MEM_HOST)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string column %u: mem must be YTGPU_MEM_DEVICE or YTGPU_MEM_HOST", s);
    }
    if (*n >= (1ull << 32)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "fewer than 2^32 rows per call");
    return Status{};
}

// The compact table of the columns a program references: slot(c) numbers caller column c in the order of first reference.
struct SlotMap {
    std::vector<int> slot_of;  // caller column -> compact slot (-1: not referenced)
    std::vector<u32> cols;     // compact slot -> caller column
    u16 slot(u32 c) {
        if (c >= slot_of.size()) slot_of.resize(c + 1, -1);
        if (slot_of[c] < 0) {
            slot_of[c] = (int)cols.size();
            cols.push_back(c);
        }
        return (u16)slot_of[c];
    }
};

// The referenced columns on the device in compact order (HOST inputs uploaded): their views and the buffers behind them.
struct StagedProgramColumns {
    std::vector<StagedColumn> scalar_bufs;
    std::vector<ColumnDev> scalars;
    std::vector<StagedStrings> string_bufs;
    std::vector<StringDev> strings;
    Status stage(Context* ctx, const ytgpu_column_view* columns, const SlotMap& scalar_slots, const ytgpu_string_column* string_columns,
                 const SlotMap& string_slots) {
        scalar_bufs = std::vector<StagedColumn>(scalar_slots.cols.size());
        scalars.resize(scalar_bufs.size());
        for (size_t k = 0; k < scalars.size(); ++k) {
            YTGPU_TRY(stage_column(ctx, &columns[scalar_slots.cols[k]], &scalar_bufs[k]));
            scalars[k] = scalar_bufs[k].dev;
        }
        string_bufs = std::vector<StagedStrings>(string_slots.cols.size());
        strings.resize(string_bufs.size());
        for (size_t k = 0; k < strings.size(); ++k) {
            YTGPU_TRY(stage_strings(ctx, string_columns[string_slots.cols[k]], &string_bufs[k]));
            strings[k] = string_bufs[k].dev;
        }
        return Status{};
    }
};

// A call's read-only inputs in one device buffer and one copy: add() places a section at a 16-byte boundary, padded to
// whole 16-byte units (a kernel may stage it in those units), and at(offset) is its device address after upload().
struct ProgramBlob {
    std::vector<u8> host;
    DevBuf<u8> dev;
    size_t add(const void* p, size_t bytes) {
        const size_t off = host.size();
        host.resize(off + ((bytes + 15) & ~(size_t)15), 0);
        if (bytes) memcpy(host.data() + off, p, bytes);
        return off;
    }
    Status upload(Context* ctx) {
        YTGPU_TRY(dev.allocate(ctx, host.size()));
        YTGPU_CUDA_TRY(cudaMemcpyAsync(dev.p, host.data(), host.size(), cudaMemcpyHostToDevice, ctx->stream));
        return Status{};
    }
    template <class T>
    const T* at(size_t off) const {
        return reinterpret_cast<const T*>(dev.p + off);
    }
};

}  // namespace
