// strings.cuh — a flat string column (ytgpu_string_column) on the device: bounds-checked value access, QL string order
// and the upload of HOST columns.  Shared by the string aggregates of groupby_multi.cu and the WHERE evaluator of
// filter.cu.  Everything is TU-local (anonymous namespace) so several .cu files may include it.
#pragma once

#include "common.cuh"
#include "context.cuh"
#include "keys.cuh"

namespace {

using namespace ytgpu;

struct StringDev {
    const u8* heap;
    u64 heap_bytes;
    const u64* starts;
    const u32* lengths;
    const u8* nulls;  // nullable bytemap
    u32 present;      // 0: the argument is a scalar ColumnDev
};

// Value i of a string argument: false for NULL; a value that leaves the heap sets the error bit and counts as absent, so
// no later read goes outside the heap.
__device__ __forceinline__ bool string_at(const StringDev& c, u64 i, ytgpu_value* v, u32* bad) {
    if (c.nulls && c.nulls[i]) return false;
    const u64 s = c.starts[i];
    const u32 l = c.lengths[i];
    if (s > c.heap_bytes || (u64)l > c.heap_bytes - s) {
        *bad = 1;
        return false;
    }
    v->type = YTGPU_TYPE_STRING;
    v->length = l;
    v->data = s;
    return true;
}

__device__ __forceinline__ ytgpu_value string_of(const StringDev& c, u64 row) {
    ytgpu_value v{};
    v.type = YTGPU_TYPE_STRING;
    v.length = c.lengths[row];
    v.data = c.starts[row];
    return v;
}

// QL string order through the width-free key words of keys.cuh (a one-column, required, ascending String key): the order
// the long-key sort and the ordered partitioner already use.  Words are prefix-free, so the first differing word decides.
// Two-heap form: a's bytes live in heap_a, b's in heap_b (a column value against a constant of the caller's buffer).
__device__ __forceinline__ int string_compare2(const u8* heap_a, const ytgpu_value& a, const u8* heap_b, const ytgpu_value& b) {
    KeyColLayout L{};
    L.type = YTGPU_TYPE_STRING;
    const u32 na = key_string_blocks(a.length), nb = key_string_blocks(b.length);
    const u32 nw = na < nb ? na : nb;
    for (u32 w = 0; w < nw; ++w) {
        const u64 x = key_col_word(L, a, heap_a, w), y = key_col_word(L, b, heap_b, w);
        if (x != y) return x < y ? -1 : 1;
    }
    return 0;
}

__device__ __forceinline__ int string_compare(const u8* heap, const ytgpu_value& a, const ytgpu_value& b) {
    return string_compare2(heap, a, heap, b);
}

// A string column on the device (HOST inputs are uploaded).
struct StagedStrings {
    StringDev dev{};
    DevBuf<u8> heap, nulls;
    DevBuf<u64> starts;
    DevBuf<u32> lengths;
};

Status stage_strings(Context* ctx, const ytgpu_string_column& c, StagedStrings* s) {
    StringDev& d = s->dev;
    d.heap_bytes = c.heap_bytes;
    d.present = 1;
    if (c.mem != YTGPU_MEM_HOST) {
        d.heap = c.heap;
        d.starts = c.starts;
        d.lengths = c.lengths;
        d.nulls = c.null_bytemap;
        return Status{};
    }
    const u64 n = c.row_count;
    YTGPU_TRY(s->heap.allocate(ctx, c.heap_bytes));
    YTGPU_TRY(copy_in(ctx, s->heap.p, c.heap, c.heap_bytes, YTGPU_MEM_HOST));
    YTGPU_TRY(s->starts.allocate(ctx, n));
    YTGPU_TRY(copy_in(ctx, s->starts.p, c.starts, n * 8, YTGPU_MEM_HOST));
    YTGPU_TRY(s->lengths.allocate(ctx, n));
    YTGPU_TRY(copy_in(ctx, s->lengths.p, c.lengths, n * 4, YTGPU_MEM_HOST));
    d.heap = s->heap.p;
    d.starts = s->starts.p;
    d.lengths = s->lengths.p;
    d.nulls = nullptr;
    if (c.null_bytemap) {
        YTGPU_TRY(s->nulls.allocate(ctx, n));
        YTGPU_TRY(copy_in(ctx, s->nulls.p, c.null_bytemap, n, YTGPU_MEM_HOST));
        d.nulls = s->nulls.p;
    }
    return Status{};
}

}  // namespace
