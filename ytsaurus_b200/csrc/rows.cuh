// rows.cuh — key extraction / normalisation and row gather kernels.
#pragma once

#include "context.cuh"
#include "keys.cuh"
#include "radix_sort.cuh"

namespace ytgpu {

struct ChunkPtrs {
    u64* p[kMaxKeyChunks];
};

// Fixed rows -> normalised key chunks (fast path for a single 8-byte scalar key).
// When `hist` is non-null and the key is a single 8-byte scalar, the digit histogram of chunk 0 is
// accumulated in the same pass over the table (*hist_done = true); otherwise the sort builds it.
Status normalize_fixed_rows(Context* ctx, const KeyLayout& L, const u8* rows_dev, u64 n, u32 row_bytes,
                            const ChunkPtrs& chunks, u32* hist = nullptr, bool* hist_done = nullptr);

// Rowset values -> normalised key chunks; type / width violations land in the context error word.
Status normalize_rowset(Context* ctx, const KeyLayout& L, const ytgpu_value* values_dev, u32 value_count,
                        const u8* heap_dev, u64 n, const ChunkPtrs& chunks);

// Maximum string length per key column (for width == 0), result in host array max_len[ncols].
Status measure_string_widths(Context* ctx, const ytgpu_sort_spec* spec, const ytgpu_value* values_dev,
                             u32 value_count, u64 n, u32* max_len_host);

// out[j] = in[perm[j]] for rows of row_bytes (multiple of 16) bytes.
Status gather_rows(Context* ctx, const u8* in_dev, const PermRef& perm, u8* out_dev, u64 n, u32 row_bytes);

// chunk[i] = (u64)(u32)index[i]: a partition index array as a radix-sort key chunk.
Status widen_index(Context* ctx, const i32* index_dev, u64 n, u64* chunk_dev);

// The whole fixed-row sort (capi_sort.cu): key extraction -> radix sort -> row gather / permutation.  Used by the
// C ABI entry point and by the in-box shuffle's local sort.
Status sort_fixed_rows_impl(Context* ctx, const ytgpu_fixed_rows_view* in, const ytgpu_sort_spec* spec, u8* out_rows,
                            u32* out_perm, int out_mem);

}  // namespace ytgpu
