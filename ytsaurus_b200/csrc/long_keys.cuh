// long_keys.cuh — rowset sort by keys whose fixed-width normalised form does not fit in kMaxKeyChunks chunks.
#pragma once

#include "context.cuh"
#include "keys.cuh"

namespace ytgpu {

// Type / schema / declared-width errors of every key value, into the context error word (check_device_errors).
Status check_long_keys(Context* ctx, const KeyLayout& L, const ytgpu_value* values_dev, u32 value_count, u64 n);

// Stable sort of the rows by the width-free key words of keys.cuh, by MSD refinement rounds: perm_dev[j] = row at
// position j.  Records the rounds in ctx->last_sort_refine_rounds / last_sort_refine_rows.  n < 2^30.
Status long_key_sort(Context* ctx, const KeyLayout& L, const ytgpu_value* values_dev, u32 value_count, const u8* heap_dev,
                     u64 n, u32* perm_dev);

}  // namespace ytgpu
