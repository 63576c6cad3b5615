// radix_sort.cuh — stable LSD radix sort of (multi-chunk u64 key, u32 row index) on one GPU.
//
// Single-pass-per-digit ("onesweep") design: one upfront histogram of every 8-bit digit of every key
// chunk, then per digit ONE kernel that reads each (key, index) pair once and writes it once, using
// decoupled look-back over per-tile digit counts for the global scatter offsets.  Digits whose
// histogram has a single non-empty bin are skipped (a device-side plan records which buffers the
// surviving passes ping-pong between; single-chunk sorts of >= 2^18 rows read it back once to launch
// only the active passes).
//
// Algorithmic HBM bytes per row: 8*C (histogram) + sum over active passes of 2*(8+4)
// (first pass of a round reads no index when the permutation is still the identity).  Packed sorts
// (SortPlan::packed) move one 8-byte word per row instead: 8 + 8 per pass, 8 + 4 (+ 4) in the last.
#pragma once

#include "context.cuh"

namespace ytgpu {

constexpr int kMaxKeyChunks = 32;   // normalised keys up to 256 bytes
constexpr int kRadixBits = 8;
constexpr int kRadix = 1 << kRadixBits;
constexpr int kPassesPerChunk = 8;

struct PassDesc {
    u8 active;
    u8 src_kind;  // 0: keys straight from the chunk, identity permutation; 1: keys gathered from the chunk
                  // through the current permutation; 2: keys from a work buffer
    u8 key_src;   // work buffer 0/1 (src_kind == 2)
    u8 idx_src;   // permutation buffer 0/1 (src_kind != 0)
    u8 key_dst;
    u8 idx_dst;
    u8 last;      // final pass of the sort: only the permutation is consumed, the key write is skipped
    u8 write_prefix;  // packed hybrid schedule, last pass: also writes the u32 prefixes to idx[idx_dst ^ 1]
};

struct SortPlan {
    PassDesc pass[kMaxKeyChunks * kPassesPerChunk];
    u32 final_idx;  // 0/1 = permutation buffer holding the result, 2 = identity
    u32 active_passes;
    // Hybrid schedule for single-chunk keys (see radix_sort.cu): `pass` then only covers the most significant
    // active digits and the hybrid tail orders the runs of equal prefixes.  When the tail finds clustered keys the
    // host sorts the chunk again with the plain schedule, which replaces this plan.
    u32 hybrid;
    u32 hybrid_shift;   // keys with equal (key >> hybrid_shift) form one run after the hybrid passes
    u32 final_key_a;    // work buffer holding the keys after the hybrid passes
    u32 final_key;      // keep_keys sorts: buffer holding the sorted keys (0/1, 2 = the chunk itself)
    // Packed format (single-chunk sorts of >= 2^18 rows whose scheduled digits fit in 32 bits, not keep_keys): the
    // passes of `pass` move one u64 per row, (prefix << 32) | row index, where prefix byte k is the key digit of the k-th
    // scheduled digit (least significant first).  The last pass writes the row indices to idx[final_idx] and, for the
    // hybrid schedule, the prefixes to idx[final_idx ^ 1].
    u32 packed;
    u32 prefix_sel;   // __byte_perm selector over the key's two halves: nibble k = key digit of prefix byte k
    u32 prefix_mask;  // prefix bytes in use
    // Packed hybrid schedule: 8 when the passes sort prefix bytes 1-3 only and leave byte 0 to the hybrid tail, else 0.
    // Rows with equal (prefix >> run_shift) form one run for the tail.
    u32 run_shift;
};

// Buffer holding the sorted keys of a keep_keys sort (0/1 = work buffer, 2 = the input chunk: no pass moved data).
__device__ __forceinline__ u32 plan_final_key(const SortPlan* plan) {
    return plan->hybrid ? plan->final_key_a : plan->final_key;
}

// Result handle: the permutation lives in idx[plan->final_idx] (or is the identity).
struct PermRef {
    const SortPlan* plan = nullptr;  // device
    const u32* idx[2] = {nullptr, nullptr};
};

__device__ __forceinline__ u32 perm_at(const SortPlan* plan, const u32* a, const u32* b, u64 i) {
    u32 f = plan->final_idx;
    return f == 2 ? (u32)i : (f == 0 ? a[i] : b[i]);
}

// Fixed rows the sort may move itself: out[j] = rows[perm[j]].
struct RowGatherRequest {
    const u8* rows = nullptr;  // device, row_bytes apart; nullptr: no request
    u8* out = nullptr;         // device, n * row_bytes
    u32 row_bytes = 0;         // a multiple of 16
    bool want_perm = true;     // the caller reads the permutation as well
};

// Serves ONE sort of one set of keys: the sort records state in it (hist_precomputed, and no_hybrid after a re-sort of
// clustered keys), so a second sort of different keys needs a fresh SortScratch.
struct SortScratch {
    DevBuf<u64> keys[2];
    DevBuf<u32> idx[2];
    DevBuf<u32> hist;      // [chunks*8][256] digit counts
    DevBuf<u32> offsets;   // [chunks*8][256] exclusive digit offsets (plan_kernel)
    DevBuf<u32> status;    // [8][tiles][256] look-back words for one round
    DevBuf<u32> counters;  // [chunks*8] dynamic tile counters
    DevBuf<SortPlan> plan;
    bool hist_precomputed = false;  // `hist` holds the keys' counts: filled by the caller (see prepare_histogram /
                                    // hist_accumulate) or by the sort itself, so that a re-sort of the keys reuses them
    bool keep_keys = false;         // the final pass writes the keys too: keys[plan_final_key()] holds them sorted
    bool no_hybrid = false;         // always the plain schedule (side sorts, re-sorts of clustered keys)
    // The three-pass packed hybrid schedule moves the requested rows in its tail and sets rows_gathered; every other
    // schedule leaves the gather to the caller.  With rows_gathered and !gather.want_perm the permutation is NOT complete.
    RowGatherRequest gather;
    bool rows_gathered = false;
};

// Shared-memory digit histogram of one key chunk: 8 digits x 256 bins.  Warp-uniform digits (constant
// high bytes, duplicated keys) are detected with one REDUX per half word and counted with a single add
// per warp instead of 32 same-address atomics.  Call with all 32 lanes of the warp.
__device__ __forceinline__ void hist_accumulate(u32* sh, u64 key, bool valid) {
    const bool all_valid = __all_sync(0xffffffffu, valid);
    u32 diff_lo = 0xffffffffu, diff_hi = 0xffffffffu;
    u64 k0 = 0;
    if (all_valid) {
        k0 = __shfl_sync(0xffffffffu, key, 0);
        u64 x = key ^ k0;
        diff_lo = __reduce_or_sync(0xffffffffu, (u32)x);
        diff_hi = __reduce_or_sync(0xffffffffu, (u32)(x >> 32));
    }
    const u64 diff = ((u64)diff_hi << 32) | diff_lo;
    const u32 lane = threadIdx.x & 31;
#pragma unroll
    for (int p = 0; p < kPassesPerChunk; ++p) {
        if (((diff >> (8 * p)) & 0xff) == 0) {
            if (lane == 0) atomicAdd(&sh[p * kRadix + (u32)((k0 >> (8 * p)) & 0xff)], 32u);
        } else if (valid) {
            atomicAdd(&sh[p * kRadix + (u32)((key >> (8 * p)) & 0xff)], 1u);
        }
    }
}

// Allocates and zeroes scratch->hist for `nchunks` chunks so that a key-producing kernel can fill chunk
// c's histogram at hist.p + c*8*256 (then set scratch->hist_precomputed).
Status prepare_histogram(Context* ctx, int nchunks, SortScratch* scratch);

// chunks: host array of `nchunks` device pointers, chunk 0 = most significant 8 key bytes.
// n < 2^30 (look-back words carry 30-bit counts).
Status radix_sort_chunks(Context* ctx, const u64* const* chunks, int nchunks, u64 n, SortScratch* scratch,
                         PermRef* out);

// Stable sort by a multi-chunk key.  One chunk: radix_sort_chunks.  Several chunks (composite / string keys): instead
// of one LSD pass per active byte of the whole key, the 8 MOST SIGNIFICANT ACTIVE bytes are packed into one synthetic
// 64-bit "prefix chunk", that chunk is sorted with the single-chunk machinery (hybrid schedule included), and rows whose
// prefix chunks tie are ordered by their full keys (short runs) — when a long run of equal prefixes mixes different keys
// the complete LSD schedule over all chunks runs instead.  Synchronises the stream once (multi-chunk keys only).
// chunk_hist_done: scratch->hist already holds the raw digit counts of every chunk.
Status radix_sort_keys(Context* ctx, const u64* const* chunks, int nchunks, u64 n, SortScratch* scratch, PermRef* out);

// Writes the permutation as a plain u32[n] device array.
Status materialize_perm(Context* ctx, const PermRef& perm, u64 n, u32* dst_dev);

}  // namespace ytgpu
