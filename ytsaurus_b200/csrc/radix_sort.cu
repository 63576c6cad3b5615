// radix_sort.cu — onesweep LSD radix sort core (see radix_sort.cuh).
//
// Replaces the comparison sorts of the reference's sort jobs:
//   std::sort over row pointers      yt/yt/ytlib/table_client/sorting_reader.cpp:179-187
//   10k-bucket std::sort + heap merge yt/yt/ytlib/table_client/partition_sort_reader.cpp:461-529
// with a stable radix sort over order-preserving normalised keys (keys.cuh).
#include <algorithm>
#include <utility>
#include <vector>

#include "radix_sort.cuh"
#include "rows.cuh"

namespace ytgpu {
namespace {

constexpr int kSortThreads = 256;  // one thread per digit bin in the tile's digit phase

constexpr u32 kFlagPartial = 1u << 30;
constexpr u32 kFlagInclusive = 2u << 30;
constexpr u32 kValueMask = (1u << 30) - 1;

// ---------------------------------------------------------------------------------------------
// Upfront histogram of all 8 digits of one key chunk.  Algorithmic traffic: 8 B per row (read).
// Warp-uniform digits (constant high bytes, duplicated keys) are detected with one REDUX per half
// word and counted with a single shared-memory add per warp instead of 32 same-address atomics.
// ---------------------------------------------------------------------------------------------
constexpr int kHistThreads = 512;
constexpr int kHistItems = 4;

__global__ void __launch_bounds__(kHistThreads) histogram_kernel(const u64* __restrict__ keys, u64 n,
                                                                 u32* __restrict__ hist) {
    __shared__ u32 sh[kPassesPerChunk * kRadix];
    for (int i = threadIdx.x; i < kPassesPerChunk * kRadix; i += kHistThreads) sh[i] = 0;
    __syncthreads();

    const u64 stride = (u64)gridDim.x * kHistThreads * kHistItems;
    for (u64 base = (u64)blockIdx.x * kHistThreads * kHistItems; base < n; base += stride) {
        u64 key[kHistItems];
        bool valid[kHistItems];
#pragma unroll
        for (int k = 0; k < kHistItems; ++k) {
            u64 i = base + (u64)k * kHistThreads + threadIdx.x;
            valid[k] = i < n;
            key[k] = valid[k] ? ld_stream_u64(keys + i) : 0;
        }
#pragma unroll
        for (int k = 0; k < kHistItems; ++k) hist_accumulate(sh, key[k], valid[k]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kPassesPerChunk * kRadix; i += kHistThreads) {
        u32 c = sh[i];
        if (c) atomicAdd(&hist[i], c);
    }
}

// ---------------------------------------------------------------------------------------------
// Plan: turns the counts into exclusive digit offsets, finds skippable digits, and fixes the buffer
// ping-pong schedule for every (chunk, digit) pass.  One block of 256 threads.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ u32 block_exclusive_scan_256(u32 v, u32* s_warp_tot) {
    const u32 lane = lane_id(), warp = threadIdx.x >> 5;
    u32 inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        u32 t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= (u32)o) inc += t;
    }
    if (lane == 31) s_warp_tot[warp] = inc;
    __syncthreads();
    u32 wp = 0;
#pragma unroll
    for (int w = 0; w < 8; ++w) wp += (w < (int)warp) ? s_warp_tot[w] : 0;
    __syncthreads();
    return inc - v + wp;
}

// Builds the ping-pong schedule over the passes listed in `sel` (execution order).  Returns the final
// permutation buffer (2 = identity) and reports the final key buffer and the last scheduled pass.
__device__ void build_schedule(PassDesc* descs, const int* sel, int nsel, bool mark_last, u32* final_idx, u32* final_key) {
    u32 cur_idx = 2, cur_key = 2;
    int last = -1;
    for (int k = 0; k < nsel; ++k) {
        PassDesc d{};
        d.active = 1;
        d.src_kind = cur_key == 2 ? (cur_idx == 2 ? 0 : 1) : 2;
        d.key_src = (u8)(cur_key & 1);
        d.idx_src = (u8)(cur_idx & 1);
        d.key_dst = cur_key == 2 ? 0 : (u8)(cur_key ^ 1);
        d.idx_dst = cur_idx == 2 ? 0 : (u8)(cur_idx ^ 1);
        cur_key = d.key_dst;
        cur_idx = d.idx_dst;
        descs[sel[k]] = d;
        last = sel[k];
    }
    if (mark_last && last >= 0) descs[last].last = 1;  // only the permutation is consumed: skip the key write
    *final_idx = cur_idx;
    *final_key = cur_key;
}

// allow_packed: single-chunk sort of >= kHybridMinRows rows that only consumes the permutation.
__global__ void __launch_bounds__(256) plan_kernel(const u32* hist, u32* offsets, int nchunks, u32 n, SortPlan* plan, int allow_hybrid,
                                                   int keep_keys, int allow_packed) {
    __shared__ u32 s_warp_tot[8];
    __shared__ u8 s_active[kMaxKeyChunks * kPassesPerChunk];
    __shared__ u8 s_skewed[kPassesPerChunk];
    const int total = nchunks * kPassesPerChunk;
    for (int rp = 0; rp < total; ++rp) {
        u32 c = hist[rp * kRadix + threadIdx.x];
        int full = __syncthreads_or(c == n);
        // a bin with more than twice its uniform share: > 2 n / 256 rows (see the three-pass schedule below)
        const int skewed = nchunks == 1 ? __syncthreads_or(c > (n >> 7)) : 0;
        u32 ex = block_exclusive_scan_256(c, s_warp_tot);
        offsets[rp * kRadix + threadIdx.x] = ex;
        if (threadIdx.x == 0) {
            s_active[rp] = !full;
            if (nchunks == 1) s_skewed[rp] = (u8)skewed;
        }
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    for (int rp = 0; rp < total; ++rp) plan->pass[rp] = PassDesc{};
    plan->hybrid = plan->hybrid_shift = plan->final_key_a = 0;
    plan->final_key = 2;
    plan->packed = plan->prefix_sel = plan->prefix_mask = plan->run_shift = 0;
    u32 final_key = 2;
    if (nchunks == 1) {
        int act[kPassesPerChunk], m = 0;
        for (int p = 0; p < kPassesPerChunk; ++p)
            if (s_active[p]) act[m++] = p;
        // Hybrid: sort by the `need` most significant active digits only, where 256^need >= 16 n keeps the
        // expected share of rows in runs of equal prefixes small; worth it when it saves >= 2 passes.
        int need = 1;
        unsigned long long span = 256;
        while (span < 16ull * n && need < kPassesPerChunk) { span <<= 8; ++need; }
        const bool hybrid = allow_hybrid && m >= need + 2;
        const int* sched = hybrid ? act + (m - need) : act;  // scheduled digits, least significant first
        const int t = hybrid ? need : m;
        const bool packed = allow_packed && t >= 1 && t <= 4;
        // Three of four: prefix byte 0 is in every packed word already, so the passes sort bytes 1-3 only and
        // tie_fix_runs_kernel orders each run of equal 24-bit prefixes by the whole prefix (and the full key where
        // prefixes tie).  n <= 2^27 keeps the mean run at <= 8 rows.  A sorted digit with a bin of more than twice its
        // uniform share means clustered keys, whose long runs would mix different keys: those keep the fourth pass.
        // (For uniform keys the largest of 256 bins of >= 2^20 rows is within a few percent of n / 256.)
        bool skip_byte0 = hybrid && packed && need == 4 && n <= (1u << 27);
        for (int k = 1; k < need && skip_byte0; ++k) skip_byte0 = !s_skewed[sched[k]];
        const int skip = skip_byte0 ? 1 : 0;
        if (hybrid) {
            build_schedule(plan->pass, sched + skip, need - skip, packed, &plan->final_idx, &final_key);
            plan->hybrid = 1;
            plan->hybrid_shift = 8u * (u32)sched[0];
            plan->final_key_a = plan->pass[act[m - 1]].key_dst;
            plan->active_passes = (u32)(need - skip);
        } else {
            build_schedule(plan->pass, act, m, !keep_keys, &plan->final_idx, &plan->final_key);
            plan->active_passes = (u32)m;
        }
        if (packed) {
            // prefix byte k = digit sched[k]; active digits need not be adjacent, so this is a byte selection, not a shift
            u32 sel = 0;
            for (int k = 0; k < t; ++k) sel |= (u32)sched[k] << (4 * k);
            plan->packed = 1;
            plan->prefix_sel = sel;
            plan->prefix_mask = t == 4 ? 0xffffffffu : (1u << (8 * t)) - 1;
            plan->pass[sched[t - 1]].write_prefix = hybrid ? 1 : 0;
            plan->run_shift = 8u * (u32)skip;
        }
        return;
    }
    // multi-chunk keys: chunks from least to most significant, eight digits each, one continuous ping-pong
    u32 cur_idx = 2, active = 0;
    int last_rp = -1;
    for (int r = nchunks - 1; r >= 0; --r) {
        u32 cur_key = 2;  // the chunk itself
        for (int p = 0; p < kPassesPerChunk; ++p) {
            int rp = r * kPassesPerChunk + p;
            if (!s_active[rp]) continue;
            PassDesc d{};
            d.active = 1;
            d.src_kind = cur_key == 2 ? (cur_idx == 2 ? 0 : 1) : 2;
            d.key_src = (u8)(cur_key & 1);
            d.idx_src = (u8)(cur_idx & 1);
            d.key_dst = cur_key == 2 ? 0 : (u8)(cur_key ^ 1);
            d.idx_dst = cur_idx == 2 ? 0 : (u8)(cur_idx ^ 1);
            cur_key = d.key_dst;
            cur_idx = d.idx_dst;
            ++active;
            last_rp = rp;
            plan->pass[rp] = d;
        }
    }
    if (last_rp >= 0) plan->pass[last_rp].last = 1;
    plan->final_idx = cur_idx;
    plan->active_passes = active;
}

// After the hybrid passes the (key, index) pairs are ordered by the top digits and, inside a run of equal
// top digits, still in input order.  tie_fix_kernel:
//   * runs of <= kMaxTieRun equal prefixes: the run-start thread orders them by the full key (stable insertion sort;
//     runs are 2-3 rows long when the keys spread over the prefix space);
//   * longer runs are only REGISTERED (the element 32 places into the run appends the run's start to a list), and
//     every warp stores which of its 32 positions hold "same prefix as the left neighbour, different key" — a long run of
//     EQUAL keys (duplicates, "maniac" keys) has no such position and is already in its final stable order.
// classify_long_runs_kernel then finds each long run's end and looks for a marked position inside it: runs that mix
// different keys go to the mixed list.  The host reads the summary once and either is done, re-sorts the few mixed runs
// in a side buffer (sort_mixed_runs), or — clustered keys: many / very long mixed runs — sorts the chunk again with the
// plain schedule.
constexpr int kMaxTieRun = 32;
constexpr u32 kMixedCap = 16384;       // mixed long runs handled individually; more = clustered keys = complete schedule
constexpr u64 kHybridMinRows = 1u << 18;  // smaller sorts are launch bound: plain schedule, no host round trip

struct MixedRun {
    u32 s, e;
};
struct HybridSummary {
    u32 hybrid, final_idx, final_key;
    u32 long_count, mixed_count;
    unsigned long long mixed_elems;
};

// Sorted words the hybrid tail reads: the prefix-sorted keys (pair format; prefix = word >> hybrid_shift) or the u32
// prefixes the last packed pass wrote (prefix = word >> run_shift).  Full keys: the word itself, or chunk[idx[j]].
template <bool PACKED>
struct TailWords {
    const u64* keys;
    const u32* pre;
    u32 shift;
    __device__ __forceinline__ TailWords(const SortPlan* plan, const u64* keys0, const u64* keys1, const u32* idx0, const u32* idx1) {
        keys = plan->final_key_a ? keys1 : keys0;
        pre = plan->final_idx ? idx0 : idx1;
        shift = PACKED ? plan->run_shift : plan->hybrid_shift;
    }
    __device__ __forceinline__ u64 operator[](u32 j) const { return PACKED ? (u64)pre[j] : keys[j]; }
};

template <bool PACKED>
__global__ void __launch_bounds__(256) tie_fix_kernel(SortPlan* plan, const u64* __restrict__ chunk, u64* keys0, u64* keys1, u32* idx0,
                                                      u32* idx1, u32 n, u32* __restrict__ mixedmask, u32* __restrict__ longlist,
                                                      HybridSummary* sum) {
    if (!plan->hybrid) return;
    const TailWords<PACKED> words(plan, keys0, keys1, idx0, idx1);
    u64* keys = plan->final_key_a ? keys1 : keys0;
    u32* idx = plan->final_idx ? idx1 : idx0;
    const u32 shift = words.shift;
    const u32 lane = threadIdx.x & 31;
    for (u64 base = (u64)blockIdx.x * blockDim.x; base < n; base += (u64)gridDim.x * blockDim.x) {  // warp-uniform trips
        const u64 i64 = base + threadIdx.x;
        const bool in = i64 < n;
        const u32 i = (u32)i64;
        const u64 key = in ? words[i] : 0;
        const u64 pref = key >> shift;
        // neighbours through shuffles; only the edge lanes touch memory again
        u64 pkey = __shfl_up_sync(0xffffffffu, key, 1);
        u64 next = __shfl_down_sync(0xffffffffu, pref, 1);
        if (in && lane == 0) pkey = i > 0 ? words[i - 1] : ~key;
        if (in && (lane == 31 || i + 1 >= n)) next = i + 1 < n ? (words[i + 1] >> shift) : ~pref;
        const bool same_prev = in && i > 0 && (pkey >> shift) == pref;
        // (a short run may be permuted concurrently by its start thread: harmless, only long runs consult the mask)
        bool differs;
        if constexpr (PACKED) differs = same_prev && chunk[idx[i]] != chunk[idx[i - 1]];  // full keys only inside runs
        else differs = same_prev && pkey != key;
        const u32 mixed = __ballot_sync(0xffffffffu, differs);
        if (lane == 0 && in) mixedmask[i >> 5] = mixed;  // base is a multiple of 32: one word per warp trip
        if (!in) continue;
        if (same_prev) {
            // the element kMaxTieRun places into a run registers it as long
            if (i >= (u32)kMaxTieRun && (words[i - kMaxTieRun] >> shift) == pref &&
                (i == (u32)kMaxTieRun || (words[i - kMaxTieRun - 1] >> shift) != pref))
                longlist[atomicAdd(&sum->long_count, 1u)] = i - kMaxTieRun;  // at most n / 33 entries
            continue;
        }
        if (next != pref) continue;  // run of one
        u32 len = 2;
        while (i + len < n && len <= (u32)kMaxTieRun && (words[i + len] >> shift) == pref) ++len;
        if (len > (u32)kMaxTieRun) continue;  // long run: registered by its 33rd element
        for (u32 a = 1; a < len; ++a) {  // stable insertion sort by the full key
            const u32 v = idx[i + a];
            u32 b = a;
            if constexpr (PACKED) {  // the prefixes are equal: only the row indices move
                const u64 k = chunk[v];
                while (b > 0 && chunk[idx[i + b - 1]] > k) {
                    idx[i + b] = idx[i + b - 1];
                    --b;
                }
            } else {
                const u64 k = keys[i + a];
                while (b > 0 && keys[i + b - 1] > k) {
                    keys[i + b] = keys[i + b - 1];
                    idx[i + b] = idx[i + b - 1];
                    --b;
                }
                keys[i + b] = k;
            }
            idx[i + b] = v;
        }
    }
}

// Hybrid tail of the packed three-pass schedule (run_shift == 8).  The passes sorted prefix bytes 1-3 only, so nearly
// every row sits in a run of equal 24-bit prefixes (n / 2^24 rows on average), still in input order.  A block owns the
// runs that START in its tile of kRunTile positions and stages the prefixes and row indices of the tile, with 32
// positions more on each side (a short run has at most kMaxTieRun rows), in shared memory.  Each warp walks the runs
// that start in its eighth of the tile in windows of up to 32 positions that end where a run ends, and ranks every row
// inside its run by (prefix byte 0, position) with 8 ballots, one per bit of the byte: that rank is its slot.  Rows whose
// whole prefixes are equal get adjacent slots, and only they read their full keys chunk[idx] to be ordered (stable
// insertion sort per group).  The row indices are read once and written back once, coalesced, per tile.  Long runs are
// left as they are, registered by their first row and marked where a row's key differs from its left neighbour's, as
// tie_fix_kernel does.  Only positions of short runs owned by a block are written, and a long run is never written, so
// blocks that read their neighbours' positions (halos) see either a value they ignore or a final one.
//
// GATHER: the block also moves the rows, out[j] = rows[idx[j]] for every position j it owns, so the sort's caller needs
// no separate gather and, unless it wants the permutation (write_idx), the row indices are not written back at all.
// Every position is owned by exactly one block:
//   * the positions of the short runs that start in the block's tile, halo positions after the tile included;
//   * the runs of one row and the long-run positions that lie inside the tile (a long run is gathered in input order;
//     the mixed ones are sorted on the side afterwards and their positions gathered again);
//   * but not the positions at the start of the tile that belong to a short run that began in the previous tile: that
//     block owns them.
// A block sees the run through the tile's first position the way the previous block sees it (both find its end, and
// its start when the run has <= 32 rows), so they agree on whether it is short.
constexpr int kRunTile = 1984;                 // positions owned by a block (a multiple of 32 and of 8)
constexpr int kRunSpan = kRunTile + 64;        // staged: local position l is global position tile * kRunTile - 32 + l
constexpr int kRunWords = kRunSpan / 32;
constexpr int kRunItems = kRunSpan / 256;
constexpr u32 kNoSlot = 0xffffffffu;
constexpr int kTailGatherUnroll = 4;  // 16-byte granules in flight per thread in the gathering tail

// Rows the gathering tail moves: gr 16-byte granules per row.  Granule q of a block's span belongs to position
// q / gr = (2q * gr_magic) >> 32 with gr_magic = ceil(2^31 / gr): with gr_magic = (2^31 + e) / gr, e < gr, that is exact
// while q e < 2^31, so for the span's kRunSpan * gr granules up to gr = kTailGatherMaxGranules.  (A u32 division or a
// 64-bit multiply needs more registers than 8 blocks per SM leave: either spilled.)
constexpr u32 kTailGatherMaxGranules = 1024;  // rows of up to 16 KB
struct TailGather {
    const uint4* rows;
    uint4* out;
    u32 gr, gr_magic;
    int write_idx;  // also write the final row indices back (the caller consumes the permutation)
};

__device__ __forceinline__ u32 granule_row(u32 q, const TailGather& G) { return __umulhi(q << 1, G.gr_magic); }

// 8 resident blocks per SM (26.3 KB of shared memory and 32 registers each, no spills): when gathering, with 4 granules
// in flight per thread, that matches the memory-level parallelism of gather_rows_kernel.
template <bool GATHER>
__global__ void __launch_bounds__(256, 8) tie_fix_runs_kernel(const u64* __restrict__ chunk, const u32* __restrict__ pre,
                                                                           u32* idx, u32 n, u32* __restrict__ mixedmask,
                                                                           u32* __restrict__ longlist, HybridSummary* sum,
                                                                           const TailGather G) {
    __shared__ u32 s_comp[kRunSpan];      // (prefix << 24) | l: prefix byte 0 on top
    __shared__ u32 s_idx[kRunSpan];       // row indices in position order
    __shared__ u32 s_out[kRunSpan];       // the staged prefixes; then row indices in slot order, kNoSlot: not written
    __shared__ u32 s_head[kRunWords];     // bit l: position l starts a run (positions outside [0, n) are runs of one)
    __shared__ u16 s_ties[kRunSpan / 2];  // groups of equal prefixes: first slot | (length - 1) << 11
    __shared__ u32 s_nties, s_long;
    __shared__ int s_first;               // first position of the tile that is not part of a short run of the previous tile
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int base = (int)blockIdx.x * kRunTile - 32;  // n < 2^30
    if (tid == 0) s_nties = s_long = 0;
    {
        u32 p[kRunItems], x[kRunItems];
#pragma unroll
        for (int it = 0; it < kRunItems; ++it) {
            const int g = base + it * 256 + tid;
            const bool in = g >= 0 && g < (int)n;
            p[it] = in ? pre[g] : 0;
            x[it] = in ? idx[g] : 0;
        }
#pragma unroll
        for (int it = 0; it < kRunItems; ++it) {
            s_out[it * 256 + tid] = p[it];
            s_idx[it * 256 + tid] = x[it];
        }
    }
    __syncthreads();
#pragma unroll
    for (int it = 0; it < kRunItems; ++it) {
        const int l = it * 256 + tid, g = base + l;
        const u32 p = s_out[l];
        // Local position 0 counts as a head: a run through it that reaches position 32 or later has > 32 rows anyway.
        const bool head = l == 0 || g <= 0 || g >= (int)n || ((p ^ s_out[l - 1]) >> 8) != 0;
        const u32 hb = __ballot_sync(0xffffffffu, head);
        if (lane == 0) s_head[l >> 5] = hb;
        s_comp[l] = (p << 24) | l;
    }
    __syncthreads();
#pragma unroll
    for (int it = 0; it < kRunItems; ++it) s_out[it * 256 + tid] = kNoSlot;
    // first head at or after local position x (kRunSpan if none)
    auto next_head = [&](int x) -> int {
        if (x >= kRunSpan) return kRunSpan;
        int w = x >> 5;
        u32 m = s_head[w] & (0xffffffffu << (x & 31));
        while (m == 0) {
            if (++w == kRunWords) return kRunSpan;
            m = s_head[w];
        }
        return w * 32 + __ffs(m) - 1;
    };
    if (tid == 0) {
        // the run through position 32 started in the previous tile: long, or short and owned by the previous block
        const int nh = next_head(33);
        const bool crosses = !(s_head[1] & 1);
        const bool long_cross = crosses && nh - (31 - __clz(s_head[0])) > kMaxTieRun;
        if (long_cross) s_long = 1;
        s_first = crosses && !long_cross ? nh : 32;
    }
    __syncthreads();

    const u32 lt_mask = lanemask_lt();
    {
        const int rs = 32 + warp * (kRunTile / 8), re = rs + kRunTile / 8;
        int ws = next_head(rs);
        while (ws < re) {  // warp-uniform: ws is a head
            // heads at positions ws .. ws + 32 (bit 0: ws itself)
            const u64 win = ((((u64)s_head[(ws >> 5) + 1] << 32) | s_head[ws >> 5]) >> (ws & 31)) & ((2ull << 32) - 1);
            const u64 later = win & ~1ull;
            if (later == 0) {  // a run of more than kMaxTieRun rows: left to classify_long_runs_kernel
                if (lane == 0) s_long = 1;
                ws = next_head(ws + kMaxTieRun + 1);
                continue;
            }
            // the window ends at its last head, or at the first head of the next warp's runs
            int len = 63 - __clzll(later);
            if (re - ws <= kMaxTieRun) {
                const u64 beyond = later >> (re - ws);
                if (beyond) len = re - ws + __ffsll(beyond) - 1;
            }
            const u32 hb = (u32)win;
            const bool act = lane < len;
            const u32 c = act ? s_comp[ws + lane] : 0;
            const int start = 31 - __clz(hb & (0xffffffffu >> (31 - lane)));
            const u32 after = hb & (0xfffffffeu << lane);
            const int end = after ? __ffs(after) - 1 : 32;
            // rank inside the run [start, end) by byte 0, MSB first, then by position
            u32 lt = 0, eq = (0xffffffffu >> (32 - end)) & (0xffffffffu << start);
#pragma unroll
            for (int b = 7; b >= 0; --b) {
                const bool bit = (c >> (24 + b)) & 1;
                const u32 v = __ballot_sync(0xffffffffu, bit);
                if (bit) {
                    lt |= eq & ~v;
                    eq &= v;
                } else {
                    eq &= ~v;
                }
            }
            if (act && end - start >= 2) {
                const int first = ws + start + __popc(lt);  // slot of the first row with this prefix
                s_out[first + __popc(eq & lt_mask)] = s_idx[ws + lane];
                if (__popc(eq) > 1 && (eq & lt_mask) == 0) s_ties[atomicAdd(&s_nties, 1u)] = (u16)(first | ((__popc(eq) - 1) << 11));
            }
            ws += len;
        }
    }
    __syncthreads();

    // equal prefixes: stable insertion sort by the full key
    for (u32 t = tid; t < s_nties; t += 256) {
        const u32 q = s_ties[t] & 0x7ff, e = q + (s_ties[t] >> 11) + 1;
        for (u32 a = q + 1; a < e; ++a) {
            const u32 x = s_out[a];
            const u64 k = chunk[x];
            u32 b = a;
            while (b > q && chunk[s_out[b - 1]] > k) {
                s_out[b] = s_out[b - 1];
                --b;
            }
            s_out[b] = x;
        }
    }
    if (s_long) {
        // Long runs: register each by its first row, and mark every position whose key differs from its left
        // neighbour's.  A position's run [ph, nh) comes from the head bits of its word and the two around it.
#pragma unroll 1
        for (int it = 0; it < kRunItems; ++it) {
            const int l = it * 256 + tid, w = l >> 5, g = base + l;
            if (w == 0 || l >= 32 + kRunTile) continue;  // warp-uniform
            const u64 below = (((u64)s_head[w] << 32) | s_head[w - 1]) & (~0ull >> (31 - lane));
            const u64 above = (((u64)s_head[w + 1] << 32) | s_head[w]) & (~0ull << (lane + 1));
            const int ph = w * 32 - 32 + 63 - __clzll(below), nh = w * 32 + __ffsll(above) - 1;
            const bool is_long = below == 0 || above == 0 || nh - ph > kMaxTieRun;
            const bool head = (s_head[w] >> lane) & 1;
            if (head && is_long && g < (int)n) longlist[atomicAdd(&sum->long_count, 1u)] = (u32)g;
            const bool differs = !head && is_long && g < (int)n &&
                                 (((s_comp[l] ^ s_comp[l - 1]) >> 24) != 0 || chunk[s_idx[l]] != chunk[s_idx[l - 1]]);
            const u32 mixed = __ballot_sync(0xffffffffu, differs);
            if (lane == 0 && g < (int)n) mixedmask[g >> 5] = mixed;
        }
    } else if (tid < kRunTile / 32) {
        const int g = base + 32 + tid * 32;
        if (g < (int)n) mixedmask[g >> 5] = 0;
    }
    __syncthreads();
    if constexpr (GATHER) {
        // granule q of the span is granule q % gr of position q / gr: consecutive threads read and write whole rows
        const int lo = s_first, hi = min(32 + kRunTile, (int)n - base);
        const u32 total = (u32)kRunSpan * G.gr;  // a multiple of 256 * kTailGatherUnroll: every step is whole
        static_assert(kRunSpan % (256 * kTailGatherUnroll) == 0, "whole gather steps");
        const long long out0 = (long long)base * G.gr;
        for (u32 q0 = tid; q0 < total; q0 += 256 * kTailGatherUnroll) {
            uint4 v[kTailGatherUnroll];
            bool ok[kTailGatherUnroll];
#pragma unroll
            for (int k = 0; k < kTailGatherUnroll; ++k) {
                const u32 q = q0 + k * 256;
                const u32 l = granule_row(q, G);
                u32 r = s_out[l];
                if (r == kNoSlot && (int)l >= lo && (int)l < hi) r = s_idx[l];
                ok[k] = r != kNoSlot;
                if (ok[k]) v[k] = ld_l2_u128(G.rows + (u64)r * G.gr + (q - l * G.gr));
            }
#pragma unroll
            for (int k = 0; k < kTailGatherUnroll; ++k)
                if (ok[k]) st_stream_u128(G.out + (out0 + q0 + k * 256), v[k]);
        }
    }
    if (!GATHER || G.write_idx) {
#pragma unroll
        for (int it = 0; it < kRunItems; ++it) {
            const int q = it * 256 + tid;
            if (s_out[q] != kNoSlot) idx[base + q] = s_out[q];
        }
    }
}

// Rows at the positions of the mixed long runs again, once sort_mixed_runs has rewritten their row indices.
__global__ void __launch_bounds__(256) regather_rows_kernel(const u32* __restrict__ pos, u32 m, const u32* __restrict__ idx,
                                                            const TailGather G) {
    const u64 total = (u64)m * G.gr;
    for (u64 q = (u64)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (u64)gridDim.x * blockDim.x) {
        const u64 k = q / G.gr;
        const u32 g = (u32)(q - k * G.gr), j = pos[k];
        st_stream_u128(G.out + (u64)j * G.gr + g, ld_stream_u128(G.rows + (u64)idx[j] * G.gr + g));
    }
}

// One warp per registered long run: find its end (gallop + binary search over the prefix-sorted words), then look for
// a "different key than the left neighbour" mark inside it.
template <bool PACKED>
__global__ void __launch_bounds__(256) classify_long_runs_kernel(const SortPlan* plan, const u64* keys0, const u64* keys1,
                                                                 const u32* idx0, const u32* idx1, u32 n,
                                                                 const u32* __restrict__ mixedmask, const u32* __restrict__ longlist,
                                                                 HybridSummary* sum, MixedRun* __restrict__ mixedlist) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        sum->hybrid = plan->hybrid;
        sum->final_idx = plan->final_idx;
        sum->final_key = plan->final_key_a;
    }
    if (!plan->hybrid) return;
    const TailWords<PACKED> keys(plan, keys0, keys1, idx0, idx1);
    const u32 shift = keys.shift;
    const u32 lane = threadIdx.x & 31;
    const u32 count = sum->long_count;
    const u32 warps = gridDim.x * (blockDim.x >> 5);
    for (u32 r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < count; r += warps) {
        const u32 s = longlist[r];
        // end of the run, searched by the whole warp: lane l probes s + (32 << l) (exponential), then the bracket is cut
        // 32 ways per round — 2-4 rounds of parallel loads instead of ~2 log2(length) dependent ones
        const u64 pref = keys[s] >> shift;
        u64 lo, hi;
        {
            const u64 pos = (u64)s + ((u64)kMaxTieRun << lane);
            const bool diff = pos >= n || (keys[pos] >> shift) != pref;  // lane 0 probes s + 32: same prefix by construction
            const int first = __ffs(__ballot_sync(0xffffffffu, diff)) - 1;  // >= 1; lane 31 is always past the end (n < 2^30)
            lo = (u64)s + ((u64)kMaxTieRun << (first - 1));
            hi = min((u64)n, (u64)s + ((u64)kMaxTieRun << first));
        }
        while (hi - lo > 1) {  // prefix(lo) == pref; hi == n or prefix(hi) != pref
            const u64 len = hi - lo;
            const u64 pos = lo + ((len * (lane + 1)) >> 5);
            const bool diff = pos >= hi || (keys[pos] >> shift) != pref;
            const int first = __ffs(__ballot_sync(0xffffffffu, diff)) - 1;  // lane 31 probes hi: always set
            const u64 new_hi = __shfl_sync(0xffffffffu, pos, first);
            const u64 new_lo = first > 0 ? __shfl_sync(0xffffffffu, pos, first - 1) : lo;
            hi = new_hi;
            lo = new_lo;
        }
        const u32 e = (u32)hi;
        // marks at positions s+1 .. e-1
        const u32 fw = (s + 1) >> 5, lw = (e - 1) >> 5;
        bool any = false;
        for (u32 w = fw + lane; w <= lw; w += 32) {
            u32 m = mixedmask[w];
            if (w == fw) m &= 0xffffffffu << ((s + 1) & 31);
            if (w == lw && ((e & 31) != 0)) m &= (1u << (e & 31)) - 1;
            any |= m != 0;
        }
        if (__any_sync(0xffffffffu, any) && lane == 0) {
            const u32 slot = atomicAdd(&sum->mixed_count, 1u);
            if (slot < kMixedCap) mixedlist[slot] = MixedRun{s, e};
            atomicAdd(&sum->mixed_elems, (unsigned long long)(e - s));
        }
    }
}

// Side buffer of the mixed long runs (in run order == key order == position order), and the way back.  Packed format
// (keys == nullptr): the full keys are read through the permutation and only the permutation is written back.
__global__ void __launch_bounds__(256) expand_mixed_runs_kernel(const u64* __restrict__ keys, const u64* __restrict__ chunk,
                                                                const u32* __restrict__ idx, const u32* __restrict__ rs,
                                                                const u32* __restrict__ re, const u32* __restrict__ roff, u32 nruns,
                                                                u64* __restrict__ side_key, u32* __restrict__ side_idx, u32* __restrict__ side_pos) {
    for (u32 r = blockIdx.x; r < nruns; r += gridDim.x) {
        const u32 s = rs[r], len = re[r] - s, off = roff[r];
        for (u32 j = threadIdx.x; j < len; j += blockDim.x) {
            const u32 v = idx[s + j];
            side_key[off + j] = keys ? keys[s + j] : chunk[v];
            side_idx[off + j] = v;
            side_pos[off + j] = s + j;
        }
    }
}
__global__ void __launch_bounds__(256) writeback_mixed_runs_kernel(const SortPlan* splan, const u32* sa, const u32* sb, u32 m,
                                                                   const u64* __restrict__ side_key, const u32* __restrict__ side_idx,
                                                                   const u32* __restrict__ side_pos, u64* __restrict__ keys, u32* __restrict__ idx) {
    for (u32 k = blockIdx.x * blockDim.x + threadIdx.x; k < m; k += gridDim.x * blockDim.x) {
        const u32 src = perm_at(splan, sa, sb, k);  // k-th smallest side element goes to the k-th marked position
        const u32 pos = side_pos[k];
        if (keys) keys[pos] = side_key[src];
        idx[pos] = side_idx[src];
    }
}

// ---------------------------------------------------------------------------------------------
// One digit pass.  Element formats:
//   pair   (PACKED = false): read 8 B key + 4 B index, write 8 B key + 4 B index;
//   packed (PACKED = true):  one u64 word (prefix << 32) | row index.  The first pass reads the 8 B key from the chunk and
//          builds the word, the middle passes read and write 8 B, the last one writes the 4 B row index (+ the 4 B prefix
//          for the hybrid tail).
// ---------------------------------------------------------------------------------------------
struct PassParams {
    const u64* chunk;
    u64* keys[2];
    u32* idx[2];
    const u32* digit_base;  // exclusive offsets of this pass's 256 digits
    u32* status;            // [tiles][256] look-back words, zeroed
    u32* counter;           // dynamic tile id, zeroed
    const SortPlan* plan;
    int plan_index;  // into plan->pass
    int shift;       // of the digit in the key (pair) or in the packed word (32 + 8 k in the k-th packed pass)
    u32 n;
    u32 prefix_sel, prefix_mask;  // packed: SortPlan::prefix_sel / prefix_mask
    int copy16;                   // packed: chunk and key buffers are 16-byte aligned (a chunk may start at any word)
};

// Element region of a tile's shared memory: packed, the staged input words and the tile-sorted words (TILE each); pair,
// the tile-sorted keys and row indices (the input keys are held in registers).
constexpr size_t tile_elem_bytes(int items, bool packed) { return (size_t)kSortThreads * items * (packed ? 2 * 8 : 12); }

// + the warp histograms [WARPS][256], the digit offsets [256], the global bases [256] and 16 words of scratch
constexpr size_t pass_smem_bytes(int items, bool packed) {
    return tile_elem_bytes(items, packed) + (size_t)(kSortThreads / 32) * kRadix * 4 + 2 * kRadix * 4 + 16 * 4;
}

__device__ __forceinline__ void cp_async_u64(u64* dst, const u64* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" :: "r"((u32)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

template <int THREADS, int ITEMS, bool FULL, bool PACKED>
__device__ __forceinline__ void onesweep_tile(const PassParams& P, const PassDesc pd, const u32 tile, unsigned char* smem_raw) {
    constexpr int WARPS = THREADS / 32;
    constexpr int TILE = THREADS * ITEMS;
    u64* s_in = reinterpret_cast<u64*>(smem_raw);                         // packed: TILE words as loaded (warp-striped)
    u64* s_keys = PACKED ? s_in + TILE : reinterpret_cast<u64*>(smem_raw);  // TILE keys / packed words, tile-sorted
    u32* s_vals = reinterpret_cast<u32*>(smem_raw + (size_t)TILE * 8);      // pair: TILE row indices, tile-sorted
    u32* s_hist = reinterpret_cast<u32*>(smem_raw + tile_elem_bytes(ITEMS, PACKED));  // [WARPS][256]
    u32* s_excl = s_hist + WARPS * kRadix;                      // [256]
    u32* s_gbase = s_excl + kRadix;                             // [256]
    u32* s_misc = s_gbase + kRadix;                             // [0..7] warp totals, [8] tile id

    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const u32 base = tile * (u32)TILE;
    const u32 tile_count = FULL ? (u32)TILE : P.n - base;

    const u64* kin = pd.src_kind == 2 ? (pd.key_src ? P.keys[1] : P.keys[0]) : P.chunk;
    const u32* iin = pd.idx_src ? P.idx[1] : P.idx[0];
    u64* kout = pd.key_dst ? P.keys[1] : P.keys[0];
    u32* iout = pd.idx_dst ? P.idx[1] : P.idx[0];
    const int shift = P.shift;

    // The row indices of this tile are needed only after ranking: pull their lines into L2 now so the
    // later loads do not expose DRAM latency (one 128-byte line per thread).
    if (!PACKED && pd.src_kind == 2) {
        const char* ibase = reinterpret_cast<const char*>(iin + base);
        const u32 ibytes = tile_count * 4;
        for (u32 off = tid * 128; off < ibytes; off += THREADS * 128)
            asm volatile("prefetch.global.L2 [%0];" :: "l"(ibase + off));
    }

    // ---- load the tile, warp-striped: item i of lane l is element warp_slot + i*32 + l of the tile ----
    // Packed: the words are staged in shared memory with cp.async.  Kept there until they are written out instead of
    // occupying 2 registers per item, they free the registers for more items per tile.  Each warp copies its own slice,
    // so the cp.async.wait_all and __syncwarp below are all the synchronisation the copies need.  16-byte copies that
    // bypass L1 take the packed pass from 0.96 to 0.89 ms (16 items at 3 CTAs per SM) against 8-byte copies through L1;
    // the 8-byte copies remain for buffers that are not 16-byte aligned.  Pair: the keys are loaded into registers
    // (staging keys and row indices with 8- and 4-byte copies measured slower: 1.32 vs 1.29 ms per pass).
    const u32 wslot = warp * (32 * ITEMS) + lane;
    const u32 wbase = base + wslot;
    u64 key[PACKED ? 1 : ITEMS];
    if constexpr (PACKED) {
        static_assert(ITEMS % 2 == 0, "16-byte copies of 8-byte words");
        if (P.copy16) {
            // the warp's slice of the tile is contiguous: 16-byte copies that bypass L1, lane l copies bytes 16 (l + 32 k)
            const u32 wfirst = base + warp * (32 * ITEMS);
            u64* sdst = s_in + warp * (32 * ITEMS);
#pragma unroll
            for (int k = 0; k < ITEMS / 2; ++k) {
                const u32 e = 2 * (lane + 32 * k);
                if (FULL || wfirst + e < P.n) {
                    const u32 bytes = (FULL || wfirst + e + 1 < P.n) ? 16 : 8;
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" :: "r"((u32)__cvta_generic_to_shared(sdst + e)),
                                 "l"(kin + wfirst + e), "r"(bytes) : "memory");
                }
            }
        } else {
#pragma unroll
            for (int i = 0; i < ITEMS; ++i)
                if (FULL || wbase + i * 32 < P.n) cp_async_u64(s_in + wslot + i * 32, kin + wbase + i * 32);
        }
    } else if (pd.src_kind == 1) {
        u32 src[ITEMS];
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) {
            u32 pos = wbase + i * 32;
            src[i] = (FULL || pos < P.n) ? ld_stream_u32(iin + pos) : 0u;
        }
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) {
            u32 pos = wbase + i * 32;
            key[i] = (FULL || pos < P.n) ? kin[src[i]] : ~0ull;
        }
    } else {
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) {
            u32 pos = wbase + i * 32;
            key[i] = (FULL || pos < P.n) ? ld_stream_u64(kin + pos) : ~0ull;
        }
    }
    // the warp's private histogram is cleared while the loads are in flight
    u32* wh = s_hist + warp * kRadix;
    reinterpret_cast<uint4*>(wh)[lane] = make_uint4(0, 0, 0, 0);
    reinterpret_cast<uint4*>(wh)[lane + 32] = make_uint4(0, 0, 0, 0);
    // Element i of this lane.  The first packed pass builds the word (prefix << 32) | row index from the chunk's key.
    // Packed items past the end of a partial tile read stale words: they are masked out of the ranking and never written.
    auto elem = [&](int i) -> u64 {
        if constexpr (PACKED) {
            const u64 v = s_in[wslot + i * 32];
            if (pd.src_kind != 0) return v;
            const u32 pref = __byte_perm((u32)v, (u32)(v >> 32), P.prefix_sel) & P.prefix_mask;
            return ((u64)pref << 32) | (wbase + i * 32);
        } else {
            return key[i];
        }
    };
    if (PACKED) cp_async_wait_all();
    __syncwarp();  // every lane's copies and histogram clear

    // ---- rank inside the warp: stable (item-major, then lane) ----
    // Peers with the same digit are found with 8 ballots (one per digit bit).  MATCH.ANY is NOT used:
    // its cost grows with the number of distinct values in the warp, and random 8-bit digits have
    // many; the ballots cost the same on any data.  The running per-digit counts of the warp live in its
    // private shared histogram.
    u32 m[ITEMS];  // peer mask, then rank inside the warp
    const u32 lt = lanemask_lt();
    auto peers = [&](u32 d, int i) -> u32 {
        u32 mm = 0xffffffffu;
#pragma unroll
        for (int b = 0; b < kRadixBits; ++b) {
            const bool bit = (d >> b) & 1;
            const u32 v = __ballot_sync(0xffffffffu, bit);
            mm &= bit ? v : ~v;
        }
        if (!FULL) mm &= __ballot_sync(0xffffffffu, wbase + i * 32 < P.n);
        return mm;
    };
    if constexpr (PACKED) {
        // Every item's peer mask is computed first (the ballots of different items are independent).  Then the lowest
        // lane of each digit group adds the group's size to the bin with one shared atomic, and the group reads the old
        // count from it with a shuffle, so no item waits for the previous item's load-store round trip.
        u32 dig[(ITEMS + 3) / 4] = {};  // the items' digits, four per word
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) {
            const u32 d = (u32)(elem(i) >> shift) & 0xff;
            dig[i / 4] |= d << (8 * (i % 4));
            m[i] = peers(d, i);
        }
        u32 prev[ITEMS];
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) {
            const u32 d = (dig[i / 4] >> (8 * (i % 4))) & 0xff;
            prev[i] = 0;
            if ((FULL || wbase + i * 32 < P.n) && (m[i] & lt) == 0) prev[i] = atomicAdd(&wh[d], (u32)__popc(m[i]));
            // The leaders of consecutive items are different lanes, and only this barrier orders their shared accesses
            // (PTX memory model): without it item i+1's add to a bin could be performed before item i's, and equal
            // digits would no longer be ranked item-major, i.e. the sort would lose its stability.
            __syncwarp();
        }
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) m[i] = __shfl_sync(0xffffffffu, prev[i], __ffs(m[i]) - 1) + __popc(m[i] & lt);
    } else {
        // Pair format (keys in registers): every lane reads its bin (same-digit lanes broadcast), the lowest lane of each
        // digit group writes the bumped count back.  The shared atomics above measured slower here (1.304 vs 1.297 ms
        // per pass of the composite workload).
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) {
            const u32 d = (u32)(key[i] >> shift) & 0xff;
            const u32 mm = peers(d, i);
            const u32 prev = wh[d];
            __syncwarp();
            if ((FULL || wbase + i * 32 < P.n) && (mm & lt) == 0) wh[d] = prev + __popc(mm);
            m[i] = prev + __popc(mm & lt);
            __syncwarp();
        }
    }
    __syncthreads();

    // ---- per digit (thread d): offsets of each warp inside the digit, tile count, publish ----
    u32 cnt = 0;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) cnt += s_hist[w * kRadix + tid];
    u32* my_status = P.status + (size_t)tile * kRadix + tid;
    st_volatile_u32(my_status, (tile == 0 ? kFlagInclusive : kFlagPartial) | cnt);
    const u32 local_excl = block_exclusive_scan_256(cnt, s_misc);
    {
        // s_hist[w][d] := position in the tile-sorted order of the first key of warp w with digit d
        u32 run = local_excl;
#pragma unroll
        for (int w = 0; w < WARPS; ++w) {
            u32 c = s_hist[w * kRadix + tid];
            s_hist[w * kRadix + tid] = run;
            run += c;
        }
    }
    __syncthreads();

    // ---- decoupled look-back, software-pipelined with the shared-memory scatter below ----
    // Thread `tid` owns the chain of digit `tid`.  Tiles reach this point every few dozen cycles but a
    // status word costs an L2 round trip, so a tile typically has to add the partial counts of ~10
    // predecessors.  Instead of spinning, one status load is kept in flight while the keys and row
    // indices are scattered into shared memory; whatever is left is finished by the loop after them.
    // (Loading the words of 4 predecessors at a time measured slower: 1.00 vs 0.94 ms per packed pass.)
    u32 lb_excl = 0;
    i32 lb_tile = (i32)tile - 1;
    bool lb_done = tile == 0;
    u32 lb_word = 0;
    auto lb_issue = [&]() {
        if (!lb_done) lb_word = ld_volatile_u32(P.status + (size_t)lb_tile * kRadix + tid);
    };
    auto lb_consume = [&]() {
        if (!lb_done) {
            const u32 f = lb_word >> 30;
            if (f != 0) {
                lb_excl += lb_word & kValueMask;
                if (f == 2) lb_done = true;
                else --lb_tile;
            }
        }
    };

    // ---- keys and row indices -> shared memory in tile-sorted order (the row index of a packed word travels inside it) ----
#pragma unroll
    for (int i = 0; i < ITEMS; ++i) {
        if ((i & 3) == 0) lb_issue();
        const u32 pos = wbase + i * 32;
        if (FULL || pos < P.n) {
            const u64 w = elem(i);
            const u32 lp = wh[(u32)(w >> shift) & 0xff] + m[i];
            m[i] = lp;
            s_keys[lp] = w;
        }
        if ((i & 3) == 3) lb_consume();
    }
    if (PACKED) {
        // the row index travels inside the word
    } else if (pd.src_kind == 0) {
#pragma unroll
        for (int i = 0; i < ITEMS; ++i) {
            if ((i & 3) == 0) lb_issue();
            const u32 pos = wbase + i * 32;
            if (FULL || pos < P.n) s_vals[m[i]] = pos;
            if ((i & 3) == 3) lb_consume();
        }
    } else {
        constexpr int VB = 4;
#pragma unroll
        for (int b0 = 0; b0 < ITEMS; b0 += VB) {
            lb_issue();
            u32 v[VB];
#pragma unroll
            for (int i = 0; i < VB; ++i) {
                const u32 pos = wbase + (b0 + i) * 32;
                v[i] = (FULL || pos < P.n) ? ld_stream_u32(iin + pos) : 0u;
            }
#pragma unroll
            for (int i = 0; i < VB; ++i) {
                const u32 pos = wbase + (b0 + i) * 32;
                if (FULL || pos < P.n) s_vals[m[b0 + i]] = v[i];
            }
            lb_consume();
        }
    }
    while (!lb_done) {
        lb_issue();
        lb_consume();
    }
    if (tile > 0) st_volatile_u32(my_status, kFlagInclusive | ((lb_excl + cnt) & kValueMask));
    s_gbase[tid] = P.digit_base[tid] + lb_excl - local_excl;
    __syncthreads();

    // ---- write out: consecutive threads -> consecutive shared slots -> runs of one digit ----
#pragma unroll
    for (int k = 0; k < ITEMS; ++k) {
        const u32 j = tid + k * THREADS;
        if (FULL || j < tile_count) {
            const u64 kk = s_keys[j];
            const u32 g = s_gbase[(u32)(kk >> shift) & 0xff] + j;
            if (!pd.last) kout[g] = kk;
            if constexpr (PACKED) {
                if (pd.last) {
                    iout[g] = (u32)kk;
                    if (pd.write_prefix) (pd.idx_dst ? P.idx[0] : P.idx[1])[g] = (u32)(kk >> 32);
                }
            } else {
                iout[g] = s_vals[j];
            }
        }
    }
}

template <int THREADS, int ITEMS, int MINB, bool PACKED>
__global__ void __launch_bounds__(THREADS, MINB) onesweep_pass_kernel(const PassParams P) {
    constexpr int WARPS = THREADS / 32;
    constexpr int TILE = THREADS * ITEMS;
    static_assert(THREADS == 256, "digit phase assumes one thread per bin");
    extern __shared__ __align__(16) unsigned char smem_raw[];
    u32* s_misc = reinterpret_cast<u32*>(smem_raw + tile_elem_bytes(ITEMS, PACKED)) + WARPS * kRadix + 2 * kRadix;

    const PassDesc pd = P.plan->pass[P.plan_index];
    if (!pd.active) return;
    // One tile per CTA, one CTA per tile.  (A persistent variant — 3 CTAs per SM looping over an atomic tile counter —
    // measured 8 % slower on the active passes: 6.51 vs 5.96 ms for 8 passes over 10^8 rows; hardware CTA launch is
    // cheaper than the extra barrier per tile.)  Tile ids still come from the atomic counter so that they are handed
    // out in start order, which the decoupled look-back relies on.
    if (threadIdx.x == 0) s_misc[8] = atomicAdd(P.counter, 1u);
    __syncthreads();
    const u32 tile = s_misc[8];
    if ((u64)(tile + 1) * TILE <= (u64)P.n) onesweep_tile<THREADS, ITEMS, true, PACKED>(P, pd, tile, smem_raw);
    else onesweep_tile<THREADS, ITEMS, false, PACKED>(P, pd, tile, smem_raw);
}

__global__ void materialize_perm_kernel(const SortPlan* plan, const u32* a, const u32* b, u64 n, u32* dst) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x)
        dst[i] = perm_at(plan, a, b, i);
}

// Shapes of the pass kernel (items per thread, min resident CTAs per SM), one per element format: the fastest measured
// on an H100 SXM at a 700 W power limit.  Pair format (15.3 vs 18.0 ms per 10^8-row sort for 16 items at 3 CTAs per SM):
// 2 CTAs per SM keep 128 registers without spills, where 3 CTAs per SM (80 registers) spill to local memory.  Packed
// format (mean pass launch over a 10^8-row sort, 4 packed passes): 16 items at 2 CTAs per SM 0.95 ms, 125 registers, no
// spills; 10 at 3 (80 registers, no spills) 1.05 ms; 12 at 3 (12 B spilled) 0.98 ms; 8 at 4 (16 B spilled) 1.16 ms.
// With the packed tile staged in shared memory and ranked by shared atomics (H100 80GB HBM3, 400 W power limit; the
// register-held kernel's 16 items at 2 CTAs: 0.98-0.99 ms on that card).  8-byte copies through L1: 16 items at 3 CTAs
// per SM 0.94-0.96 ms (80 registers, 74 KB of shared memory); 16 at 2 1.03 ms (127 registers); 12 at 3 1.01 ms (80
// registers); 8 at 4 1.18 ms (64 registers); 24 at 2 0.95 ms.  16-byte copies bypassing L1: 24 items at 2 CTAs per SM
// 0.87-0.89 ms (128 registers, 106 KB of shared memory); 16 at 3 0.89-0.90 ms (80 registers); 20 at 2 0.93 ms (128
// registers).  None of them spills.
struct PassKernel {
    int items;
    size_t smem;
    void (*kernel)(const PassParams);
    u32 tiles(u64 n) const { return (u32)((n + (u64)kSortThreads * items - 1) / ((u64)kSortThreads * items)); }
};
#define YTGPU_PASS_KERNEL(items, ctas, packed) \
    { items, pass_smem_bytes(items, packed), onesweep_pass_kernel<kSortThreads, items, ctas, packed> }
const PassKernel kPairPass = YTGPU_PASS_KERNEL(16, 2, false);
const PassKernel kPackedPass = YTGPU_PASS_KERNEL(24, 2, true);
#undef YTGPU_PASS_KERNEL

void set_sort_func_attrs(Context* ctx) {
    if (ctx->func_attrs_done & FA_SORT_PASS) return;  // per device (the attribute belongs to the current device's function)
    for (const PassKernel* x : {&kPairPass, &kPackedPass})
        cudaFuncSetAttribute(x->kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)x->smem);
    // 8 gathering tail blocks per SM need the largest shared-memory carveout
    cudaFuncSetAttribute(tie_fix_runs_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared);
    ctx->func_attrs_done |= FA_SORT_PASS;
}

// Checks the arguments and, unless the caller filled `hist`, computes the digit counts of every chunk.
Status sort_setup(Context* ctx, const u64* const* chunks, int nchunks, u64 n, SortScratch* s) {
    if (nchunks < 1 || nchunks > kMaxKeyChunks)
        return make_status(YTGPU_ERR_UNSUPPORTED, "normalised key of %d bytes exceeds the %d-byte limit",
                           nchunks * 8, kMaxKeyChunks * 8);
    if (n >= (1ull << 30))
        return make_status(YTGPU_ERR_UNSUPPORTED, "row count %llu exceeds 2^30-1 rows per sort call",
                           (unsigned long long)n);
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    if (s->hist_precomputed) return Status{};
    YTGPU_TRY(prepare_histogram(ctx, nchunks, s));
    KernelTimer t(ctx, KC_HISTOGRAM, nchunks);
    const u64 per_block = (u64)kHistThreads * kHistItems;
    const u32 blocks = (u32)std::min<u64>((n + per_block - 1) / per_block, (u64)kNumSms * 4);
    for (int c = 0; c < nchunks; ++c)
        histogram_kernel<<<blocks, kHistThreads, 0, ctx->stream>>>(chunks[c], n, s->hist.p + (size_t)c * kPassesPerChunk * kRadix);
    s->hist_precomputed = true;
    return Status{};
}

}  // namespace

// Stable re-sort of the few long runs of equal prefixes that mix different keys: their (key, index) pairs are copied
// to a side buffer in run order, sorted by the full key with the plain schedule, and written back — the k-th smallest
// side element belongs at the k-th marked position because runs are ordered by prefix, i.e. by key.  Packed format
// (packed_chunk != nullptr): the keys are read from the chunk through the permutation, only the permutation is written.
// regather: the gathering tail moved the rows already; those of the re-sorted positions are moved again.
static Status sort_mixed_runs(Context* ctx, SortScratch* s, const HybridSummary& hs, const MixedRun* mixedlist_dev,
                              const u64* packed_chunk, const TailGather* regather) {
    cudaStream_t st = ctx->stream;
    const u32 w = hs.mixed_count;
    std::vector<MixedRun> runs(w);
    YTGPU_CUDA_TRY(cudaMemcpyAsync(runs.data(), mixedlist_dev, (size_t)w * sizeof(MixedRun), cudaMemcpyDeviceToHost, st));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(st));
    std::sort(runs.begin(), runs.end(), [](const MixedRun& a, const MixedRun& b) { return a.s < b.s; });
    std::vector<u32> host(3 * (size_t)w);
    u32 total = 0;
    for (u32 r = 0; r < w; ++r) {
        host[r] = runs[r].s;
        host[w + r] = runs[r].e;
        host[2 * (size_t)w + r] = total;
        total += runs[r].e - runs[r].s;
    }
    DevBuf<u32> meta, side_idx, side_pos;
    DevBuf<u64> side_key;
    YTGPU_TRY(meta.allocate(ctx, 3 * (size_t)w));
    YTGPU_TRY(side_key.allocate(ctx, total));
    YTGPU_TRY(side_idx.allocate(ctx, total));
    YTGPU_TRY(side_pos.allocate(ctx, total));
    YTGPU_CUDA_TRY(cudaMemcpyAsync(meta.p, host.data(), host.size() * 4, cudaMemcpyHostToDevice, st));
    u64* keys = packed_chunk ? nullptr : (hs.final_key ? s->keys[1].p : s->keys[0].p);
    u32* idx = hs.final_idx ? s->idx[1].p : s->idx[0].p;
    expand_mixed_runs_kernel<<<std::min<u32>(w, (u32)kNumSms * 8), 256, 0, st>>>(keys, packed_chunk, idx, meta.p, meta.p + w, meta.p + 2 * (size_t)w,
                                                                              w, side_key.p, side_idx.p, side_pos.p);
    ctx->count_launch();
    SortScratch side;
    side.no_hybrid = true;
    PermRef sperm;
    const u64* sptr[1] = {side_key.p};
    YTGPU_TRY(radix_sort_chunks(ctx, sptr, 1, total, &side, &sperm));
    writeback_mixed_runs_kernel<<<(u32)std::min<u64>(((u64)total + 255) / 256, (u64)kNumSms * 8), 256, 0, st>>>(sperm.plan, sperm.idx[0], sperm.idx[1],
                                                                                                              total, side_key.p, side_idx.p,
                                                                                                              side_pos.p, keys, idx);
    ctx->count_launch();
    if (regather) {
        KernelTimer t(ctx, KC_GATHER);
        regather_rows_kernel<<<(u32)std::min<u64>(((u64)total * regather->gr + 255) / 256, (u64)kNumSms * 16), 256, 0, st>>>(side_pos.p, total,
                                                                                                                       idx, *regather);
    }
    YTGPU_CUDA_TRY(cudaGetLastError());
    YTGPU_CUDA_TRY(cudaStreamSynchronize(st));  // `host` / `runs` back the asynchronous upload
    return Status{};
}

Status radix_sort_chunks(Context* ctx, const u64* const* chunks, int nchunks, u64 n, SortScratch* s,
                         PermRef* out) {
    YTGPU_TRY(sort_setup(ctx, chunks, nchunks, n, s));
    set_sort_func_attrs(ctx);
    cudaStream_t st = ctx->stream;
    const u32 tiles = std::max(kPairPass.tiles(n), kPackedPass.tiles(n));  // look-back rows per pass, enough for either format
    const int total_passes = nchunks * kPassesPerChunk;

    YTGPU_TRY(s->keys[0].allocate(ctx, n));
    YTGPU_TRY(s->keys[1].allocate(ctx, n));
    YTGPU_TRY(s->idx[0].allocate(ctx, n));
    YTGPU_TRY(s->idx[1].allocate(ctx, n));
    YTGPU_TRY(s->offsets.allocate(ctx, (size_t)total_passes * kRadix));
    YTGPU_TRY(s->status.allocate(ctx, (size_t)kPassesPerChunk * tiles * kRadix));
    YTGPU_TRY(s->counters.allocate(ctx, (size_t)total_passes));
    YTGPU_TRY(s->plan.allocate(ctx, 1));

    YTGPU_CUDA_TRY(cudaMemsetAsync(s->counters.p, 0, (size_t)total_passes * 4, st));
    const int allow_hybrid = ctx->opt_sort_hybrid && !s->no_hybrid && n >= kHybridMinRows;

    // Single-chunk sorts of >= kHybridMinRows rows read the plan back: the host launches only the active passes, in the
    // plan's element format.  Smaller sorts stay free of host round trips and launch every digit's pass (inactive ones
    // return at once).
    const bool read_plan = nchunks == 1 && n >= kHybridMinRows;
    plan_kernel<<<1, 256, 0, st>>>(s->hist.p, s->offsets.p, nchunks, (u32)n, s->plan.p, allow_hybrid, s->keep_keys ? 1 : 0,
                                   read_plan && !s->keep_keys ? 1 : 0);
    ctx->count_launch();

    // plan_index: into plan->pass; slot: the pass's look-back status rows
    auto launch_pass = [&](const PassKernel& v, const u64* chunk, int plan_index, int slot, int counter, int shift, const SortPlan& hp) {
        KernelTimer t(ctx, KC_RADIX_PASS);
        PassParams P;
        P.chunk = chunk;
        P.keys[0] = s->keys[0].p;
        P.keys[1] = s->keys[1].p;
        P.idx[0] = s->idx[0].p;
        P.idx[1] = s->idx[1].p;
        P.digit_base = s->offsets.p + (size_t)plan_index * kRadix;
        P.status = s->status.p + (size_t)slot * tiles * kRadix;
        P.counter = s->counters.p + counter;
        P.plan = s->plan.p;
        P.plan_index = plan_index;
        P.shift = shift;
        P.n = (u32)n;
        P.prefix_sel = hp.prefix_sel;
        P.prefix_mask = hp.prefix_mask;
        P.copy16 = (((uintptr_t)chunk | (uintptr_t)P.keys[0] | (uintptr_t)P.keys[1]) & 15) == 0;
        v.kernel<<<v.tiles(n), kSortThreads, v.smem, st>>>(P);
    };
    SortPlan hp{};  // host copy of the plan (read_plan only)
    if (read_plan) {
        YTGPU_CUDA_TRY(cudaMemcpyAsync(&hp, s->plan.p, sizeof(SortPlan), cudaMemcpyDeviceToHost, st));
        YTGPU_CUDA_TRY(cudaStreamSynchronize(st));
        int active = 0;
        for (int p = 0; p < kPassesPerChunk; ++p) active += hp.pass[p].active;
        YTGPU_CUDA_TRY(cudaMemsetAsync(s->status.p, 0, (size_t)active * tiles * kRadix * 4, st));
        int k = 0;
        for (int p = 0; p < kPassesPerChunk; ++p) {
            if (!hp.pass[p].active) continue;
            // packed: the k-th pass sorts by prefix byte k, or k + 1 when byte 0 is left to the tail (run_shift == 8)
            const int shift = hp.packed ? 32 + (int)hp.run_shift + k * kRadixBits : p * kRadixBits;
            launch_pass(hp.packed ? kPackedPass : kPairPass, chunks[0], p, k, p, shift, hp);
            ++k;
        }
    } else {
        for (int r = nchunks - 1; r >= 0; --r) {
            YTGPU_CUDA_TRY(cudaMemsetAsync(s->status.p, 0, (size_t)kPassesPerChunk * tiles * kRadix * 4, st));
            for (int p = 0; p < kPassesPerChunk; ++p)
                launch_pass(kPairPass, chunks[r], r * kPassesPerChunk + p, p, r * kPassesPerChunk + p, p * kRadixBits, hp);
        }
    }
    s->rows_gathered = false;
    if (hp.hybrid) {
        // hybrid tail: order the short runs of equal prefixes, classify the long ones.  The three-pass packed schedule's
        // tail also moves the rows when the caller asked for them (SortScratch::gather).
        const bool gather = s->gather.rows && hp.packed && hp.run_shift == 8 && s->gather.row_bytes / 16 <= kTailGatherMaxGranules;
        TailGather tg{};
        if (gather) {
            const u32 gr = s->gather.row_bytes / 16;
            tg.rows = reinterpret_cast<const uint4*>(s->gather.rows);
            tg.out = reinterpret_cast<uint4*>(s->gather.out);
            tg.gr_magic = (u32)(((1ull << 31) + gr - 1) / gr);
            tg.gr = gr;
            tg.write_idx = s->gather.want_perm ? 1 : 0;
        }
        DevBuf<u32> mixedmask, longlist;
        DevBuf<HybridSummary> summary;
        DevBuf<MixedRun> mixedlist;
        YTGPU_TRY(mixedmask.allocate(ctx, n / 32 + 2));
        YTGPU_TRY(longlist.allocate(ctx, n / 32 + 2));
        YTGPU_TRY(summary.allocate(ctx, 1));
        YTGPU_TRY(mixedlist.allocate(ctx, kMixedCap));
        YTGPU_CUDA_TRY(cudaMemsetAsync(summary.p, 0, sizeof(HybridSummary), st));
        {
            const u32 blocks = (u32)std::min<u64>((n + 255) / 256, (u64)kNumSms * 8);
            auto classify = hp.packed ? classify_long_runs_kernel<true> : classify_long_runs_kernel<false>;
            if (hp.run_shift) {
                // the prefixes are in the permutation buffer the last pass did not write
                u32* idx = s->idx[hp.final_idx].p;
                const u32* pre = s->idx[hp.final_idx ^ 1].p;
                const u32 tail_blocks = (u32)((n + kRunTile - 1) / kRunTile);
                if (gather) {
                    KernelTimer t(ctx, KC_GATHER);
                    tie_fix_runs_kernel<true><<<tail_blocks, 256, 0, st>>>(chunks[0], pre, idx, (u32)n, mixedmask.p, longlist.p, summary.p, tg);
                } else {
                    KernelTimer t(ctx, KC_HISTOGRAM);
                    tie_fix_runs_kernel<false><<<tail_blocks, 256, 0, st>>>(chunks[0], pre, idx, (u32)n, mixedmask.p, longlist.p, summary.p, tg);
                }
            } else {
                KernelTimer t(ctx, KC_HISTOGRAM);
                auto tie_fix = hp.packed ? tie_fix_kernel<true> : tie_fix_kernel<false>;
                tie_fix<<<blocks, 256, 0, st>>>(s->plan.p, chunks[0], s->keys[0].p, s->keys[1].p, s->idx[0].p, s->idx[1].p, (u32)n,
                                                mixedmask.p, longlist.p, summary.p);
            }
            KernelTimer t(ctx, KC_HISTOGRAM);
            classify<<<kNumSms * 4, 256, 0, st>>>(s->plan.p, s->keys[0].p, s->keys[1].p, s->idx[0].p, s->idx[1].p, (u32)n, mixedmask.p,
                                                  longlist.p, summary.p, mixedlist.p);
        }
        YTGPU_CUDA_TRY(cudaGetLastError());
        // the hybrid schedule's second host round trip (sorts below kHybridMinRows rows never take the hybrid schedule)
        HybridSummary hs{};
        YTGPU_CUDA_TRY(cudaMemcpyAsync(&hs, summary.p, sizeof(hs), cudaMemcpyDeviceToHost, st));
        YTGPU_CUDA_TRY(cudaStreamSynchronize(st));
        if (hs.hybrid && hs.mixed_count > 0) {
            if (hs.mixed_count > kMixedCap || hs.mixed_elems > n / 8) {
                // Clustered keys: the chunk is sorted again with the plain schedule over every active digit, from the
                // counts still in `hist`.  The re-sort allocates the other buffers of `s` again: the stream-ordered pool
                // hands back the blocks just freed, so the peak footprint does not grow.  It leaves the rows to the
                // caller (rows_gathered = false), so rows the tail moved in the wrong order are gathered again.
                s->no_hybrid = true;
                YTGPU_TRY(radix_sort_chunks(ctx, chunks, 1, n, s, out));
                ctx->last_sort_hybrid_passes = hp.active_passes;  // after the re-sort, whose own accounting clears it
                return Status{};
            }
            YTGPU_TRY(sort_mixed_runs(ctx, s, hs, mixedlist.p, hp.packed ? chunks[0] : nullptr, gather ? &tg : nullptr));
        }
        s->rows_gathered = gather;
    }
    YTGPU_CUDA_TRY(cudaGetLastError());
    YTGPU_CUDA_TRY(cudaMemcpyAsync(ctx->host_err + 1, &s->plan.p->active_passes, 4, cudaMemcpyDeviceToHost, st));
    ctx->last_sort_hybrid_passes = 0;
    out->plan = s->plan.p;
    out->idx[0] = s->idx[0].p;
    out->idx[1] = s->idx[1].p;
    return Status{};
}

// ---------------------------------------------------------------------------------------------
// Multi-chunk keys: sort by a synthetic prefix chunk made of the 8 most significant ACTIVE bytes.
// ---------------------------------------------------------------------------------------------
namespace {

struct PrefixSel {
    u8 chunk[8];   // source chunk of prefix byte j (j = 0 most significant)
    u8 digit[8];   // digit (byte index, 0 = least significant) inside that chunk
    u32 count;     // bytes selected (< 8 when the key has fewer active bytes)
    u32 complete;  // every active byte of the key is part of the prefix: equal prefixes == equal keys
    u32 mixed_long_run;  // set by deep_tie_fix_kernel: the complete schedule has to run
};

// One block: a digit is active when no single bin holds all n keys.  hist holds RAW counts here.
__global__ void __launch_bounds__(256) select_prefix_kernel(const u32* __restrict__ hist, int nchunks, u32 n, PrefixSel* sel) {
    __shared__ u8 s_active[kMaxKeyChunks * kPassesPerChunk];
    const int total = nchunks * kPassesPerChunk;
    for (int rp = 0; rp < total; ++rp) {
        const int full = __syncthreads_or(hist[rp * kRadix + threadIdx.x] == n);
        if (threadIdx.x == 0) s_active[rp] = !full;
    }
    __syncthreads();
    if (threadIdx.x != 0) return;
    u32 cnt = 0, active = 0;
    for (int c = 0; c < nchunks; ++c)
        for (int p = kPassesPerChunk - 1; p >= 0; --p) {  // most significant byte of the key first
            if (!s_active[c * kPassesPerChunk + p]) continue;
            ++active;
            if (cnt < 8) {
                sel->chunk[cnt] = (u8)c;
                sel->digit[cnt] = (u8)p;
                ++cnt;
            }
        }
    sel->count = cnt;
    sel->complete = active <= 8;
    sel->mixed_long_run = 0;
}

struct ChunkList {
    const u64* p[kMaxKeyChunks];
};

// H[i] = the selected bytes of row i, most significant first; + the digit histogram of H (input of its sort).
__global__ void __launch_bounds__(256) build_prefix_chunk_kernel(const ChunkList chunks, const PrefixSel* __restrict__ sel, u64 n,
                                                                 u64* __restrict__ out, u32* __restrict__ hist) {
    __shared__ u32 sh[kPassesPerChunk * kRadix];
    __shared__ PrefixSel s_sel;
    for (int i = threadIdx.x; i < kPassesPerChunk * kRadix; i += 256) sh[i] = 0;
    if (threadIdx.x == 0) s_sel = *sel;
    __syncthreads();
    const u32 cnt = s_sel.count;
    const u64 stride = (u64)gridDim.x * blockDim.x;
    for (u64 base = (u64)blockIdx.x * blockDim.x; base < n; base += stride) {  // warp-uniform trips (hist_accumulate)
        const u64 i = base + threadIdx.x;
        const bool valid = i < n;
        u64 h = 0;
        if (valid) {
            u32 last_chunk = 0xffffffffu;
            u64 w = 0;
            for (u32 j = 0; j < cnt; ++j) {
                const u32 c = s_sel.chunk[j];
                if (c != last_chunk) {
                    w = ld_stream_u64(chunks.p[c] + i);
                    last_chunk = c;
                }
                h |= ((w >> (8 * s_sel.digit[j])) & 0xff) << (8 * (7 - j));
            }
            out[i] = h;
        }
        hist_accumulate(sh, h, valid);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kPassesPerChunk * kRadix; i += 256) {
        const u32 c = sh[i];
        if (c) atomicAdd(&hist[i], c);
    }
}

__device__ __forceinline__ int compare_full_keys(const ChunkList& chunks, int nchunks, u32 a, u32 b) {
    for (int c = 0; c < nchunks; ++c) {
        const u64 x = chunks.p[c][a], y = chunks.p[c][b];
        if (x != y) return x < y ? -1 : 1;
    }
    return 0;
}

// After the prefix chunk is sorted: rows whose prefixes tie are ordered by their full keys.  Same structure as
// tie_fix_kernel — the run-start thread insertion-sorts a short run (only the permutation moves: the prefixes are equal);
// a run longer than kMaxTieRun is fine when all of its full keys are equal, adjacent different keys inside a long run
// request the complete schedule.  Full keys are read through the permutation (random 8-byte loads), so a table made of
// few distinct composite keys pays ~2 extra passes' worth of traffic here; keys that differ inside the prefix pay nothing.
__global__ void __launch_bounds__(256) deep_tie_fix_kernel(const SortPlan* plan, const u64* chunk_h, const u64* keys0, const u64* keys1,
                                                           u32* idx0, u32* idx1, const ChunkList chunks, int nchunks, PrefixSel* sel, u32 n) {
    if (sel->complete) return;
    const u32 fk = plan_final_key(plan);
    const u64* keys = fk == 2 ? chunk_h : (fk ? keys1 : keys0);
    const u32 fi = plan->final_idx;
    u32* idx = fi ? idx1 : idx0;  // fi == 2 (identity, no pass ran) means every prefix is equal: handled as one long run
    const u32 lane = threadIdx.x & 31;
    for (u64 base = (u64)blockIdx.x * blockDim.x; base < n; base += (u64)gridDim.x * blockDim.x) {
        const u64 i64 = base + threadIdx.x;
        const bool in = i64 < n;
        const u32 i = (u32)i64;
        const u64 h = in ? keys[i] : 0;
        u64 prev = __shfl_up_sync(0xffffffffu, h, 1);
        u64 next = __shfl_down_sync(0xffffffffu, h, 1);
        if (!in) continue;
        if (lane == 0) prev = i > 0 ? keys[i - 1] : ~h;
        if (lane == 31 || i + 1 >= n) next = i + 1 < n ? keys[i + 1] : ~h;
        if (i > 0 && prev == h) {
            const u32 a = fi == 2 ? i - 1 : idx[i - 1], b = fi == 2 ? i : idx[i];
            if (compare_full_keys(chunks, nchunks, a, b) != 0) {
                u32 s = i;
                while (s > 0 && i - s < (u32)kMaxTieRun && keys[s - 1] == h) --s;
                bool long_run = i - s >= (u32)kMaxTieRun;
                if (!long_run) {
                    u32 e = i + 1;
                    while (e < n && e - s <= (u32)kMaxTieRun && keys[e] == h) ++e;
                    long_run = e - s > (u32)kMaxTieRun;
                }
                if (long_run || fi == 2) sel->mixed_long_run = 1;
            }
            continue;
        }
        if (next != h || fi == 2) continue;
        u32 len = 2;
        while (i + len < n && len <= (u32)kMaxTieRun && keys[i + len] == h) ++len;
        if (len > (u32)kMaxTieRun) continue;
        for (u32 a = 1; a < len; ++a) {  // stable insertion sort of the permutation by the full key
            const u32 v = idx[i + a];
            u32 b = a;
            while (b > 0 && compare_full_keys(chunks, nchunks, idx[i + b - 1], v) > 0) {
                idx[i + b] = idx[i + b - 1];
                --b;
            }
            idx[i + b] = v;
        }
    }
}

}  // namespace

Status radix_sort_keys(Context* ctx, const u64* const* chunks, int nchunks, u64 n, SortScratch* s, PermRef* out) {
    if (nchunks == 1 || n < 2) return radix_sort_chunks(ctx, chunks, nchunks, n, s, out);
    // 1. raw digit counts of every chunk (the complete schedule needs them as well)
    YTGPU_TRY(sort_setup(ctx, chunks, nchunks, n, s));
    cudaStream_t st = ctx->stream;
    // 2. prefix chunk of the 8 most significant active bytes + its histogram
    DevBuf<PrefixSel> sel;
    DevBuf<u64> hchunk;
    SortScratch hs;
    YTGPU_TRY(sel.allocate(ctx, 1));
    YTGPU_TRY(hchunk.allocate(ctx, n));
    YTGPU_TRY(prepare_histogram(ctx, 1, &hs));
    ChunkList cl{};
    for (int c = 0; c < nchunks; ++c) cl.p[c] = chunks[c];
    {
        KernelTimer t(ctx, KC_EXTRACT, 2);
        select_prefix_kernel<<<1, 256, 0, st>>>(s->hist.p, nchunks, (u32)n, sel.p);
        const u32 blocks = (u32)std::min<u64>((n + 255) / 256, (u64)kNumSms * 8);
        build_prefix_chunk_kernel<<<blocks, 256, 0, st>>>(cl, sel.p, n, hchunk.p, hs.hist.p);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    hs.hist_precomputed = true;
    hs.keep_keys = true;
    // 3. sort it (hybrid schedule and all), then order the rows whose prefixes tie
    PermRef hperm;
    const u64* hptr[1] = {hchunk.p};
    YTGPU_TRY(radix_sort_chunks(ctx, hptr, 1, n, &hs, &hperm));
    {
        KernelTimer t(ctx, KC_HISTOGRAM);
        const u32 blocks = (u32)std::min<u64>((n + 255) / 256, (u64)kNumSms * 8);
        deep_tie_fix_kernel<<<blocks, 256, 0, st>>>(hs.plan.p, hchunk.p, hs.keys[0].p, hs.keys[1].p, hs.idx[0].p, hs.idx[1].p, cl, nchunks, sel.p,
                                                    (u32)n);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    // 4. the one host round trip of the multi-chunk path: did a long run of equal prefixes mix different keys?
    PrefixSel hsel;
    YTGPU_CUDA_TRY(cudaMemcpyAsync(&hsel, sel.p, sizeof(PrefixSel), cudaMemcpyDeviceToHost, st));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(st));
    if (hsel.mixed_long_run) return radix_sort_chunks(ctx, chunks, nchunks, n, s, out);  // complete LSD over every active byte
    // hand the prefix sort's buffers over to the caller's scratch (they hold the permutation)
    s->plan = std::move(hs.plan);
    s->idx[0] = std::move(hs.idx[0]);
    s->idx[1] = std::move(hs.idx[1]);
    out->plan = s->plan.p;
    out->idx[0] = s->idx[0].p;
    out->idx[1] = s->idx[1].p;
    return Status{};
}

Status prepare_histogram(Context* ctx, int nchunks, SortScratch* s) {
    const size_t words = (size_t)nchunks * kPassesPerChunk * kRadix;
    YTGPU_TRY(s->hist.allocate(ctx, words));
    YTGPU_CUDA_TRY(cudaMemsetAsync(s->hist.p, 0, words * 4, ctx->stream));
    return Status{};
}

Status materialize_perm(Context* ctx, const PermRef& perm, u64 n, u32* dst_dev) {
    if (n == 0) return Status{};
    u32 blocks = (u32)std::min<u64>((n + 255) / 256, (u64)kNumSms * 8);
    materialize_perm_kernel<<<blocks, 256, 0, ctx->stream>>>(perm.plan, perm.idx[0], perm.idx[1], n, dst_dev);
    ctx->count_launch();
    YTGPU_CUDA_TRY(cudaGetLastError());
    return Status{};
}

}  // namespace ytgpu
