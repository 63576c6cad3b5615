// column_writer.cu — columnar write side (SURVEY.md §8(f) rank 3): rows -> integer column -> scan-optimised segments.
//
// ytgpu_convert_integer_column  : TIntegerColumnConverter<T>::Convert, library/column_converters/integer_column_converter.cpp:69-161
// ytgpu_encode_integer_column   : TUnversionedIntegerColumnWriter<T>, ytlib/table_chunk_format/integer_column_writer.cpp:318-590
//
// The reference walks the values once on one core, keeping min/max, a hash map value -> first-seen id and a run counter,
// then re-walks them to emit the chosen layout.  Here every segment of the column is processed at once:
//   1. stats    : encode (zig-zag), per-segment min/max (block reduce + one atomic), and a per-segment open-addressing
//                 table value -> smallest row index holding it — the "first seen" order without any order of
//                 execution; a slot is one 64-bit word (fingerprint, row index), see kEmptySlot below;
//   2. flags    : per row (run start, is first occurrence) packed in one u64, exclusive scan over the column: the scan
//                 at a first occurrence IS its dictionary id, the scan at a run start IS its run index;
//   3. scatter  : dictionary entries and run starts land at their ranks;
//   4. decide   : one thread per segment evaluates the four size estimates and picks the layout (first minimum in enum
//                 order), a serial prefix gives the data offsets;
//   5. pack     : one thread per OUTPUT word composes it from the elements that overlap it (headers, bit-packed
//                 payloads, bitmaps) — no atomics, no zero-fill pass, every word written exactly once.
// HBM-bound integer work; algorithmic bytes per row: 8 (+1) read, (width/8 + 1/8) written for a DirectDense segment.
#include <algorithm>
#include <vector>

#include "context.cuh"
#include "scan.cuh"

using namespace ytgpu;

namespace {

constexpr u32 kNone = 0xffffffffu;
constexpr int kStatThreads = 256;
constexpr int kStatRowsPerBlock = 2048;
constexpr u64 kRowsPerBlock = 2048;  // flags / scatter kernels

struct SegStats {
    u64 vmin;  // init ~0
    u64 vmax;  // init 0
};

// Per-segment open-addressing table.  A slot is ONE 64-bit word: (32-bit fingerprint of the value << 32) | index of a
// row of the segment that holds the value — the value itself is not stored, it is read back through that row.  Once a
// slot is claimed (CAS from empty) it belongs to one value for good; the only later change is atomicMin lowering the
// row index, so the word converges to (fingerprint, FIRST row with that value).  One atomic per new value, none for a
// duplicate that comes after the recorded row (the common case: rows are visited in roughly increasing order).
constexpr u64 kEmptySlot = ~0ull;

__device__ __forceinline__ u64 zigzag_enc(i64 v) { return ((u64)v << 1) ^ (u64)(v >> 63); }
__device__ __forceinline__ u32 width_of(u64 v) { return v == 0 ? 0u : 64u - (u32)__clzll((long long)v); }
__device__ __forceinline__ u64 packed_bytes(u64 max_value, u64 count) { return 8ull * (1ull + (((u64)width_of(max_value) * count + 63ull) >> 6)); }
__device__ __forceinline__ u64 mix64(u64 x) {
    x ^= x >> 33;
    x *= 0xff51afd7ed558ccdull;
    x ^= x >> 33;
    return x;
}

__global__ void __launch_bounds__(256) init_stats_kernel(SegStats* stats, u32 nseg) {
    for (u32 s = blockIdx.x * blockDim.x + threadIdx.x; s < nseg; s += gridDim.x * blockDim.x) stats[s] = SegStats{~0ull, 0ull};
}

// 1. stats: blocks_per_seg consecutive blocks cover one segment.
__global__ void __launch_bounds__(kStatThreads) stats_kernel(const u64* __restrict__ raw, const u8* __restrict__ nulls, u64 n,
                                                            int is_signed, u32 max_values, u32 blocks_per_seg,
                                                            u64* __restrict__ enc, SegStats* __restrict__ stats,
                                                            u64* table, u32 cap) {
    const u32 s = blockIdx.x / blocks_per_seg, b = blockIdx.x % blocks_per_seg;
    const u64 seg_begin = (u64)s * max_values;
    const u64 seg_rows = min((u64)max_values, n - seg_begin);
    u64* slots = table + (u64)s * cap;
    const u32 mask = cap - 1;
    u64 lmin = ~0ull, lmax = 0;
    const u64 lo = (u64)b * kStatRowsPerBlock, hi = min(seg_rows, lo + kStatRowsPerBlock);
    for (u64 i = lo + threadIdx.x; i < hi; i += kStatThreads) {
        const u64 g = seg_begin + i;
        const bool nl = nulls && nulls[g];
        u64 e = 0;
        if (!nl) {
            e = is_signed ? zigzag_enc((i64)raw[g]) : raw[g];
            lmin = min(lmin, e);
            lmax = max(lmax, e);
            const u64 mx = mix64(e);
            const u32 fp = (u32)(mx >> 32);
            const u64 want = ((u64)fp << 32) | (u64)i;
            u32 h = (u32)mx & mask;
            for (;;) {
                u64 cur = *reinterpret_cast<volatile u64*>(slots + h);
                if (cur == kEmptySlot) {
                    cur = atomicCAS((unsigned long long*)&slots[h], (unsigned long long)kEmptySlot, (unsigned long long)want);
                    if (cur == kEmptySlot) break;  // claimed: this row is (so far) the first with its value
                }
                if ((u32)(cur >> 32) == fp) {
                    // same fingerprint: compare the VALUE through the row the slot points at (the input is immutable)
                    const u32 j = (u32)cur;
                    const u64 other = is_signed ? zigzag_enc((i64)raw[seg_begin + j]) : raw[seg_begin + j];
                    if (other == e) {
                        if ((u32)i < j) atomicMin((unsigned long long*)&slots[h], (unsigned long long)want);
                        break;
                    }
                }
                h = (h + 1) & mask;
            }
        }
        enc[g] = e;
    }
    // block reduce min/max
    __shared__ u64 s_min[kStatThreads / 32], s_max[kStatThreads / 32];
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        lmin = min(lmin, __shfl_xor_sync(0xffffffffu, lmin, o));
        lmax = max(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
    }
    if ((threadIdx.x & 31) == 0) {
        s_min[threadIdx.x >> 5] = lmin;
        s_max[threadIdx.x >> 5] = lmax;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kStatThreads / 32; ++w) {
            lmin = min(lmin, s_min[w]);
            lmax = max(lmax, s_max[w]);
        }
        if (lmin != ~0ull || lmax != 0) {  // at least one non-null value (or only zeros, which change nothing but are harmless)
            atomicMin((unsigned long long*)&stats[s].vmin, (unsigned long long)lmin);
            atomicMax((unsigned long long*)&stats[s].vmax, (unsigned long long)lmax);
        }
    }
}

// 2. flags: low 32 bits = "this row is the first occurrence of its value in the segment", high = "this row starts a run".
__global__ void __launch_bounds__(256) flags_kernel(const u64* __restrict__ enc, const u8* __restrict__ nulls, u64 n, u32 max_values,
                                                    const u64* __restrict__ table, u32 cap, u32* __restrict__ first_of,
                                                    u64* __restrict__ flags) {
    const u32 mask = cap - 1;
    // consecutive blocks take consecutive row ranges: the blocks in flight probe the tables of a few neighbouring segments
    // (L2-resident) instead of all of them
    const u64 lo = (u64)blockIdx.x * kRowsPerBlock, hi = min(n + 1, lo + kRowsPerBlock);
    for (u64 g = lo + threadIdx.x; g < hi; g += blockDim.x) {
        if (g == n) {
            flags[g] = 0;  // sentinel so that scan[n] is the grand total
            break;
        }
        const u32 s = (u32)(g / max_values);
        const u32 i = (u32)(g - (u64)s * max_values);
        const bool nl = nulls && nulls[g];
        const u64 e = enc[g];
        bool run_start = i == 0;
        if (!run_start) {
            const bool pnl = nulls && nulls[g - 1];
            run_start = pnl != nl || enc[g - 1] != e;
        }
        u32 f = kNone;
        if (!nl) {
            const u64* slots = table + (u64)s * cap;
            const u64 seg_begin = (u64)s * max_values;
            const u64 mx = mix64(e);
            const u32 fp = (u32)(mx >> 32);
            u32 h = (u32)mx & mask;
            for (;;) {  // the value was inserted by stats_kernel, so the probe ends at its slot
                const u64 w = slots[h];
                if ((u32)(w >> 32) == fp && w != kEmptySlot && enc[seg_begin + (u32)w] == e) {
                    f = (u32)w;
                    break;
                }
                h = (h + 1) & mask;
            }
        }
        first_of[g] = f;
        flags[g] = ((u64)run_start << 32) | (u64)(f == i);
    }
}

// 3. scatter dictionary entries and run starts to their ranks (segment-relative slots in row-sized scratch arrays).
__global__ void __launch_bounds__(256) scatter_kernel(const u64* __restrict__ enc, const u64* __restrict__ scan, u64 n, u32 max_values,
                                                      const SegStats* __restrict__ stats, const u32* __restrict__ first_of,
                                                      u64* __restrict__ dict, u32* __restrict__ run_start) {
    const u64 lo = (u64)blockIdx.x * kRowsPerBlock, hi = min(n, lo + kRowsPerBlock);
    for (u64 g = lo + threadIdx.x; g < hi; g += blockDim.x) {
        const u32 s = (u32)(g / max_values);
        const u64 begin = (u64)s * max_values;
        const u32 i = (u32)(g - begin);
        const u64 here = scan[g], next = scan[g + 1], base = scan[begin];
        if ((u32)next != (u32)here) dict[begin + (u32)(here - base)] = enc[g] - stats[s].vmin;          // first occurrence
        if ((next >> 32) != (here >> 32)) run_start[begin + (u32)((here >> 32) - (base >> 32))] = i;   // run start
    }
}

struct SegWork {  // device-side companion of the public descriptor
    u32 distinct, runs;
    u64 word_offset;  // first output word of the segment
};

// 4. decide: sizes (integer_column_writer.cpp:353-381), layout choice (:493-496), part sizes; then offsets.
__global__ void __launch_bounds__(256) decide_kernel(const u64* __restrict__ scan, u64 n, u32 max_values, u32 nseg, u64 chunk_row_offset,
                                                     const SegStats* __restrict__ stats, const u32* __restrict__ run_start,
                                                     ytgpu_integer_segment* __restrict__ segs, SegWork* __restrict__ work,
                                                     u64* __restrict__ total_bytes) {
    for (u32 s = threadIdx.x; s < nseg; s += blockDim.x) {
        const u64 begin = (u64)s * max_values;
        const u64 count = min((u64)max_values, n - begin);
        const u64 a = scan[begin], b = scan[begin + count];
        const u64 nd = (u32)(b - a);
        const u64 runs = (u32)((b >> 32) - (a >> 32));
        const u64 chunk_rows = chunk_row_offset + begin + count;
        const u64 range = stats[s].vmax - stats[s].vmin;  // wraps to 1 when the segment holds no value, as the reference does
        const i32 sizes[4] = {
            (i32)(packed_bytes(range, nd) + packed_bytes(nd + 1, runs) + packed_bytes(chunk_rows, runs)),
            (i32)(packed_bytes(range, nd) + packed_bytes(nd + 1, count)),
            (i32)(packed_bytes(range, runs) + packed_bytes(chunk_rows, runs) + runs / 8),
            (i32)(packed_bytes(range, count) + count / 8),
        };
        u32 type = 0;
        for (u32 t = 1; t < 4; ++t)
            if (sizes[t] < sizes[type]) type = t;
        ytgpu_integer_segment d{};
        d.type = type;
        d.row_count = (u32)count;
        d.chunk_row_count = chunk_rows;
        d.min_value = stats[s].vmin;
        d.direct = type >= 2;
        d.values_width = (u8)width_of(range);
        const u64 last_run = run_start[begin + runs - 1];
        if (type == 3) {
            d.values_size = (u32)count;
            d.part_bytes[0] = packed_bytes(range, count);
            d.part_bytes[1] = 8 * ((count + 63) / 64);
        } else if (type == 1) {
            d.values_size = (u32)nd;
            d.ids_size = (u32)count;
            d.ids_width = (u8)width_of(nd + 1);
            d.part_bytes[0] = packed_bytes(range, nd);
            d.part_bytes[1] = packed_bytes(nd + 1, count);
        } else if (type == 2) {
            d.values_size = (u32)runs;
            d.row_indexes_size = (u32)runs;
            d.row_indexes_width = (u8)width_of(last_run);
            d.part_bytes[0] = packed_bytes(range, runs);
            d.part_bytes[1] = 8 * ((runs + 63) / 64);
            d.part_bytes[2] = packed_bytes(last_run, runs);
        } else {
            d.values_size = (u32)nd;
            d.ids_size = (u32)runs;
            d.ids_width = (u8)width_of(nd + 1);
            d.row_indexes_size = (u32)runs;
            d.row_indexes_width = (u8)width_of(last_run);
            d.part_bytes[0] = packed_bytes(range, nd);
            d.part_bytes[1] = packed_bytes(nd + 1, runs);
            d.part_bytes[2] = packed_bytes(last_run, runs);
        }
        d.data_bytes = d.part_bytes[0] + d.part_bytes[1] + d.part_bytes[2];
        segs[s] = d;
        work[s].distinct = (u32)nd;
        work[s].runs = (u32)runs;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        u64 at = 0;
        for (u32 s = 0; s < nseg; ++s) {
            segs[s].data_offset = at;
            work[s].word_offset = at / 8;
            at += segs[s].data_bytes;
        }
        work[nseg].word_offset = at / 8;
        *total_bytes = at;
    }
}

struct PackArgs {
    const u64* enc;
    const u8* nulls;
    const u32* first_of;
    const u64* scan;
    const u64* dict;
    const u32* run_start;
    const ytgpu_integer_segment* segs;
    const SegWork* work;
    u32 nseg, max_values;
    u64 total_words;
};

enum PartKind { PK_DENSE_VALUES, PK_DICT, PK_DENSE_IDS, PK_RLE_VALUES, PK_RLE_IDS, PK_ROW_INDEXES, PK_DENSE_NULLS, PK_RLE_NULLS };

__device__ __forceinline__ u64 part_elem(const PackArgs& a, u64 begin, u64 vmin, int kind, u64 j) {
    switch (kind) {
        case PK_DENSE_VALUES: {
            const u64 g = begin + j;
            return (a.nulls && a.nulls[g]) ? 0 : a.enc[g] - vmin;
        }
        case PK_DICT: return a.dict[begin + j];
        case PK_RLE_VALUES: {
            const u64 g = begin + a.run_start[begin + j];
            return (a.nulls && a.nulls[g]) ? 0 : a.enc[g] - vmin;
        }
        case PK_DENSE_IDS:
        case PK_RLE_IDS: {
            const u64 g = kind == PK_DENSE_IDS ? begin + j : begin + a.run_start[begin + j];
            const u32 f = a.first_of[g];
            return f == kNone ? 0 : (u64)(u32)(a.scan[begin + f] - a.scan[begin]) + 1;
        }
        case PK_ROW_INDEXES: return a.run_start[begin + j];
        case PK_DENSE_NULLS: return (a.nulls && a.nulls[begin + j]) ? 1 : 0;
        default: return (a.nulls && a.nulls[begin + a.run_start[begin + j]]) ? 1 : 0;  // PK_RLE_NULLS
    }
}

// 5. pack: one thread per output word.
__global__ void __launch_bounds__(256) pack_kernel(PackArgs a, u64* __restrict__ out) {
    for (u64 w = (u64)blockIdx.x * blockDim.x + threadIdx.x; w < a.total_words; w += (u64)gridDim.x * blockDim.x) {
        // segment holding word w: last s with work[s].word_offset <= w
        u32 lo = 0, hi = a.nseg;
        while (hi - lo > 1) {
            const u32 mid = (lo + hi) >> 1;
            if (a.work[mid].word_offset <= w) lo = mid;
            else hi = mid;
        }
        const u32 s = lo;
        const ytgpu_integer_segment& d = a.segs[s];
        u64 lw = w - a.work[s].word_offset;
        int p = 0;
        while (lw >= d.part_bytes[p] / 8) {
            lw -= d.part_bytes[p] / 8;
            ++p;
        }
        const u64 begin = (u64)s * a.max_values;
        int kind;
        u64 count;
        u32 width;
        bool bitmap = false;
        if (d.type == 3) {
            kind = p == 0 ? PK_DENSE_VALUES : PK_DENSE_NULLS;
            count = d.row_count;
            width = d.values_width;
            bitmap = p == 1;
        } else if (d.type == 1) {
            kind = p == 0 ? PK_DICT : PK_DENSE_IDS;
            count = p == 0 ? d.values_size : d.ids_size;
            width = p == 0 ? d.values_width : d.ids_width;
        } else if (d.type == 2) {
            kind = p == 0 ? PK_RLE_VALUES : (p == 1 ? PK_RLE_NULLS : PK_ROW_INDEXES);
            count = d.values_size;
            width = p == 0 ? d.values_width : d.row_indexes_width;
            bitmap = p == 1;
        } else {
            kind = p == 0 ? PK_DICT : (p == 1 ? PK_RLE_IDS : PK_ROW_INDEXES);
            count = p == 0 ? d.values_size : d.ids_size;
            width = p == 0 ? d.values_width : (p == 1 ? d.ids_width : d.row_indexes_width);
        }
        u64 word = 0;
        if (bitmap) {
            const u64 j0 = lw * 64, j1 = min(count, j0 + 64);
            for (u64 j = j0; j < j1; ++j) word |= part_elem(a, begin, d.min_value, kind, j) << (j - j0);
        } else if (lw == 0) {
            word = count | ((u64)width << 56);
        } else {
            const u64 bit0 = (lw - 1) * 64;  // this word covers payload bits [bit0, bit0 + 64)
            for (u64 j = bit0 / width; j < count && j * width < bit0 + 64; ++j) {
                const u64 v = part_elem(a, begin, d.min_value, kind, j);
                const i64 pos = (i64)(j * width) - (i64)bit0;
                word |= pos >= 0 ? (v << pos) : (v >> (-pos));
            }
        }
        out[w] = word;
    }
}

inline u32 grid_for(u64 items, int threads, int per_sm) {
    return (u32)std::max<u64>(1, std::min<u64>((items + threads - 1) / threads, (u64)kNumSms * per_sm));
}

Status encode_impl(Context* ctx, const u64* values, const u8* null_bytemap, u64 n, int is_signed, u32 max_values, u64 chunk_row_offset,
                   int mem, u8* out_data, u64 out_capacity, u64* out_bytes, ytgpu_integer_segment* out_segments, u32 seg_capacity,
                   u32* out_seg_count) {
    if (!out_bytes || !out_seg_count) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    *out_bytes = 0;
    *out_seg_count = 0;
    if (max_values == 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "max_segment_value_count must be positive");
    if (n == 0) return Status{};
    if (!values) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null values");
    if (n >= (1ull << 32)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "one call encodes fewer than 2^32 rows");
    const u64 nseg64 = (n + max_values - 1) / max_values;
    if (nseg64 > (1u << 24)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "too many segments (%llu)", (unsigned long long)nseg64);
    const u32 nseg = (u32)nseg64;
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));

    InBuf<u64> raw;
    InBuf<u8> staged_nulls;
    YTGPU_TRY(raw.stage(ctx, values, n, mem));
    YTGPU_TRY(staged_nulls.stage(ctx, null_bytemap, n, mem));
    const u8* nulls = staged_nulls.p;

    // per-segment table: power of two >= 2 x rows of a segment
    const u64 seg_rows = std::min<u64>(max_values, n);
    u32 cap = 8;
    while ((u64)cap < 2 * seg_rows) cap <<= 1;
    const u32 blocks_per_seg = (u32)((seg_rows + kStatRowsPerBlock - 1) / kStatRowsPerBlock);

    DevBuf<u64> enc, flags, dict, table, sums, total;
    DevBuf<u32> first_of, run_start;
    DevBuf<SegStats> stats;
    DevBuf<ytgpu_integer_segment> segs;
    DevBuf<SegWork> work;
    YTGPU_TRY(enc.allocate(ctx, n));
    YTGPU_TRY(flags.allocate(ctx, n + 1));
    YTGPU_TRY(dict.allocate(ctx, n));
    YTGPU_TRY(first_of.allocate(ctx, n));
    YTGPU_TRY(run_start.allocate(ctx, n));
    YTGPU_TRY(table.allocate(ctx, (u64)nseg * cap));
    YTGPU_TRY(stats.allocate(ctx, nseg));
    YTGPU_TRY(segs.allocate(ctx, nseg));
    YTGPU_TRY(work.allocate(ctx, nseg + 1));
    YTGPU_TRY(sums.allocate(ctx, scan_block_count(n + 1)));
    YTGPU_TRY(total.allocate(ctx, 2));
    YTGPU_CUDA_TRY(cudaMemsetAsync(table.p, 0xff, (u64)nseg * cap * 8, ctx->stream));
    {
        KernelTimer t(ctx, KC_DECODE, 7);
        init_stats_kernel<<<grid_for(nseg, 256, 4), 256, 0, ctx->stream>>>(stats.p, nseg);
        stats_kernel<<<nseg * blocks_per_seg, kStatThreads, 0, ctx->stream>>>(raw.p, nulls, n, is_signed, max_values, blocks_per_seg, enc.p,
                                                                             stats.p, table.p, cap);
        flags_kernel<<<(u32)((n + kRowsPerBlock) / kRowsPerBlock), 256, 0, ctx->stream>>>(enc.p, nulls, n, max_values, table.p, cap, first_of.p,
                                                                                         flags.p);
        exclusive_scan_u64(ctx->stream, flags.p, n + 1, sums.p, total.p);
        scatter_kernel<<<(u32)((n + kRowsPerBlock - 1) / kRowsPerBlock), 256, 0, ctx->stream>>>(enc.p, flags.p, n, max_values, stats.p, first_of.p, dict.p, run_start.p);
        decide_kernel<<<1, 256, 0, ctx->stream>>>(flags.p, n, max_values, nseg, chunk_row_offset, stats.p, run_start.p, segs.p, work.p,
                                                  total.p + 1);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    u64 bytes = 0;
    YTGPU_CUDA_TRY(cudaMemcpyAsync(&bytes, total.p + 1, 8, cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    *out_bytes = bytes;
    *out_seg_count = nseg;
    if (!out_segments || nseg > seg_capacity)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "column needs %u segment descriptors, capacity is %u", nseg, seg_capacity);
    if (!out_data || bytes > out_capacity)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "column data needs %llu bytes, capacity is %llu", (unsigned long long)bytes,
                           (unsigned long long)out_capacity);
    YTGPU_CUDA_TRY(cudaMemcpyAsync(out_segments, segs.p, (size_t)nseg * sizeof(ytgpu_integer_segment), cudaMemcpyDeviceToHost, ctx->stream));

    if (mem != YTGPU_MEM_HOST && (reinterpret_cast<uintptr_t>(out_data) & 7))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "out_data must be 8-byte aligned");
    OutBuf<u64> dst;
    YTGPU_TRY(dst.prepare(ctx, reinterpret_cast<u64*>(out_data), bytes / 8, mem));
    PackArgs args{enc.p, nulls, first_of.p, flags.p, dict.p, run_start.p, segs.p, work.p, nseg, max_values, bytes / 8};
    {
        KernelTimer t(ctx, KC_DECODE, 1);
        pack_kernel<<<grid_for(bytes / 8, 256, 8), 256, 0, ctx->stream>>>(args, dst.p);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_TRY(dst.download(ctx, bytes / 8));  // segment data are whole words
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return Status{};
}

// ---- rows -> column (TIntegerColumnConverter) ----
__global__ void __launch_bounds__(256) convert_kernel(const ytgpu_value* __restrict__ values, u64 nrows, u32 value_count, u32 column,
                                                      u8 value_type, u64* __restrict__ out_values, u64* __restrict__ out_bitmap,
                                                      u32* __restrict__ dev_err) {
    // one thread per row; a warp's ballot gives 32 bitmap bits, lane 0 / lane 16... -> simpler: two ballots per u64 word
    const u64 words = (nrows + 63) / 64;
    for (u64 w = (u64)blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5); w < words; w += (u64)gridDim.x * (blockDim.x / 32)) {
        const u32 lane = threadIdx.x & 31;
        u64 bits = 0;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const u64 r = w * 64 + half * 32 + lane;
            bool nl = false;
            if (r < nrows) {
                const uint4 rawv = *reinterpret_cast<const uint4*>(values + r * value_count + column);
                const u8 type = (u8)((rawv.x >> 16) & 0xff);
                const u64 data = ((u64)rawv.w << 32) | rawv.z;
                u64 word = 0;
                if (type == YTGPU_TYPE_NULL) {
                    nl = true;
                } else if (type != value_type) {
                    atomicOr(dev_err, DE_SCHEMA_VIOLATION);
                } else {
                    const u64 e = value_type == YTGPU_TYPE_INT64 ? zigzag_enc((i64)data) : data;
                    word = e - ~0ull;  // MinValue_ stays 2^64-1 in the reference (integer_column_converter.cpp:139-161)
                }
                out_values[r] = word;
            }
            const u32 b = __ballot_sync(0xffffffffu, nl);
            bits |= (u64)b << (32 * half);
        }
        if (lane == 0) out_bitmap[w] = bits;
    }
}

Status convert_impl(Context* ctx, const ytgpu_rowset_view* rows, u32 column, u8 value_type, u64* out_values, u8* out_bitmap,
                    u64* out_base, int out_mem) {
    if (!rows || !out_values || !out_bitmap || !out_base) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    if (value_type != YTGPU_TYPE_INT64 && value_type != YTGPU_TYPE_UINT64)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "integer column converter takes Int64 or Uint64");
    if (column >= rows->value_count) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "column index out of range");
    *out_base = ~0ull;
    const u64 n = rows->row_count;
    if (n == 0) return Status{};
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    const u64 words = (n + 63) / 64;
    InBuf<ytgpu_value> vals;
    OutBuf<u64> ov, ob;
    YTGPU_TRY(vals.stage(ctx, rows->values, n * rows->value_count, rows->mem));
    YTGPU_TRY(ov.prepare(ctx, out_values, n, out_mem));
    YTGPU_TRY(ob.prepare(ctx, reinterpret_cast<u64*>(out_bitmap), words, out_mem));
    {
        KernelTimer t(ctx, KC_DECODE, 1);
        convert_kernel<<<grid_for(words * 32, 256, 8), 256, 0, ctx->stream>>>(vals.p, n, rows->value_count, column, value_type, ov.p, ob.p,
                                                                              ctx->dev_err);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_TRY(ov.download(ctx, n));
    YTGPU_TRY(ob.download(ctx, words));
    return check_device_errors(ctx);
}

}  // namespace

extern "C" {

int ytgpu_convert_integer_column(ytgpu_context* h, const ytgpu_rowset_view* rows, uint32_t column_index, uint8_t value_type,
                                 uint64_t* out_values, uint8_t* out_null_bitmap, uint64_t* out_base_value, int out_mem,
                                 ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, convert_impl(as_context(h), rows, column_index, value_type, out_values, out_null_bitmap, out_base_value, out_mem));
}

int ytgpu_encode_integer_column(ytgpu_context* h, const uint64_t* values, const uint8_t* null_bytemap, uint64_t row_count,
                                int is_signed, uint32_t max_segment_value_count, uint64_t chunk_row_offset, int mem,
                                uint8_t* out_data, uint64_t out_capacity, uint64_t* out_data_bytes,
                                ytgpu_integer_segment* out_segments, uint32_t segment_capacity, uint32_t* out_segment_count,
                                ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, encode_impl(as_context(h), values, null_bytemap, row_count, is_signed, max_segment_value_count,
                                       chunk_row_offset, mem, out_data, out_capacity, out_data_bytes, out_segments, segment_capacity,
                                       out_segment_count));
}

}  // extern "C"
