// columnar_flags.cu — the null / dictionary-index helpers of the column readers
// (yt/yt/client/table_client/columnar.h:13-200, columnar.cpp:60-768): validity bitmaps, null bytemaps, dictionary
// indexes, null / one counts, total string length and RLE index translation.
//
// The reference walks rows sequentially with a run cursor (BuildBitmapFromRleImpl :137-194, BuildBytemapFromRleImpl
// :196-241).  Here every thread owns a fixed chunk of OUTPUT (one 32-bit bitmap word, eight bytemap bytes), so no output
// word is shared between threads (no atomics, no zero fill) and runs longer than a chunk cost one step.  A warp walks a
// contiguous share of the output front to back: ONE binary search over the runs per warp, every later lookup gallops
// forward from the previous one (a binary search per trip is a chain of ~20 dependent loads at 10^6 runs and made these
// kernels latency bound).  Dictionary indexes addressed directly become bitmap bytes through 16-byte loads and one
// shuffle per load.  Counts over RLE sources are sums over RUNS, not rows.
#include "columnar.cuh"
#include "context.cuh"

using namespace ytgpu;

namespace {

struct FlagSrc {
    int kind;
    const void* data;
    u64 data_count;
    const u64* rle;
    u64 rle_count;
};

constexpr u64 kNoThreshold = ~0ull;

__device__ __forceinline__ bool value_flag(const FlagSrc& s, u64 k) {
    return s.kind == YTGPU_FLAGS_DICTIONARY_ZERO ? __ldg(static_cast<const u32*>(s.data) + k) == 0
                                                 : raw_bit_at(static_cast<const u8*>(s.data), k);
}

// Flags of successive rows starting at `row`.
template <bool RLE>
struct FlagCursor {
    const FlagSrc& s;
    u64 row, run, run_end;
    bool cur;
    // run_hint: a run known to start at or before first_row (kNoRleHint: binary search)
    __device__ __forceinline__ FlagCursor(const FlagSrc& src, u64 first_row, u64 run_hint = kNoRleHint)
        : s(src), row(first_row), run(0), run_end(0), cur(false) {
        if (RLE) {
            run = run_hint == kNoRleHint ? rle_pos(s.rle, s.rle_count, first_row) : rle_pos_gallop(s.rle, s.rle_count, first_row, run_hint);
            run_end = run + 1 < s.rle_count ? __ldg(s.rle + run + 1) : kNoThreshold;
            cur = value_flag(s, run);
        }
    }
    // rows left in the current run (RLE only)
    __device__ __forceinline__ u64 run_left() const { return run_end - row; }
    __device__ __forceinline__ void skip(u64 rows) { row += rows; }
    __device__ __forceinline__ bool next() {
        if (!RLE) return value_flag(s, row++);
        if (row >= run_end) {
            do {  // run starts are strictly increasing in what the writers produce; an empty run is stepped over
                ++run;
                run_end = run + 1 < s.rle_count ? __ldg(s.rle + run + 1) : kNoThreshold;
            } while (row >= run_end);
            cur = value_flag(s, run);
        }
        ++row;
        return cur;
    }
};

// The run holding the first row of lane 0, found once per warp: the chunks of a warp are neighbours, so every lane
// reaches its own run by a short walk from there (rle_pos_from) instead of a binary search over all runs.
// All 32 lanes must call; lane 0's row must be valid.
// `prev`: the hint of the warp's previous trip (the warp walks its share of the output front to back, so the next
// search starts where the last one ended); kNoRleHint on the first trip = one binary search per warp.
__device__ __forceinline__ u64 warp_run_hint(const u64* __restrict__ rle, u64 rle_count, u64 lane0_row, u64 prev) {
    u64 k = 0;
    if (lane_id() == 0) k = prev == kNoRleHint ? rle_pos(rle, rle_count, lane0_row) : rle_pos_gallop(rle, rle_count, lane0_row, prev);
    return __shfl_sync(0xffffffffu, k, 0);
}

// The share of `units` output pieces one warp walks front to back: [*begin, *end), whole multiples of 32 except at the tail.
__device__ __forceinline__ void warp_share(u64 units, u64* begin, u64* end) {
    const u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5, warps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u64 per_warp = ((units + warps * 32 - 1) / (warps * 32)) * 32;
    *begin = min(units, warp * per_warp);
    *end = min(units, *begin + per_warp);
}

// 32 bits of a bitmap starting at bit `p`; bits at or beyond `nbits` read as 0.  Byte loads: any alignment.
__device__ __forceinline__ u32 read_bits32(const u8* __restrict__ bm, u64 nbits, u64 p) {
    if (p >= nbits) return 0;
    const u64 nbytes = (nbits + 7) >> 3, b = p >> 3;
    u64 v = 0;
#pragma unroll
    for (int j = 0; j < 5; ++j)
        if (b + j < nbytes) v |= (u64)__ldg(bm + b + j) << (8 * j);
    u32 w = (u32)(v >> (p & 7));
    const u64 valid = nbits - p;
    if (valid < 32) w &= (1u << valid) - 1;
    return w;
}

__device__ __forceinline__ void store_bitmap_word(u8* __restrict__ dst, u64 word_index, u32 w, u64 bits_total) {
    const u64 nbytes = (bits_total + 7) >> 3, b0 = word_index * 4;
    if (b0 + 4 <= nbytes && ((reinterpret_cast<uintptr_t>(dst) & 3) == 0)) {
        reinterpret_cast<u32*>(dst)[word_index] = w;
        return;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j)
        if (b0 + j < nbytes) dst[b0 + j] = (u8)(w >> (8 * j));
}

// Dictionary indexes addressed directly: a warp turns 1024 rows into 32 words (one coalesced load + one ballot per word).
__global__ void __launch_bounds__(256) dict_bitmap_kernel(const u32* __restrict__ idx, u64 start, u64 end, u32 negate,
                                                          u8* __restrict__ dst) {
    const u64 bits = end - start, words = (bits + 31) >> 5;
    const u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5, warps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u32 lane = lane_id();
    for (u64 w0 = warp * 32; w0 < words; w0 += warps * 32) {
        u32 mine = 0;
#pragma unroll 4
        for (u32 j = 0; j < 32; ++j) {
            const u64 r = (w0 + j) * 32 + lane;
            if ((w0 + j) * 32 >= bits) break;  // warp-uniform
            const bool f = r < bits && ((ld_stream_u32(idx + start + r) == 0) != (negate != 0));
            const u32 b = __ballot_sync(0xffffffffu, f);
            if (j == lane) mine = b;
        }
        if (w0 + lane < words) store_bitmap_word(dst, w0 + lane, mine, bits);
    }
}

// The same when the first index is 16-byte aligned: a warp step turns 256 rows into 32 bytes — two coalesced 16-byte loads
// per lane (rows 4l.. and 128 + 4l..), each lane's four flags form a nibble, neighbouring lanes exchange nibbles (one
// shuffle per load) so that even lanes hold the bytes of the first 128 rows and odd lanes those of the second.
__global__ void __launch_bounds__(256) dict_bitmap_vec_kernel(const uint4* __restrict__ idx4, u64 rows, u32 negate, u8* __restrict__ dst) {
    const u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5, warps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u32 lane = lane_id();
    const u64 full = rows / 256;  // whole 256-row steps; the caller finishes the tail with the generic kernel
    const u32 flip = negate ? 0xFu : 0u;
    for (u64 step = warp; step < full; step += warps) {
        const uint4 a = ld_stream_u128(idx4 + step * 64 + lane), b = ld_stream_u128(idx4 + step * 64 + 32 + lane);
        const u32 na = ((u32)(a.x == 0) | (u32)(a.y == 0) << 1 | (u32)(a.z == 0) << 2 | (u32)(a.w == 0) << 3) ^ flip;
        const u32 nb = ((u32)(b.x == 0) | (u32)(b.y == 0) << 1 | (u32)(b.z == 0) << 2 | (u32)(b.w == 0) << 3) ^ flip;
        const u32 pa = __shfl_xor_sync(0xffffffffu, na, 1), pb = __shfl_xor_sync(0xffffffffu, nb, 1);
        const u32 byte = (lane & 1) ? (pb | nb << 4) : (na | pa << 4);
        dst[step * 32 + (lane & 1) * 16 + (lane >> 1)] = (u8)byte;
    }
}

// One output word per thread: bitmap -> bitmap (shifted copy) and every RLE source.
template <bool RLE>
__global__ void __launch_bounds__(256) flags_bitmap_kernel(const FlagSrc s, u64 start, u64 end, u32 negate, u8* __restrict__ dst) {
    const u64 bits = end - start, words = (bits + 31) >> 5;
    // warp-uniform trip count: the run hint is a warp-wide exchange
    u64 share_begin, share_end, hint = kNoRleHint;
    warp_share(words, &share_begin, &share_end);
    for (u64 base = share_begin; base < share_end; base += 32) {
        if (RLE) hint = warp_run_hint(s.rle, s.rle_count, start + base * 32, hint);
        const u64 w = base + lane_id();
        if (w >= words) continue;
        const u64 r0 = w * 32;
        const u32 n = (u32)min((u64)32, bits - r0);
        u32 word = 0;
        if (!RLE && s.kind == YTGPU_FLAGS_BITMAP) {
            word = read_bits32(static_cast<const u8*>(s.data), end, start + r0);
        } else {
            FlagCursor<RLE> c(s, start + r0, hint);
            u32 done = 0;
            while (done < n) {
                if (RLE && c.row < c.run_end) {  // the rest of the current run in one step
                    const u32 take = (u32)min((u64)(n - done), c.run_left());
                    if (c.cur) word |= (take == 32 ? ~0u : ((1u << take) - 1)) << done;
                    c.skip(take);
                    done += take;
                } else {
                    if (c.next()) word |= 1u << done;
                    ++done;
                }
            }
        }
        if (negate) word = ~word;
        if (n < 32) word &= (1u << n) - 1;
        store_bitmap_word(dst, w, word, bits);
    }
}

// Eight bytemap bytes per thread.
template <bool RLE>
__global__ void __launch_bounds__(256) flags_bytemap_kernel(const FlagSrc s, u64 start, u64 end, u32 negate, u8* __restrict__ dst) {
    const u64 rows = end - start, chunks = (rows + 7) >> 3;
    const bool aligned = (reinterpret_cast<uintptr_t>(dst) & 7) == 0;
    u64 share_begin, share_end, hint = kNoRleHint;
    warp_share(chunks, &share_begin, &share_end);
    for (u64 base = share_begin; base < share_end; base += 32) {
        if (RLE) hint = warp_run_hint(s.rle, s.rle_count, start + base * 8, hint);
        const u64 t = base + lane_id();
        if (t >= chunks) continue;
        const u64 r0 = t * 8;
        const u32 n = (u32)min((u64)8, rows - r0);
        u64 packed = 0;
        if (!RLE && s.kind == YTGPU_FLAGS_BITMAP) {
            const u32 w = read_bits32(static_cast<const u8*>(s.data), end, start + r0);
#pragma unroll
            for (u32 j = 0; j < 8; ++j) packed |= (u64)((w >> j) & 1) << (8 * j);
        } else {
            FlagCursor<RLE> c(s, start + r0, hint);
            if (RLE && c.run_left() >= n) {
                packed = c.cur ? 0x0101010101010101ull : 0;
            } else {
                for (u32 j = 0; j < n; ++j) packed |= (u64)c.next() << (8 * j);
            }
        }
        if (negate) packed ^= 0x0101010101010101ull;
        if (n == 8 && aligned) {
            reinterpret_cast<u64*>(dst)[t] = packed;
        } else {
            for (u32 j = 0; j < n; ++j) dst[r0 + j] = (u8)(packed >> (8 * j));
        }
    }
}

// dst[i] = idx[i] - 1 (direct): four per thread when both sides are 16-byte aligned, else one.
__global__ void __launch_bounds__(256) dict_minus_one_kernel(const u32* __restrict__ idx, u64 n, u32* __restrict__ dst) {
    const bool vec = ((reinterpret_cast<uintptr_t>(idx) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0;
    const u64 tid = (u64)blockIdx.x * blockDim.x + threadIdx.x, nth = (u64)gridDim.x * blockDim.x;
    if (vec) {
        for (u64 q = tid; q < (n >> 2); q += nth) {
            uint4 v = ld_stream_u128(reinterpret_cast<const uint4*>(idx) + q);
            v.x -= 1; v.y -= 1; v.z -= 1; v.w -= 1;
            reinterpret_cast<uint4*>(dst)[q] = v;
        }
        for (u64 i = (n & ~3ull) + tid; i < n; i += nth) dst[i] = idx[i] - 1;
    } else {
        for (u64 i = tid; i < n; i += nth) dst[i] = idx[i] - 1;
    }
}

// RLE: a warp step covers 128 consecutive rows, lane l taking rows l, l + 32, l + 64, l + 96 of it — consecutive lanes
// store consecutive words, and the four run lookups of a lane are independent loads in flight together.
// idx == nullptr: the run number counted from the run that holds `start`.
__global__ void __launch_bounds__(256) rle_dict_indexes_kernel(const u32* __restrict__ idx, const u64* __restrict__ rle, u64 rle_count,
                                                               u64 start, u64 end, u32* __restrict__ dst) {
    __shared__ u64 s_first_run;
    if (threadIdx.x == 0) s_first_run = rle_pos(rle, rle_count, start);
    __syncthreads();
    const u64 first_run = s_first_run;
    const u64 rows = end - start, steps = (rows + 127) >> 7;
    const u64 warp = ((u64)blockIdx.x * blockDim.x + threadIdx.x) >> 5, warps = ((u64)gridDim.x * blockDim.x) >> 5;
    const u64 per_warp = (steps + warps - 1) / warps;
    const u64 step_begin = min(steps, warp * per_warp), step_end = min(steps, step_begin + per_warp);
    u64 hint = kNoRleHint;
    for (u64 st = step_begin; st < step_end; ++st) {
        hint = warp_run_hint(rle, rle_count, start + st * 128, hint);
        u64 run[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const u64 r = st * 128 + (u64)k * 32 + lane_id();
            run[k] = r < rows ? rle_pos_gallop(rle, rle_count, start + r, hint) : hint;
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const u64 r = st * 128 + (u64)k * 32 + lane_id();
            if (r < rows) dst[r] = idx ? __ldg(idx + run[k]) - 1 : (u32)(run[k] - first_run);
        }
    }
}

__device__ __forceinline__ void block_add(unsigned long long v, unsigned long long* out) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    if (lane_id() == 0 && v) atomicAdd(out, v);
}

// Direct sources: one 32-row chunk per thread step.
__global__ void __launch_bounds__(256) count_direct_kernel(const FlagSrc s, u64 start, u64 end, unsigned long long* out) {
    unsigned long long acc = 0;
    const u64 tid = (u64)blockIdx.x * blockDim.x + threadIdx.x, nth = (u64)gridDim.x * blockDim.x;
    if (s.kind == YTGPU_FLAGS_DICTIONARY_ZERO) {
        const u32* idx = static_cast<const u32*>(s.data);
        u64 first = start;
        if ((reinterpret_cast<uintptr_t>(idx + start) & 15) == 0) {  // 16-byte loads over the aligned body
            const uint4* idx4 = reinterpret_cast<const uint4*>(idx + start);
            const u64 quads = (end - start) >> 2;
            for (u64 q = tid; q < quads; q += nth) {
                const uint4 v = ld_stream_u128(idx4 + q);
                acc += (v.x == 0) + (v.y == 0) + (v.z == 0) + (v.w == 0);
            }
            first = start + quads * 4;
        }
        for (u64 i = first + tid; i < end; i += nth) acc += ld_stream_u32(idx + i) == 0;
    } else {
        const u8* bm = static_cast<const u8*>(s.data);
        for (u64 p = start + tid * 32; p < end; p += nth * 32) acc += __popc(read_bits32(bm, end, p));
    }
    block_add(acc, out);
}

// RLE sources: a sum over the runs that intersect [start, end).  lengths != nullptr: total string length
// (CountTotalStringLengthInRleDictionaryIndexesWithZeroNull) — the run's rows times the length of its dictionary string.
__global__ void __launch_bounds__(256) count_rle_kernel(const FlagSrc s, u64 start, u64 end, const i32* __restrict__ lengths,
                                                        u64 string_count, unsigned long long* out, u32* dev_err) {
    __shared__ u64 s_runs[2];
    if (threadIdx.x == 0) {
        s_runs[0] = rle_pos(s.rle, s.rle_count, start);
        s_runs[1] = rle_pos(s.rle, s.rle_count, end - 1);
    }
    __syncthreads();
    const u64 first = s_runs[0], last = s_runs[1];
    unsigned long long acc = 0;
    for (u64 k = first + (u64)blockIdx.x * blockDim.x + threadIdx.x; k <= last; k += (u64)gridDim.x * blockDim.x) {
        const u64 lo = max(start, __ldg(s.rle + k));
        const u64 hi = k + 1 < s.rle_count ? min(end, __ldg(s.rle + k + 1)) : end;
        const u64 rows = hi > lo ? hi - lo : 0;
        if (lengths) {
            const u32 d = __ldg(static_cast<const u32*>(s.data) + k);
            if (d != 0) {
                if (d - 1 >= string_count) atomicOr(dev_err, DE_PART_OUT_OF_BOUNDS);
                else acc += rows * (unsigned long long)(long long)__ldg(lengths + d - 1);
            }
        } else if (value_flag(s, k)) {
            acc += rows;
        }
    }
    block_add(acc, out);
}

__global__ void __launch_bounds__(256) translate_rle_kernel(const u64* __restrict__ rle, u64 rle_count, const i64* __restrict__ indexes,
                                                            u64 n, int end_flavour, i64* __restrict__ out) {
    for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (u64)gridDim.x * blockDim.x) {
        const i64 x = indexes[j];
        i64 r;
        if (end_flavour) r = x <= 0 ? 0 : (i64)rle_pos(rle, rle_count, (u64)(x - 1)) + 1;  // TranslateRleEndIndex :759-768
        else r = x < 0 ? -1 : (i64)rle_pos(rle, rle_count, (u64)x);
        out[j] = r;
    }
}

// The first run start must be 0 (YT_VERIFY(rleIndexes[0] == 0)).
__global__ void check_rle_kernel(const u64* __restrict__ rle, u32* dev_err) {
    if (rle[0] != 0) atomicOr(dev_err, DE_SCHEMA_VIOLATION);
}

inline unsigned grid_for(u64 items, unsigned per_block) {
    const u64 blocks = (items + per_block - 1) / per_block;
    return (unsigned)std::max<u64>(1, std::min<u64>(blocks, (u64)kNumSms * 16));
}

// A flag source staged on the device (HOST flavour copies the arrays in).
struct StagedSource {
    FlagSrc dev{};
    InBuf<u8> data;
    InBuf<u64> rle;
};

Status validate_source(const ytgpu_flag_source* src, i64 start, i64 end, bool need_rle = false) {
    if (!src) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null flag source");
    if (src->kind != YTGPU_FLAGS_DICTIONARY_ZERO && src->kind != YTGPU_FLAGS_BITMAP)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "unknown flag source kind %d", src->kind);
    if (start < 0 || start > end) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "bad row range [%lld, %lld)", (long long)start, (long long)end);
    if (need_rle && !src->rle_indexes) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "rle_indexes required");
    if (src->rle_indexes) {
        if (src->rle_count == 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "empty rle_indexes");
        if (src->data_count < src->rle_count) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "fewer values than runs");
    } else if ((u64)end > src->data_count) {
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "row range ends past the source (%lld > %llu)", (long long)end,
                           (unsigned long long)src->data_count);
    }
    if (!src->data && src->data_count) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null source data");
    return Status{};
}

Status stage_source(Context* ctx, const ytgpu_flag_source* src, int mem, StagedSource* st) {
    const size_t bytes = src->kind == YTGPU_FLAGS_DICTIONARY_ZERO ? (size_t)src->data_count * 4 : (size_t)((src->data_count + 7) >> 3);
    YTGPU_TRY(st->data.stage(ctx, static_cast<const u8*>(src->data), bytes, mem));
    if (mem == YTGPU_MEM_HOST) {
        if (src->rle_indexes && src->rle_indexes[0] != 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "rle_indexes[0] != 0");
    } else if (src->rle_indexes) {
        check_rle_kernel<<<1, 1, 0, ctx->stream>>>(src->rle_indexes, ctx->dev_err);
        YTGPU_CUDA_TRY(cudaGetLastError());
        ctx->count_launch();
    }
    YTGPU_TRY(st->rle.stage(ctx, src->rle_indexes, src->rle_count, mem));
    st->dev.kind = src->kind;
    st->dev.data = st->data.p;
    st->dev.data_count = src->data_count;
    st->dev.rle = st->rle.p;
    st->dev.rle_count = src->rle_indexes ? src->rle_count : 0;
    return Status{};
}

Status build_map_impl(Context* ctx, const ytgpu_flag_source* src, i64 start, i64 end, int negate, u8* dst, int mem, bool bitmap) {
    YTGPU_TRY(validate_source(src, start, end));
    const u64 rows = (u64)(end - start);
    if (rows == 0) return Status{};
    if (!dst) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null dst");
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    StagedSource st;
    YTGPU_TRY(stage_source(ctx, src, mem, &st));
    const size_t out_bytes = bitmap ? (size_t)((rows + 7) >> 3) : (size_t)rows;
    OutBuf<u8> out;
    YTGPU_TRY(out.prepare(ctx, dst, out_bytes, mem));
    u8* o = out.p;
    {
        KernelTimer t(ctx, KC_DECODE);
        const bool rle = st.dev.rle != nullptr;
        if (bitmap) {
            if (!rle && st.dev.kind == YTGPU_FLAGS_DICTIONARY_ZERO) {
                const u32* first = static_cast<const u32*>(st.dev.data) + start;
                u64 done = 0;  // rows handled by the vector kernel (a multiple of 256, so the tail starts on a byte boundary)
                if ((reinterpret_cast<uintptr_t>(first) & 15) == 0 && rows >= 256) {
                    done = rows / 256 * 256;
                    dict_bitmap_vec_kernel<<<grid_for(done / 256, 8), 256, 0, ctx->stream>>>(reinterpret_cast<const uint4*>(first), done,
                                                                                            (u32)(negate != 0), o);
                    ctx->count_launch();
                }
                if (done < rows)
                    dict_bitmap_kernel<<<grid_for((rows - done + 31) / 32, 8 * 32), 256, 0, ctx->stream>>>(
                        static_cast<const u32*>(st.dev.data), (u64)start + done, (u64)end, (u32)(negate != 0), o + done / 8);
            }
            else if (rle) flags_bitmap_kernel<true><<<grid_for((rows + 31) / 32, 256), 256, 0, ctx->stream>>>(st.dev, (u64)start, (u64)end, (u32)(negate != 0), o);
            else flags_bitmap_kernel<false><<<grid_for((rows + 31) / 32, 256), 256, 0, ctx->stream>>>(st.dev, (u64)start, (u64)end, (u32)(negate != 0), o);
        } else {
            if (rle) flags_bytemap_kernel<true><<<grid_for((rows + 7) / 8, 256), 256, 0, ctx->stream>>>(st.dev, (u64)start, (u64)end, (u32)(negate != 0), o);
            else flags_bytemap_kernel<false><<<grid_for((rows + 7) / 8, 256), 256, 0, ctx->stream>>>(st.dev, (u64)start, (u64)end, (u32)(negate != 0), o);
        }
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    if (mem == YTGPU_MEM_HOST) {
        YTGPU_TRY(out.download(ctx, out_bytes));
        YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    } else if (st.dev.rle) {
        Status s = check_device_errors(ctx);  // rle_indexes[0] != 0 on the device
        if (!s.ok()) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "rle_indexes[0] != 0");
    }
    return Status{};
}

// Runs `launch(counter)` and returns the 64-bit counter to the host.
template <class F>
Status run_count(Context* ctx, i64* out, F&& launch) {
    DevBuf<unsigned long long> counter;
    YTGPU_TRY(counter.allocate(ctx, 1));
    YTGPU_CUDA_TRY(cudaMemsetAsync(counter.p, 0, 8, ctx->stream));
    {
        KernelTimer t(ctx, KC_DECODE);
        launch(counter.p);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    unsigned long long host = 0;
    YTGPU_CUDA_TRY(cudaMemcpyAsync(&host, counter.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
    Status s = check_device_errors(ctx);  // synchronises the stream
    if (!s.ok()) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "malformed rle / dictionary indexes: %s", s.msg);
    *out = (i64)host;
    return Status{};
}

}  // namespace

extern "C" {

int ytgpu_build_bitmap_from_flags(ytgpu_context* h, const ytgpu_flag_source* source, int64_t start_index, int64_t end_index,
                                  int negate, uint8_t* dst, int mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, build_map_impl(as_context(h), source, start_index, end_index, negate, dst, mem, true));
}

int ytgpu_build_bytemap_from_flags(ytgpu_context* h, const ytgpu_flag_source* source, int64_t start_index, int64_t end_index,
                                   int negate, uint8_t* dst, int mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, build_map_impl(as_context(h), source, start_index, end_index, negate, dst, mem, false));
}

int ytgpu_count_flags(ytgpu_context* h, const ytgpu_flag_source* source, int64_t start_index, int64_t end_index,
                      int64_t* out_count, int mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    Context* ctx = as_context(h);
    auto run = [&]() -> Status {
        YTGPU_TRY(validate_source(source, start_index, end_index));
        if (!out_count) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null out_count");
        *out_count = 0;
        if (start_index == end_index) return Status{};
        YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
        StagedSource st;
        YTGPU_TRY(stage_source(ctx, source, mem, &st));
        const u64 s = (u64)start_index, e = (u64)end_index;
        return run_count(ctx, out_count, [&](unsigned long long* counter) {
            if (st.dev.rle)
                count_rle_kernel<<<grid_for(std::min<u64>(st.dev.rle_count, e - s), 256), 256, 0, ctx->stream>>>(st.dev, s, e, nullptr, 0, counter,
                                                                                                                  ctx->dev_err);
            else
                count_direct_kernel<<<grid_for(st.dev.kind == YTGPU_FLAGS_BITMAP ? (e - s + 31) / 32 : e - s, 256 * 4), 256, 0, ctx->stream>>>(
                    st.dev, s, e, counter);
        });
    };
    return fill_error(err, run());
}

int ytgpu_build_dictionary_indexes(ytgpu_context* h, const uint32_t* dictionary_indexes, uint64_t dictionary_index_count,
                                   const uint64_t* rle_indexes, uint64_t rle_count, int64_t start_index, int64_t end_index,
                                   uint32_t* dst, int mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    Context* ctx = as_context(h);
    auto run = [&]() -> Status {
        if (!dictionary_indexes && !rle_indexes) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "dictionary_indexes or rle_indexes required");
        ytgpu_flag_source src{};
        src.kind = YTGPU_FLAGS_DICTIONARY_ZERO;
        src.data = dictionary_indexes;
        src.data_count = dictionary_indexes ? dictionary_index_count : rle_count;
        src.rle_indexes = rle_indexes;
        src.rle_count = rle_count;
        if (dictionary_indexes) {
            YTGPU_TRY(validate_source(&src, start_index, end_index));
        } else {
            if (start_index < 0 || start_index > end_index) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "bad row range");
            if (rle_count == 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "empty rle_indexes");
        }
        const u64 rows = (u64)(end_index - start_index);
        if (rows == 0) return Status{};
        if (!dst) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null dst");
        YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
        StagedSource st;
        if (dictionary_indexes) {
            YTGPU_TRY(stage_source(ctx, &src, mem, &st));
        } else {  // iota: only the run starts are needed
            src.data = rle_indexes;  // placeholder so that the staging code has something to copy
            src.kind = YTGPU_FLAGS_BITMAP;
            src.data_count = 0;
            YTGPU_TRY(stage_source(ctx, &src, mem, &st));
        }
        OutBuf<u32> o;
        YTGPU_TRY(o.prepare(ctx, dst, rows, mem));
        {
            KernelTimer t(ctx, KC_DECODE);
            const u32* idx = dictionary_indexes ? static_cast<const u32*>(st.dev.data) : nullptr;
            if (st.dev.rle) rle_dict_indexes_kernel<<<grid_for((rows + 127) / 128, 8), 256, 0, ctx->stream>>>(idx, st.dev.rle, st.dev.rle_count,
                                                                                                            (u64)start_index, (u64)end_index, o.p);
            else dict_minus_one_kernel<<<grid_for(rows, 256 * 4), 256, 0, ctx->stream>>>(idx + start_index, rows, o.p);
            YTGPU_CUDA_TRY(cudaGetLastError());
        }
        if (mem == YTGPU_MEM_HOST) {
            YTGPU_TRY(o.download(ctx, rows));
            YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
        } else if (st.dev.rle) {
            Status s = check_device_errors(ctx);
            if (!s.ok()) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "rle_indexes[0] != 0");
        }
        return Status{};
    };
    return fill_error(err, run());
}

int ytgpu_count_total_string_length(ytgpu_context* h, const uint32_t* dictionary_indexes, const uint64_t* rle_indexes,
                                    uint64_t rle_count, const int32_t* string_lengths, uint64_t string_count,
                                    int64_t start_index, int64_t end_index, int64_t* out_total, int mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    Context* ctx = as_context(h);
    auto run = [&]() -> Status {
        ytgpu_flag_source src{};
        src.kind = YTGPU_FLAGS_DICTIONARY_ZERO;
        src.data = dictionary_indexes;
        src.data_count = rle_count;
        src.rle_indexes = rle_indexes;
        src.rle_count = rle_count;
        YTGPU_TRY(validate_source(&src, start_index, end_index, true));
        if (!out_total || (!string_lengths && string_count)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
        *out_total = 0;
        if (start_index == end_index) return Status{};
        YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
        StagedSource st;
        YTGPU_TRY(stage_source(ctx, &src, mem, &st));
        InBuf<i32> dlen;
        YTGPU_TRY(dlen.stage(ctx, string_lengths, string_count, mem));
        const i32* lengths = dlen.p;
        static const i32 kNoLengths = 0;
        if (!lengths) lengths = &kNoLengths;  // never read: every index is out of range and reported
        const u64 s = (u64)start_index, e = (u64)end_index;
        return run_count(ctx, out_total, [&](unsigned long long* counter) {
            count_rle_kernel<<<grid_for(std::min<u64>(st.dev.rle_count, e - s), 256), 256, 0, ctx->stream>>>(st.dev, s, e, lengths, string_count,
                                                                                                              counter, ctx->dev_err);
        });
    };
    return fill_error(err, run());
}

int ytgpu_translate_rle_indexes(ytgpu_context* h, const uint64_t* rle_indexes, uint64_t rle_count, const int64_t* indexes,
                                uint64_t count, int end_flavour, int64_t* out, int mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    Context* ctx = as_context(h);
    auto run = [&]() -> Status {
        if (!rle_indexes || rle_count == 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "empty rle_indexes");
        if (count == 0) return Status{};
        if (!indexes || !out) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
        YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
        if (mem == YTGPU_MEM_HOST) {
            if (rle_indexes[0] != 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "rle_indexes[0] != 0");
            for (u64 j = 0; j < count; ++j)
                if (indexes[j] < 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "negative index");
        }
        InBuf<u64> r;
        InBuf<i64> q;
        OutBuf<i64> o;
        YTGPU_TRY(r.stage(ctx, rle_indexes, rle_count, mem));
        YTGPU_TRY(q.stage(ctx, indexes, count, mem));
        YTGPU_TRY(o.prepare(ctx, out, count, mem));
        {
            KernelTimer t(ctx, KC_DECODE);
            translate_rle_kernel<<<grid_for(count, 256), 256, 0, ctx->stream>>>(r.p, rle_count, q.p, count, end_flavour, o.p);
            YTGPU_CUDA_TRY(cudaGetLastError());
        }
        if (mem == YTGPU_MEM_HOST) {
            YTGPU_TRY(o.download(ctx, count));
            YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
        }
        return Status{};
    };
    return fill_error(err, run());
}

}  // extern "C"
