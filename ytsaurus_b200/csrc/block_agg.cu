// block_agg.cu — YQL block aggregators, "combine all" form (SURVEY.md §8 a18 / (f) rank 4):
//   IBlockAggregatorCombineAll::AddMany   yql/essentials/minikql/comp_nodes/mkql_block_agg_factory.h:34-45
//   sum / avg                              mkql_block_agg_sum.cpp:160-232, 421-485
//   min / max (fixed width)                mkql_block_agg_minmax.cpp:20-52 (AggLess: NaN is the biggest), 697-770
//   count / count_all                      mkql_block_agg_count.cpp
// The reference runs one aggregator per pass over an Arrow array; here ONE pass over the array produces every
// fixed-width aggregate at once (sum, count, count_all, min, max): 8 bytes of value + 1 filter byte + 1 validity bit
// read per row, nothing written — a pure HBM-bound reduction.  Per-block partials are combined by a second, single
// block in a fixed order, so floating-point sums are reproducible for a given array length.
#include <algorithm>
#include <cmath>
#include <cstring>

#include "context.cuh"

using namespace ytgpu;

namespace {

constexpr int kThreads = 256;
constexpr int kGroup = 8;  // consecutive elements per thread trip: one validity byte pair, one 8-byte filter word

struct Partial {
    u64 sum;        // bit pattern (integers wrap, double)
    u64 selected;   // valid & passed the filter
    u64 passed;     // passed the filter
    u64 valid;      // valid (filter ignored): len - GetNullCount()
    u64 min_key;    // order-preserving keys of the selected values
    u64 max_key;
    u64 min_pos;    // element index of the min / max candidate: of equal keys the larger index stays, as the
    u64 max_pos;    // reference's sequential loop keeps the last AggLess-equal value in row order
};

// The result of one batch: the combined partial and the bits of the elements at min_pos / max_pos.
struct BatchResult {
    Partial p;
    u64 min_bits;
    u64 max_bits;
};

template <int TYPE>
__device__ __forceinline__ u64 order_key(u64 bits) {
    if (TYPE == YTGPU_TYPE_UINT64) return bits;
    if (TYPE == YTGPU_TYPE_INT64) return bits ^ (1ull << 63);
    // double: the classes of AggLess (mkql_block_agg_minmax.cpp:22-31): every NaN is the biggest value, and negating
    // the bits of a negative value maps -0.0 onto the key of +0.0
    if ((bits & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) return ~0ull;
    return (bits >> 63) ? 0 - bits : bits ^ (1ull << 63);
}

template <int TYPE>
__device__ __forceinline__ u64 add_bits(u64 a, u64 b) {
    if (TYPE == YTGPU_TYPE_DOUBLE) return (u64)__double_as_longlong(__longlong_as_double((long long)a) + __longlong_as_double((long long)b));
    return a + b;
}

template <int TYPE>
__device__ __forceinline__ void combine(Partial& a, const Partial& b) {
    a.sum = add_bits<TYPE>(a.sum, b.sum);
    a.selected += b.selected;
    a.passed += b.passed;
    a.valid += b.valid;
    // (key, position) is a total order, so the result does not depend on the operand order
    if (b.min_key < a.min_key || (b.min_key == a.min_key && b.min_pos > a.min_pos)) {
        a.min_key = b.min_key;
        a.min_pos = b.min_pos;
    }
    if (b.max_key > a.max_key || (b.max_key == a.max_key && b.max_pos > a.max_pos)) {
        a.max_key = b.max_key;
        a.max_pos = b.max_pos;
    }
}

template <int TYPE>
__device__ __forceinline__ Partial shuffle_xor(const Partial& p, int o) {
    Partial r;
    r.sum = __shfl_xor_sync(0xffffffffu, p.sum, o);
    r.selected = __shfl_xor_sync(0xffffffffu, p.selected, o);
    r.passed = __shfl_xor_sync(0xffffffffu, p.passed, o);
    r.valid = __shfl_xor_sync(0xffffffffu, p.valid, o);
    r.min_key = __shfl_xor_sync(0xffffffffu, p.min_key, o);
    r.max_key = __shfl_xor_sync(0xffffffffu, p.max_key, o);
    r.min_pos = __shfl_xor_sync(0xffffffffu, p.min_pos, o);
    r.max_pos = __shfl_xor_sync(0xffffffffu, p.max_pos, o);
    return r;
}

// The block's combined partial, in thread 0.
template <int TYPE>
__device__ __forceinline__ Partial block_reduce(Partial p) {
    __shared__ Partial s_part[kThreads / 32];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {  // fixed butterfly order
        Partial q = shuffle_xor<TYPE>(p, o);
        // keep the operand order independent of the lane so every lane holds the same bits
        if ((threadIdx.x & o) == 0) combine<TYPE>(p, q);
        else {
            combine<TYPE>(q, p);
            p = q;
        }
    }
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = p;
    __syncthreads();
    if (threadIdx.x == 0)
        for (int w = 1; w < kThreads / 32; ++w) combine<TYPE>(p, s_part[w]);
    return p;
}

__device__ __forceinline__ Partial empty_partial() { return Partial{0, 0, 0, 0, ~0ull, 0ull, 0ull, 0ull}; }

// values = buffers[1] + offset (element pointer); validity bit of element i is bit (i + offset) of `validity`.
template <int TYPE, bool VEC>
__global__ void __launch_bounds__(kThreads) combine_all_kernel(const u64* __restrict__ values, const u8* __restrict__ validity,
                                                               u64 offset, u64 length, const u8* __restrict__ filter,
                                                               Partial* __restrict__ partials) {
    Partial p = empty_partial();
    const u64 groups = (length + kGroup - 1) / kGroup;
    const u64 bitmap_bytes = (offset + length + 7) / 8;
    const u64 first = (u64)blockIdx.x * kThreads + threadIdx.x, stride = (u64)gridDim.x * kThreads;
    // the candidates' positions among this thread's elements (trip * kGroup + k), made global after the loop
    u32 at = 0, min_at = 0, max_at = 0;
    for (u64 g = first; g < groups; g += stride, at += kGroup) {
        const u64 i0 = g * kGroup;
        const u32 cnt = (u32)min((u64)kGroup, length - i0);
        u32 vbits = 0xff;
        if (validity) {
            const u64 bit = i0 + offset, byte = bit >> 3;
            u32 two = validity[byte];
            if (byte + 1 < bitmap_bytes) two |= (u32)validity[byte + 1] << 8;
            vbits = (two >> (bit & 7)) & 0xff;
        }
        u32 fbits = 0xff;
        if (filter) {
            fbits = 0;
            if (cnt == kGroup && ((reinterpret_cast<uintptr_t>(filter) + i0) & 7) == 0) {
                const u64 f = *reinterpret_cast<const u64*>(filter + i0);
#pragma unroll
                for (int k = 0; k < kGroup; ++k) fbits |= ((f >> (8 * k)) & 0xff) ? (1u << k) : 0u;
            } else {
                for (u32 k = 0; k < cnt; ++k) fbits |= filter[i0 + k] ? (1u << k) : 0u;
            }
        }
        const u32 live = cnt == kGroup ? 0xffu : ((1u << cnt) - 1u);
        vbits &= live;
        fbits &= live;
        const u32 sel = vbits & fbits;
        p.valid += __popc(vbits);
        p.passed += __popc(fbits);
        p.selected += __popc(sel);
        u64 v[kGroup];
        if (VEC && cnt == kGroup) {
#pragma unroll
            for (int k = 0; k < kGroup; k += 2) {
                const ulonglong2 t = *reinterpret_cast<const ulonglong2*>(values + i0 + k);
                v[k] = t.x;
                v[k + 1] = t.y;
            }
        } else {
#pragma unroll
            for (int k = 0; k < kGroup; ++k) v[k] = (u32)k < cnt ? values[i0 + k] : 0;
        }
#pragma unroll
        for (int k = 0; k < kGroup; ++k) {
            if (sel & (1u << k)) {
                p.sum = add_bits<TYPE>(p.sum, v[k]);
                // a thread visits its elements in row order: the later of equal keys replaces the candidate
                const u64 key = order_key<TYPE>(v[k]);
                if (key <= p.min_key) {
                    p.min_key = key;
                    min_at = at + k;
                }
                if (key >= p.max_key) {
                    p.max_key = key;
                    max_at = at + k;
                }
            }
        }
    }
    if (p.selected) {  // an empty partial keeps position 0, so it never wins a tie against a real candidate
        p.min_pos = (first + (u64)(min_at / kGroup) * stride) * kGroup + min_at % kGroup;
        p.max_pos = (first + (u64)(max_at / kGroup) * stride) * kGroup + max_at % kGroup;
    }
    p = block_reduce<TYPE>(p);
    if (threadIdx.x == 0) partials[blockIdx.x] = p;
}

template <int TYPE>
__global__ void __launch_bounds__(kThreads) combine_partials_kernel(const Partial* __restrict__ partials, u32 count,
                                                                    const u64* __restrict__ values, BatchResult* __restrict__ out) {
    Partial p = empty_partial();
    // contiguous chunk per thread, in index order
    const u32 per = (count + kThreads - 1) / kThreads;
    const u32 lo = threadIdx.x * per, hi = min(count, lo + per);
    for (u32 i = lo; i < hi; ++i) combine<TYPE>(p, partials[i]);
    p = block_reduce<TYPE>(p);
    if (threadIdx.x == 0) {
        out->p = p;
        out->min_bits = p.selected ? values[p.min_pos] : 0;
        out->max_bits = p.selected ? values[p.max_pos] : 0;
    }
}

// AggLess, mkql_block_agg_minmax.cpp:22-31
bool agg_less(u8 type, u64 a, u64 b) {
    if (type == YTGPU_TYPE_UINT64) return a < b;
    if (type == YTGPU_TYPE_INT64) return (i64)a < (i64)b;
    double x, y;
    std::memcpy(&x, &a, 8);
    std::memcpy(&y, &b, 8);
    if (std::isunordered(x, y)) return std::isnan(x) < std::isnan(y);
    return x < y;
}

template <int TYPE>
Status launch(Context* ctx, const u64* vals, const u8* validity, u64 offset, u64 length, const u8* filter, Partial* partials, u32 grid,
              BatchResult* result) {
    const bool vec = (reinterpret_cast<uintptr_t>(vals) & 15) == 0;
    if (vec) combine_all_kernel<TYPE, true><<<grid, kThreads, 0, ctx->stream>>>(vals, validity, offset, length, filter, partials);
    else combine_all_kernel<TYPE, false><<<grid, kThreads, 0, ctx->stream>>>(vals, validity, offset, length, filter, partials);
    combine_partials_kernel<TYPE><<<1, kThreads, 0, ctx->stream>>>(partials, grid, vals, result);
    YTGPU_CUDA_TRY(cudaGetLastError());
    return Status{};
}

Status combine_all_impl(Context* ctx, const ytgpu_arrow_array* col, const u8* filter, ytgpu_block_agg_state* state) {
    if (!col || !state) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    const u8 type = col->value_type;
    if (type != YTGPU_TYPE_INT64 && type != YTGPU_TYPE_UINT64 && type != YTGPU_TYPE_DOUBLE)
        return make_status(YTGPU_ERR_UNSUPPORTED, "block aggregators take Int64, Uint64 or Double columns");
    if (state->value_type != type) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "state was initialised for another value type");
    if (col->offset < 0 || col->length < 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "negative offset or length");
    const u64 length = (u64)col->length, offset = (u64)col->offset;
    if (length == 0) return Status{};
    if (!col->values) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null values buffer");
    if (col->mem != YTGPU_MEM_HOST && reinterpret_cast<uintptr_t>(col->values) % 8)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "device values buffer must be 8-byte aligned");
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));

    InBuf<u64> vals;
    InBuf<u8> nulls, flt;
    const u8* validity = col->nullable ? col->validity : nullptr;  // IsNullable ? GetNullCount() : 0
    u64 bit_offset = offset, validity_bytes = 0;
    if (validity && col->mem == YTGPU_MEM_HOST) {  // upload only the bytes that cover the rows
        const u64 first = offset / 8;
        validity += first;
        validity_bytes = (offset + length + 7) / 8 - first;
        bit_offset = offset % 8;
    }
    YTGPU_TRY(vals.stage(ctx, static_cast<const u64*>(col->values) + offset, length, col->mem));
    YTGPU_TRY(nulls.stage(ctx, validity, validity_bytes, col->mem));
    YTGPU_TRY(flt.stage(ctx, filter, length, col->mem));
    const u64 groups = (length + kGroup - 1) / kGroup;
    const u32 grid = (u32)std::max<u64>(1, std::min<u64>((groups + kThreads - 1) / kThreads, (u64)kNumSms * 8));
    DevBuf<Partial> partials;
    DevBuf<BatchResult> result;
    YTGPU_TRY(partials.allocate(ctx, grid));
    YTGPU_TRY(result.allocate(ctx, 1));
    {
        KernelTimer t(ctx, KC_GROUPBY, 2);
        if (type == YTGPU_TYPE_INT64) YTGPU_TRY((launch<YTGPU_TYPE_INT64>(ctx, vals.p, nulls.p, bit_offset, length, flt.p, partials.p, grid, result.p)));
        else if (type == YTGPU_TYPE_UINT64) YTGPU_TRY((launch<YTGPU_TYPE_UINT64>(ctx, vals.p, nulls.p, bit_offset, length, flt.p, partials.p, grid, result.p)));
        else YTGPU_TRY((launch<YTGPU_TYPE_DOUBLE>(ctx, vals.p, nulls.p, bit_offset, length, flt.p, partials.p, grid, result.p)));
    }
    BatchResult br{};
    YTGPU_CUDA_TRY(cudaMemcpyAsync(&br, result.p, sizeof(BatchResult), cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    const Partial& r = br.p;

    // ---- fold the batch into the state exactly as AddMany does ----
    state->count_all += filter ? r.passed : length;  // CountAll: += filtered ? *filtered : batchLength
    const u64 null_count = (col->nullable && col->validity) ? length - r.valid : 0;
    if (length - null_count == 0) return Status{};  // `if (!count) return;`
    state->count += r.selected;
    // sum (mkql_block_agg_sum.cpp:183-231): IsValid is raised even when the filter let nothing through, unless the batch has nulls
    if (type == YTGPU_TYPE_DOUBLE) {
        double a, b;
        std::memcpy(&a, &state->sum, 8);
        std::memcpy(&b, &r.sum, 8);
        a += b;
        std::memcpy(&state->sum, &a, 8);
    } else {
        state->sum += r.sum;
    }
    const u8 raised = (!filter || null_count == 0) ? 1 : (r.selected ? 1 : 0);
    if (col->nullable) state->sum_valid |= raised;
    // min / max (mkql_block_agg_minmax.cpp:721-768): without a filter IsValid = 1, with one IsValid |= validCount != 0
    // the batch comes after the state in row order, so it wins ties, as in the reference's loop
    if (r.selected) {
        state->min_value = agg_less(type, state->min_value, br.min_bits) ? state->min_value : br.min_bits;   // UpdateMinMax<true>(x, y)
        state->max_value = agg_less(type, br.max_bits, state->max_value) ? state->max_value : br.max_bits;   // UpdateMinMax<false>(x, y)
    }
    if (col->nullable) {
        const u8 mm = !filter ? 1 : (r.selected ? 1 : 0);
        state->min_valid |= mm;
        state->max_valid |= mm;
    }
    return Status{};
}

}  // namespace

extern "C" {

void ytgpu_block_agg_state_init(ytgpu_block_agg_state* state, uint8_t value_type, uint8_t nullable) {
    if (!state) return;
    std::memset(state, 0, sizeof(*state));
    state->value_type = value_type;
    // InitialStateValue, mkql_block_agg_minmax.cpp:76-101
    if (value_type == YTGPU_TYPE_DOUBLE) {
        state->min_value = 0x7ff8000000000000ull;  // quiet NaN: the biggest value of the aggregate ordering
        state->max_value = 0xfff0000000000000ull;  // -inf
    } else if (value_type == YTGPU_TYPE_INT64) {
        state->min_value = 0x7fffffffffffffffull;
        state->max_value = 0x8000000000000000ull;
    } else {
        state->min_value = ~0ull;
        state->max_value = 0;
    }
    // a non-optional column has no IsValid flag: its aggregates are always defined
    state->sum_valid = state->min_valid = state->max_valid = nullable ? 0 : 1;
}

int ytgpu_block_combine_all(ytgpu_context* h, const ytgpu_arrow_array* column, const uint8_t* filter, ytgpu_block_agg_state* state,
                            ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, combine_all_impl(as_context(h), column, filter, state));
}

}  // extern "C"
