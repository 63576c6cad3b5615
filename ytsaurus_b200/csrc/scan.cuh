// scan.cuh — exclusive scan of u64 in place (three phases over 4096-element blocks), shared by the block codec, the
// column writers, the evaluators, the sorts and the count matrix of the row exchange (peer_kernels.cuh).  Everything is
// TU-local (static) so several .cu files may include it.
#pragma once

#include "common.cuh"
#include "context.cuh"

namespace ytgpu {

constexpr int kScanThreads = 256;
constexpr int kScanItems = 16;  // 4096 elements per block: the serial phase 2 stays short (24 K sums at 10^8 elements)
constexpr int kScanBlock = kScanThreads * kScanItems;

static __device__ __forceinline__ u64 block_scan_exclusive(u64 v, u64* s_warp, u64* total) {
    const u32 lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u64 inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        u64 t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= (u32)o) inc += t;
    }
    if (lane == 31) s_warp[warp] = inc;
    __syncthreads();
    u64 wp = 0, tot = 0;
#pragma unroll
    for (int w = 0; w < kScanThreads / 32; ++w) {
        u64 x = s_warp[w];
        if (w < (int)warp) wp += x;
        tot += x;
    }
    __syncthreads();
    *total = tot;
    return inc - v + wp;
}

// phase 1/3: per-block sums; phase 3 writes exclusive prefixes (in place) given scanned block offsets.
template <bool WRITE>
static __global__ void __launch_bounds__(kScanThreads) scan_blocks_kernel(u64* data, u64 n, u64* block_sums) {
    __shared__ u64 s_warp[kScanThreads / 32];
    const u64 base = (u64)blockIdx.x * kScanBlock + (u64)threadIdx.x * kScanItems;
    u64 v[kScanItems], sum = 0;
#pragma unroll
    for (int i = 0; i < kScanItems; ++i) {
        v[i] = base + i < n ? data[base + i] : 0;
        sum += v[i];
    }
    u64 total;
    u64 ex = block_scan_exclusive(sum, s_warp, &total);
    if (!WRITE) {
        if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
    } else {
        u64 run = ex + block_sums[blockIdx.x];
#pragma unroll
        for (int i = 0; i < kScanItems; ++i) {
            if (base + i < n) data[base + i] = run;
            run += v[i];
        }
    }
}

// phase 2: one block scans the block sums serially in chunks (nblocks <= a few thousand in practice)
static __global__ void __launch_bounds__(kScanThreads) scan_sums_kernel(u64* sums, u64 nblocks, u64* grand_total) {
    __shared__ u64 s_warp[kScanThreads / 32];
    __shared__ u64 s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (u64 base = 0; base < nblocks; base += kScanThreads) {
        const u64 i = base + threadIdx.x;
        const u64 v = i < nblocks ? sums[i] : 0;
        u64 total;
        const u64 ex = block_scan_exclusive(v, s_warp, &total);
        if (i < nblocks) sums[i] = ex + s_carry;
        __syncthreads();
        if (threadIdx.x == 0) s_carry += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) *grand_total = s_carry;
}

inline u64 scan_block_count(u64 n) { return (n + kScanBlock - 1) / kScanBlock; }

//! data[i] <- sum(data[0..i)) for i < n; *grand_total (device) <- sum of all.  `block_sums` holds scan_block_count(n) words.
static inline void exclusive_scan_u64(cudaStream_t stream, u64* data, u64 n, u64* block_sums, u64* grand_total) {
    const u64 nblocks = scan_block_count(n);
    scan_blocks_kernel<false><<<(u32)nblocks, kScanThreads, 0, stream>>>(data, n, block_sums);
    scan_sums_kernel<<<1, kScanThreads, 0, stream>>>(block_sums, nblocks, grand_total);
    scan_blocks_kernel<true><<<(u32)nblocks, kScanThreads, 0, stream>>>(data, n, block_sums);
}

}  // namespace ytgpu
