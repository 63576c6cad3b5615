// peer_kernels.cuh — the streaming slab scatter (rows read sequentially, written to stable per-destination slots in
// local or peer-mapped memory) shared by peer.cu (ytgpu_scatter_rows_to_peers) and shuffle.cu (ytgpu_shuffle_sort).
// Kernels are `static` (TU-local) so both translation units may include it.
#pragma once

#include <algorithm>

#include "context.cuh"
#include "scan.cuh"

namespace ytgpu {

// ---------------------------------------------------------------------------------------------
// Streaming scatter for few partitions (the in-box shuffle: one partition per GPU).  Rows are read
// SEQUENTIALLY (no 128-byte read amplification of random 64-byte accesses, DESIGN.md §4) and each row is
// written to its stable destination slot:  slot = (rows of its partition in earlier tiles) + (rank inside
// the tile).  Per-tile partition counts come from a counting pass over the 4-byte partition index; one
// exclusive scan over the partition-major count matrix [partition][tile] yields every tile's base slot.
// ---------------------------------------------------------------------------------------------
constexpr int kStreamThreads = 256;
constexpr int kStreamItems = 4;
constexpr int kStreamTile = kStreamThreads * kStreamItems;  // rows per tile
constexpr int kStreamMaxParts = 32;

struct DestTable {
    uint4* base[kStreamMaxParts];  // destination of partition p's slab
    u64 start[kStreamMaxParts];    // global slot of its first row (scan value of tile 0)
};

static __global__ void __launch_bounds__(kStreamThreads) scatter_stream_kernel(const uint4* __restrict__ in, const i32* __restrict__ index,
                                                                        u64 n, u32 gr, u32 parts, u32 part_bits, u64 tiles,
                                                                        const u64* __restrict__ tile_base /*[parts][tiles]*/,
                                                                        const DestTable D) {
    constexpr int WARPS = kStreamThreads / 32;
    __shared__ u32 s_wcnt[WARPS][kStreamMaxParts];  // running per-warp counts -> warp offsets inside the tile
    __shared__ u64 s_slot[kStreamMaxParts];         // first slot of this tile per partition
    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid < WARPS * kStreamMaxParts) (&s_wcnt[0][0])[tid] = 0;
    __syncthreads();
    const u64 tile = blockIdx.x;
    const u64 wbase = tile * kStreamTile + (u64)warp * (32 * kStreamItems) + lane;  // warp-striped: stable (item, lane) order
    u32 part[kStreamItems], rank[kStreamItems], pos[kStreamItems];
    u32 lt;
    asm("mov.u32 %0, %%lanemask_lt;" : "=r"(lt));
#pragma unroll
    for (int i = 0; i < kStreamItems; ++i) {
        const u64 r = wbase + (u64)i * 32;
        const bool valid = r < n;
        part[i] = valid ? min((u32)index[r], parts - 1) : 0u;  // out-of-range values were flagged by the counting pass
        // One sweep of ballots, most significant bit first, yields both the lanes holding the same partition (eq) and
        // the lanes holding a smaller one (less); rows past the end sort after every partition.
        const u32 kk = valid ? part[i] : (1u << part_bits);
        u32 m = 0xffffffffu, less = 0;
        for (int b = (int)part_bits; b >= 0; --b) {
            const bool bit = (kk >> b) & 1;
            const u32 v = __ballot_sync(0xffffffffu, bit);
            if (bit) less |= m & ~v;
            m &= bit ? v : ~v;
        }
        const u32 prev = s_wcnt[warp][part[i]];
        __syncwarp();
        if (valid && (m & lt) == 0) s_wcnt[warp][part[i]] = prev + __popc(m);
        rank[i] = prev + __popc(m & lt);
        pos[i] = __popc(less) + __popc(m & lt);  // position of this row when the round is ordered by destination
        __syncwarp();
    }
    __syncthreads();
    if (tid < parts) {
        u32 run = 0;
#pragma unroll
        for (int w = 0; w < WARPS; ++w) {
            const u32 c = s_wcnt[w][tid];
            s_wcnt[w][tid] = run;
            run += c;
        }
        s_slot[tid] = tile_base[(u64)tid * tiles + tile];
    }
    __syncthreads();
    if (gr == 4) {
        // 64-byte rows: a thread loads its whole row, the warp transposes through shared memory so that four
        // consecutive lanes store the four 16-byte granules of ONE row: every store instruction writes whole
        // 64-byte rows (16-byte stores to scattered rows cost a read-modify-write in L2 and 16-byte NVLink
        // packets — measured 3x slower).  XOR swizzle keeps both the stores and the loads conflict free.
        __shared__ uint4 s_rows[WARPS][32 * 4];
        __shared__ u8 s_order[WARPS][32];  // s_order[q] = lane whose row is the q-th of the round in destination order
        uint4* wr = s_rows[warp];
#pragma unroll
        for (int i = 0; i < kStreamItems; ++i) {
            const u64 r = wbase + (u64)i * 32;
            const bool valid = r < n;
            const u32 p = part[i];
            u64 dst_addr = 0;
            if (valid) {
                const u64 slot = s_slot[p] + s_wcnt[warp][p] + rank[i] - D.start[p];
                dst_addr = reinterpret_cast<u64>(D.base[p] + slot * 4);
            }
            // the 32 rows of this round are contiguous in the input: one coalesced 2 KB copy into shared memory
            const u64 round_row0 = r - lane;
#pragma unroll
            for (u32 s = 0; s < 4; ++s) {
                const u32 q = s * 32 + lane, row = q >> 2, g = q & 3;
                if (round_row0 + row < n) wr[row * 4 + (g ^ ((row >> 1) & 3))] = ld_stream_u128(in + round_row0 * 4 + q);
            }
            // Rows leave in destination order: rows of one partition sit next to each other in its slab, so a store
            // instruction writes runs of whole rows (128 B and more) instead of isolated 64-byte rows — fewer, larger
            // NVLink write packets.  With one partition pos[i] == lane; the select on `parts` only steers ptxas (nvcc 12.9):
            // without it the partition-bit sweep above loses its uniform-register loop counters and the kernel measured
            // about 1 % slower on an H100 80GB HBM3 at 700 W (10^8 rows of 64 B, 2 to 32 partitions).
            s_order[warp][parts > 1 ? pos[i] : lane] = (u8)lane;
            __syncwarp();
#pragma unroll
            for (u32 s = 0; s < 4; ++s) {
                const u32 src_lane = s_order[warp][(lane >> 2) + 8 * s], g = lane & 3;
                const u64 d = __shfl_sync(0xffffffffu, dst_addr, src_lane);
                if (d) reinterpret_cast<uint4*>(d)[g] = wr[src_lane * 4 + (g ^ ((src_lane >> 1) & 3))];
            }
            __syncwarp();
        }
        __threadfence_system();  // peer stores are ordered before whatever signals completion to the other GPU
        return;
    }
#pragma unroll
    for (int i = 0; i < kStreamItems; ++i) {
        const u64 r = wbase + (u64)i * 32;
        if (r >= n) continue;
        const u32 p = part[i];
        const u64 slot = s_slot[p] + s_wcnt[warp][p] + rank[i] - D.start[p];
        const uint4* src = in + r * gr;
        uint4* dst = D.base[p] + slot * gr;
        for (u32 g = 0; g < gr; ++g) dst[g] = ld_stream_u128(src + g);
    }
    __threadfence_system();
}

// The [partition][tile] count matrix.  A counting pass over the partition index (tile_count_kernel in peer.cu,
// partition_count_kernel in shuffle.cu) stores the rows of partition p in tile t at cells[p * tiles + t]; scan() turns
// every cell into the global slot of that tile's first row of partition p, which scatter_stream_kernel reads.
struct TileCounts {
    u64 tiles = 0;
    DevBuf<u64> cells;
    DevBuf<u64> sums;  // the scan's block sums, then its grand total
    Status allocate(Context* ctx, u64 n, u32 parts) {
        tiles = std::max<u64>(1, (n + kStreamTile - 1) / kStreamTile);
        YTGPU_TRY(cells.allocate(ctx, (u64)parts * tiles));
        return sums.allocate(ctx, scan_block_count(cells.n) + 1);
    }
    void scan(cudaStream_t st) { exclusive_scan_u64(st, cells.p, cells.n, sums.p, sums.p + sums.n - 1); }  // three launches
};

// Row r of rows[n][row_bytes] goes to D.base[p] + (slot - D.start[p]) rows, p = index[r], its slot taken from the
// scanned counts plus its rank among the tile's rows of partition p.
static inline void launch_scatter_stream(cudaStream_t st, const void* rows, const i32* index, u64 n, u32 row_bytes, u32 parts,
                                         const TileCounts& counts, const DestTable& D) {
    u32 part_bits = 0;
    while ((1u << part_bits) < parts) ++part_bits;
    scatter_stream_kernel<<<(u32)counts.tiles, kStreamThreads, 0, st>>>(reinterpret_cast<const uint4*>(rows), index, n, row_bytes / 16, parts,
                                                                       part_bits, counts.tiles, counts.cells.p, D);
}

}  // namespace ytgpu
