// long_keys.cu — rowset sort by keys of any width: MSD refinement rounds over the width-free key words (keys.cuh).
//
// State: the permutation perm[position] plus groups, maximal runs of positions whose keys are equal so far.  A group is
// named by its first position g; cursor[g] is the key word its rows have not compared yet.  Every round, over the rows
// of the unresolved groups only (act[], positions in increasing order):
//   1. skip:    newcur[g] = min over the group's rows of the first word at or after cursor[g] where the row differs
//               from the group's first row (kKeyEnd: every key of the group is equal, it stays in input order);
//   2. split:   stable radix sort of the rows by (g, word at newcur[g]) — one chunk in the first round (one group) —
//               and scatter back into the group's own positions (a group is a contiguous position range);
//   3. classify: new groups are the runs of equal (g, word).  Runs of one row are done, runs of 2..kSmallGroup rows are
//               finished by one thread's insertion sort, longer runs stay for the next round with cursor newcur[g] + 1.
// Step 1 makes the number of rounds depend on how often groups split, not on the key length: a shared prefix of any
// length costs one pass over its words.  Scratch: O(n) words, independent of the key width.
#include <algorithm>
#include <vector>

#include "long_keys.cuh"
#include "radix_sort.cuh"
#include "scan.cuh"

namespace ytgpu {
namespace {

constexpr u32 kSmallGroup = 32;

inline u32 grid_1d(u64 n) { return (u32)std::max<u64>(1, std::min<u64>((n + 255) / 256, (u64)kNumSms * 8)); }

#define LK_FOR(j, n) for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < (n); j += (u64)gridDim.x * blockDim.x)

__global__ void __launch_bounds__(256) long_key_errors_kernel(const KeyLayout L, const ytgpu_value* __restrict__ vals, u32 vc,
                                                              u64 n, u32* __restrict__ err_word) {
    u32 err = 0;
    LK_FOR(i, n) {
        for (u32 c = 0; c < L.ncols; ++c) err |= key_value_errors(L.col[c], vals[i * vc + L.col[c].index]);
    }
    if (err) atomicOr(err_word, err);
}

__global__ void __launch_bounds__(256) lk_init_kernel(u64 n, u32* perm, u32* act, u32* gstart) {
    LK_FOR(i, n) {
        perm[i] = (u32)i;
        act[i] = (u32)i;
        gstart[i] = 0;
    }
}

__global__ void __launch_bounds__(256) lk_reset_kernel(const u32* __restrict__ act, u64 m, const u32* __restrict__ gstart,
                                                       u64* __restrict__ newcur) {
    LK_FOR(j, m) {
        const u32 p = act[j];
        if (gstart[p] == p) newcur[p] = kKeyEnd;
    }
}

__global__ void __launch_bounds__(256) lk_skip_kernel(const KeyLayout L, const ytgpu_value* __restrict__ vals, u32 vc,
                                                      const u8* __restrict__ heap, const u32* __restrict__ act, u64 m,
                                                      const u32* __restrict__ perm, const u32* __restrict__ gstart,
                                                      const u64* __restrict__ cursor, u64* newcur) {
    LK_FOR(j, m) {
        const u32 p = act[j], g = gstart[p];
        if (p == g) continue;
        const u64 d = key_first_diff(L, vals + (u64)perm[p] * vc, vals + (u64)perm[g] * vc, heap, cursor[g]);
        // most rows of a large group find the minimum already there: skip the same-address atomic
        if (d < *(volatile u64*)&newcur[g]) atomicMin((unsigned long long*)&newcur[g], (unsigned long long)d);
    }
}

__global__ void __launch_bounds__(256) lk_keys_kernel(const KeyLayout L, const ytgpu_value* __restrict__ vals, u32 vc,
                                                      const u8* __restrict__ heap, const u32* __restrict__ act, u64 m,
                                                      const u32* __restrict__ perm, const u32* __restrict__ gstart,
                                                      const u64* __restrict__ newcur, u64* __restrict__ k0, u64* __restrict__ k1) {
    LK_FOR(j, m) {
        const u32 p = act[j], g = gstart[p];
        k0[j] = g;
        k1[j] = key_word_at(L, vals + (u64)perm[p] * vc, heap, newcur[g]);
    }
}

// Sorted order j <- element sidx[j]; the rows go back into the same positions act[0..m) (scatter kernel).
__global__ void __launch_bounds__(256) lk_permute_kernel(const u32* __restrict__ sidx, const u32* __restrict__ act, u64 m,
                                                         const u32* __restrict__ perm, const u64* __restrict__ k0,
                                                         const u64* __restrict__ k1, u32* __restrict__ trow,
                                                         u32* __restrict__ tg, u64* __restrict__ tword) {
    LK_FOR(j, m) {
        const u32 s = sidx[j];
        trow[j] = perm[act[s]];
        tg[j] = (u32)k0[s];
        tword[j] = k1[s];
    }
}

__global__ void __launch_bounds__(256) lk_scatter_kernel(const u32* __restrict__ act, u64 m, const u32* __restrict__ trow,
                                                         const u32* __restrict__ tg, const u64* __restrict__ tword,
                                                         u32* __restrict__ perm, u64* __restrict__ head) {
    LK_FOR(j, m) {
        perm[act[j]] = trow[j];
        head[j] = (j == 0 || tg[j] != tg[j - 1] || tword[j] != tword[j - 1]) ? 1 : 0;
    }
}

// scanned = exclusive scan of the run heads: run of j = incl(j) - 1, and j heads its run iff incl(j) != scanned[j].
__device__ __forceinline__ u64 lk_incl(const u64* scanned, const u64* total, u64 m, u64 j) {
    return j + 1 < m ? scanned[j + 1] : *total;
}

__global__ void __launch_bounds__(256) lk_run_start_kernel(const u64* __restrict__ scanned, const u64* __restrict__ total, u64 m,
                                                           u32* __restrict__ run_start) {
    LK_FOR(j, m) {
        const u64 inc = lk_incl(scanned, total, m, j);
        if (inc != scanned[j]) run_start[inc - 1] = (u32)j;
    }
}

__global__ void __launch_bounds__(256) lk_classify_kernel(const KeyLayout L, const ytgpu_value* __restrict__ vals, u32 vc,
                                                          const u8* __restrict__ heap, const u32* __restrict__ act, u64 m,
                                                          const u64* __restrict__ scanned, const u64* __restrict__ total,
                                                          const u32* __restrict__ run_start, const u32* __restrict__ tg,
                                                          const u64* __restrict__ newcur, u32* __restrict__ perm,
                                                          u32* __restrict__ gstart, u64* __restrict__ cursor, u64* __restrict__ keep) {
    const u64 runs = *total;
    LK_FOR(j, m) {
        const u64 s = lk_incl(scanned, total, m, j) - 1;
        const u32 start = run_start[s];
        const u32 end = s + 1 < runs ? run_start[s + 1] : (u32)m;
        const u32 size = end - start;
        const u64 cur = newcur[tg[j]];
        const u32 p = act[j], pnew = act[start];  // the run covers positions pnew .. pnew + size - 1
        const bool next_round = cur != kKeyEnd && size > kSmallGroup;
        keep[j] = next_round ? 1 : 0;
        if (next_round) {
            gstart[p] = pnew;
            if (j == start) cursor[pnew] = cur + 1;  // its rows agree on the word at cur
        } else if (j == start && cur != kKeyEnd && size > 1) {
            // stable insertion sort of a small run (its rows are in input order)
            u32 r[kSmallGroup];
            for (u32 i = 0; i < size; ++i) r[i] = perm[pnew + i];
            for (u32 i = 1; i < size; ++i) {
                const u32 x = r[i];
                u32 k = i;
                while (k > 0 && key_compare_from(L, vals + (u64)x * vc, vals + (u64)r[k - 1] * vc, heap, cur + 1) < 0) {
                    r[k] = r[k - 1];
                    --k;
                }
                r[k] = x;
            }
            for (u32 i = 0; i < size; ++i) perm[pnew + i] = r[i];
        }
    }
}

__global__ void __launch_bounds__(256) lk_compact_kernel(const u32* __restrict__ act, u64 m, const u64* __restrict__ pos,
                                                         const u64* __restrict__ total, u32* __restrict__ out) {
    LK_FOR(j, m) {
        const u64 next = j + 1 < m ? pos[j + 1] : *total;
        if (next != pos[j]) out[pos[j]] = act[j];
    }
}

}  // namespace

Status check_long_keys(Context* ctx, const KeyLayout& L, const ytgpu_value* values_dev, u32 value_count, u64 n) {
    if (n == 0) return Status{};
    KernelTimer t(ctx, KC_EXTRACT);
    long_key_errors_kernel<<<grid_1d(n), 256, 0, ctx->stream>>>(L, values_dev, value_count, n, ctx->dev_err);
    YTGPU_CUDA_TRY(cudaGetLastError());
    return Status{};
}

Status long_key_sort(Context* ctx, const KeyLayout& L, const ytgpu_value* vals, u32 vc, const u8* heap, u64 n, u32* perm) {
    ctx->last_sort_refine_rounds = 0;
    ctx->last_sort_refine_rows.clear();
    if (n == 0) return Status{};
    if (n >= (1ull << 30))
        return make_status(YTGPU_ERR_UNSUPPORTED, "row count %llu exceeds 2^30-1 rows per sort call", (unsigned long long)n);
    cudaStream_t st = ctx->stream;
    DevBuf<u32> act[2], gstart, sidx, trow, tg, run_start;
    DevBuf<u64> cursor, newcur, k0, k1, tword, head, keep, sums, totals;
    for (auto* b : {&act[0], &act[1], &gstart, &sidx, &trow, &tg, &run_start}) YTGPU_TRY(b->allocate(ctx, n));
    for (auto* b : {&cursor, &newcur, &k0, &k1, &tword, &head, &keep}) YTGPU_TRY(b->allocate(ctx, n));
    YTGPU_TRY(sums.allocate(ctx, scan_block_count(n)));
    YTGPU_TRY(totals.allocate(ctx, 2));
    {
        KernelTimer t(ctx, KC_SCATTER);
        lk_init_kernel<<<grid_1d(n), 256, 0, st>>>(n, perm, act[0].p, gstart.p);
        YTGPU_CUDA_TRY(cudaMemsetAsync(cursor.p, 0, 8, st));  // group 0: cursor (0, 0)
    }
    u64 m = n;
    int cur_act = 0;
    while (m > 0) {
        ctx->last_sort_refine_rows.push_back(m);
        ++ctx->last_sort_refine_rounds;
        const u32* a = act[cur_act].p;
        const u32 blocks = grid_1d(m);
        {
            KernelTimer t(ctx, KC_EXTRACT, 3);
            lk_reset_kernel<<<blocks, 256, 0, st>>>(a, m, gstart.p, newcur.p);
            lk_skip_kernel<<<blocks, 256, 0, st>>>(L, vals, vc, heap, a, m, perm, gstart.p, cursor.p, newcur.p);
            lk_keys_kernel<<<blocks, 256, 0, st>>>(L, vals, vc, heap, a, m, perm, gstart.p, newcur.p, k0.p, k1.p);
            YTGPU_CUDA_TRY(cudaGetLastError());
        }
        {
            // the first round has one group: its rows sort by the word alone
            SortScratch s;
            PermRef sp;
            const u64* chunks[2] = {k0.p, k1.p};
            const bool one_group = ctx->last_sort_refine_rounds == 1;
            YTGPU_TRY(radix_sort_keys(ctx, one_group ? chunks + 1 : chunks, one_group ? 1 : 2, m, &s, &sp));
            YTGPU_TRY(materialize_perm(ctx, sp, m, sidx.p));
        }
        {
            KernelTimer t(ctx, KC_SCATTER, 9);
            lk_permute_kernel<<<blocks, 256, 0, st>>>(sidx.p, a, m, perm, k0.p, k1.p, trow.p, tg.p, tword.p);
            lk_scatter_kernel<<<blocks, 256, 0, st>>>(a, m, trow.p, tg.p, tword.p, perm, head.p);
            exclusive_scan_u64(st, head.p, m, sums.p, totals.p);
            lk_run_start_kernel<<<blocks, 256, 0, st>>>(head.p, totals.p, m, run_start.p);
            lk_classify_kernel<<<blocks, 256, 0, st>>>(L, vals, vc, heap, a, m, head.p, totals.p, run_start.p, tg.p, newcur.p, perm,
                                                       gstart.p, cursor.p, keep.p);
            exclusive_scan_u64(st, keep.p, m, sums.p, totals.p + 1);
            lk_compact_kernel<<<blocks, 256, 0, st>>>(a, m, keep.p, totals.p + 1, act[cur_act ^ 1].p);
            YTGPU_CUDA_TRY(cudaGetLastError());
        }
        YTGPU_CUDA_TRY(cudaMemcpyAsync(&m, totals.p + 1, 8, cudaMemcpyDeviceToHost, st));
        YTGPU_CUDA_TRY(cudaStreamSynchronize(st));
        cur_act ^= 1;
    }
    return Status{};
}

}  // namespace ytgpu

// ---- host-side self check of the key words (CPU tests; not part of ytgpu.h) ----
using namespace ytgpu;

extern "C" {

// Every row's concatenated key words (keys.cuh), computed by the host-compiled code: row i's words are
// out_words[out_offsets[i] .. out_offsets[i + 1]).  String widths of 0 are measured as the sort measures them.
// Returns YTGPU_ERR_INVALID_ARGUMENT when `capacity` words are not enough.
int ytgpu_hostcheck_key_words(const ytgpu_value* values, uint32_t value_count, const uint8_t* heap, uint64_t n,
                              const ytgpu_sort_spec* spec, uint64_t* out_words, uint64_t capacity, uint64_t* out_offsets,
                              uint32_t* out_err) {
    if (!spec || spec->column_count == 0 || spec->column_count > (u32)kMaxKeyColumns) return YTGPU_ERR_INVALID_ARGUMENT;
    std::vector<ytgpu_key_column> cols(spec->columns, spec->columns + spec->column_count);
    for (auto& k : cols) {
        if ((k.type == YTGPU_TYPE_STRING || k.type == 0) && k.width == 0)
            for (u64 i = 0; i < n; ++i) {
                const ytgpu_value& v = values[i * value_count + k.index];
                if (v.type == YTGPU_TYPE_STRING) k.width = std::max(k.width, v.length);
            }
    }
    ytgpu_sort_spec rs{cols.data(), (u32)cols.size()};
    KeyLayout L;
    Status s = build_key_layout(&rs, false, false, &L);
    if (!s.ok() && !(s.code == YTGPU_ERR_UNSUPPORTED && L.nchunks > (u32)kMaxKeyChunks)) return s.code;
    u32 err = 0;
    u64 o = 0;
    for (u64 i = 0; i < n; ++i) {
        out_offsets[i] = o;
        const ytgpu_value* row = values + i * value_count;
        for (u32 c = 0; c < L.ncols; ++c) {
            const KeyColLayout& k = L.col[c];
            err |= key_value_errors(k, row[k.index]);
            const u32 nw = key_col_words(k, row[k.index]);
            if (o + nw > capacity) return YTGPU_ERR_INVALID_ARGUMENT;
            for (u32 w = 0; w < nw; ++w) out_words[o++] = key_col_word(k, row[k.index], heap, w);
        }
    }
    out_offsets[n] = o;
    *out_err = err;
    return YTGPU_OK;
}

}  // extern "C"
