// capi_sort.cu — C ABI: sort / merge entry points (see include/ytgpu.h for the reference interfaces).
#include <vector>

#include "columnar.cuh"
#include "context.cuh"
#include "keys.cuh"
#include "long_keys.cuh"
#include "merge.cuh"
#include "radix_sort.cuh"
#include "rows.cuh"
#include "scan.cuh"

using namespace ytgpu;

namespace {

struct ChunkSet {
    std::vector<DevBuf<u64>> bufs;
    ChunkPtrs ptrs{};
    const u64* cptrs[kMaxKeyChunks] = {nullptr};
    Status allocate(Context* ctx, u32 nchunks, u64 n) {
        bufs = std::vector<DevBuf<u64>>(nchunks);
        for (u32 c = 0; c < nchunks; ++c) {
            YTGPU_TRY(bufs[c].allocate(ctx, n));
            ptrs.p[c] = bufs[c].p;
            cptrs[c] = bufs[c].p;
        }
        return Status{};
    }
};

// Resolves string widths (width == 0 -> measured on the device) into a private copy of the spec.
Status resolve_widths(Context* ctx, const ytgpu_sort_spec* spec, const ytgpu_value* values_dev, u32 value_count,
                      u64 n, std::vector<ytgpu_key_column>* cols) {
    cols->assign(spec->columns, spec->columns + spec->column_count);
    bool need = false;
    for (auto& k : *cols) {
        if (k.index >= value_count)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key column index %u >= value count %u", k.index, value_count);
        if ((k.type == YTGPU_TYPE_STRING || k.type == 0) && k.width == 0) need = true;
    }
    if (need) {
        u32 mx[kMaxKeyColumns];
        ytgpu_sort_spec tmp{cols->data(), (u32)cols->size()};
        YTGPU_TRY(measure_string_widths(ctx, &tmp, values_dev, value_count, n, mx));
        for (size_t c = 0; c < cols->size(); ++c) {
            auto& k = (*cols)[c];
            if ((k.type == YTGPU_TYPE_STRING || k.type == 0) && k.width == 0) k.width = mx[c];
        }
    }
    return Status{};
}

// Stages a rowset on the device (HOST flavour), normalises its keys and sorts them: the pieces every rowset entry
// point shares.  The buffers live as long as the object (the permutation refers to the scratch).  Keys whose
// fixed-width normalised form does not fit in kMaxKeyChunks chunks take the refinement sort of long_keys.cu instead.
struct RowsetSort {
    StagedRowset staged;
    const ytgpu_value* vals = nullptr;
    const u8* heap = nullptr;
    u32 vc = 0;
    KeyLayout L;
    bool long_keys = false;
    ChunkSet chunks;
    SortScratch scratch;
    DevBuf<u32> long_perm;
    DevBuf<SortPlan> long_plan;  // all zero: the permutation is idx[0]
    PermRef perm;

    Status run(Context* ctx, const ytgpu_rowset_view* in, const ytgpu_sort_spec* spec) {
        YTGPU_TRY(prepare(ctx, in, spec));
        return sort(ctx, in->row_count);
    }
    Status sort(Context* ctx, u64 n) {
        if (!long_keys) return radix_sort_keys(ctx, chunks.cptrs, (int)L.nchunks, n, &scratch, &perm);
        YTGPU_TRY(long_perm.allocate(ctx, n));
        YTGPU_TRY(long_plan.allocate(ctx, 1));
        YTGPU_CUDA_TRY(cudaMemsetAsync(long_plan.p, 0, sizeof(SortPlan), ctx->stream));
        YTGPU_TRY(long_key_sort(ctx, L, vals, vc, heap, n, long_perm.p));
        perm.plan = long_plan.p;
        perm.idx[0] = perm.idx[1] = long_perm.p;
        return Status{};
    }
    // Staging + key normalisation only (the merge of sorted runs needs no sort).
    Status prepare(Context* ctx, const ytgpu_rowset_view* in, const ytgpu_sort_spec* spec) {
        const u64 n = in->row_count;
        vc = in->value_count;
        YTGPU_TRY(staged.stage(ctx, in, in->mem));
        vals = staged.values.p;
        heap = staged.heap.p;
        std::vector<ytgpu_key_column> cols;
        YTGPU_TRY(resolve_widths(ctx, spec, vals, vc, n, &cols));
        ytgpu_sort_spec rs{cols.data(), (u32)cols.size()};
        const Status s = build_key_layout(&rs, /*fixed_rows*/ false, /*force_type_byte*/ false, &L);
        long_keys = s.code == YTGPU_ERR_UNSUPPORTED && L.nchunks > (u32)kMaxKeyChunks;
        if (long_keys) {
            YTGPU_TRY(check_long_keys(ctx, L, vals, vc, n));
            return check_device_errors(ctx);
        }
        YTGPU_TRY(s);
        YTGPU_TRY(chunks.allocate(ctx, L.nchunks, n));
        YTGPU_TRY(normalize_rowset(ctx, L, vals, vc, heap, n, chunks.ptrs));
        YTGPU_TRY(check_device_errors(ctx));
        return Status{};
    }
};

Status sort_rowset_impl(Context* ctx, const ytgpu_rowset_view* in, const ytgpu_sort_spec* spec, u32* out_perm,
                        ytgpu_value* out_values, int out_mem) {
    if (!in || !spec || !spec->columns) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    if (spec->column_count == 0 || spec->column_count > (u32)kMaxKeyColumns)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key column count must be in [1, %d]", kMaxKeyColumns);
    ctx->last_sort_refine_rounds = 0;
    const u64 n = in->row_count;
    if (n == 0) return Status{};
    const u32 vc = in->value_count;
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));

    RowsetSort rs;
    YTGPU_TRY(rs.run(ctx, in, spec));
    const ytgpu_value* vals = rs.vals;
    const PermRef& perm = rs.perm;

    if (out_perm) {
        OutBuf<u32> dst;
        YTGPU_TRY(dst.prepare(ctx, out_perm, n, out_mem));
        YTGPU_TRY(materialize_perm(ctx, perm, n, dst.p));
        YTGPU_TRY(dst.download(ctx, n));
    }
    if (out_values) {
        OutBuf<ytgpu_value> dst;
        YTGPU_TRY(dst.prepare(ctx, out_values, n * vc, out_mem));
        YTGPU_TRY(gather_rows(ctx, reinterpret_cast<const u8*>(vals), perm, reinterpret_cast<u8*>(dst.p), n, vc * 16));
        YTGPU_TRY(dst.download(ctx, n * vc));
    }
    if (in->mem == YTGPU_MEM_HOST || out_mem == YTGPU_MEM_HOST) YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return Status{};
}

// ---- sorted join (TSortedJoiningReader) ----
// After the stable sort of the concatenated runs by (join key, tie-break columns): position j holds row perm[j].
// head[j] = 1 when the join key (the first `prefix_bytes` bytes of the normalised key) differs from position j-1's.
struct JoinPrefix {
    const u64* chunk[kMaxKeyChunks];
    u32 full_chunks;   // chunks compared whole
    u64 tail_mask;     // mask of the partial chunk (0 = none)
};

__global__ void join_heads_kernel(JoinPrefix P, const SortPlan* plan, const u32* pa, const u32* pb, u64 n, u64* head) {
    const u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    u64 h = 1;
    if (j > 0) {
        const u32 r = perm_at(plan, pa, pb, j), q = perm_at(plan, pa, pb, j - 1);
        bool same = true;
        for (u32 c = 0; c < P.full_chunks && same; ++c) same = P.chunk[c][r] == P.chunk[c][q];
        if (same && P.tail_mask) same = ((P.chunk[P.full_chunks][r] ^ P.chunk[P.full_chunks][q]) & P.tail_mask) == 0;
        h = same ? 0 : 1;
    }
    head[j] = h;
}

// The same for keys that took the refinement sort: L holds the join key columns only.
__global__ void join_heads_long_kernel(const KeyLayout L, const ytgpu_value* vals, u32 vc, const u8* heap, const SortPlan* plan,
                                       const u32* pa, const u32* pb, u64 n, u64* head) {
    const u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    u64 h = 1;
    if (j > 0) {
        const u32 r = perm_at(plan, pa, pb, j), q = perm_at(plan, pa, pb, j - 1);
        h = key_first_diff(L, vals + (u64)r * vc, vals + (u64)q * vc, heap, 0) == kKeyEnd ? 0 : 1;
    }
    head[j] = h;
}

// gid (exclusive scan of head, so group of j = gid[j+1]-1 == gid[j] + head - 1): a primary row marks its group.
__global__ void join_mark_kernel(const SortPlan* plan, const u32* pa, const u32* pb, u64 n, u64 primary_rows,
                                 const u64* scanned, const u64* total, u8* has_primary) {
    const u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    if (perm_at(plan, pa, pb, j) < primary_rows) {
        const u64 g = (j + 1 < n ? scanned[j + 1] : *total) - 1;
        has_primary[g] = 1;
    }
}

__global__ void join_keep_kernel(const SortPlan* plan, const u32* pa, const u32* pb, u64 n, u64 primary_rows,
                                 const u64* scanned, const u64* total, const u8* has_primary, u64* keep) {
    const u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const u64 g = (j + 1 < n ? scanned[j + 1] : *total) - 1;
    keep[j] = (perm_at(plan, pa, pb, j) < primary_rows || has_primary[g]) ? 1 : 0;
}

__global__ void join_compact_kernel(const SortPlan* plan, const u32* pa, const u32* pb, u64 n, const u64* pos,
                                    const u64* total, u32* out) {
    const u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const u64 next = j + 1 < n ? pos[j + 1] : *total;
    if (next != pos[j]) out[pos[j]] = perm_at(plan, pa, pb, j);
}

Status join_sorted_impl(Context* ctx, const ytgpu_rowset_view* in, const ytgpu_sort_spec* spec, u32 join_cols,
                        u64 primary_rows, u32* out_perm, u64* out_count, int out_mem) {
    const u64 n = in->row_count;
    *out_count = 0;
    ctx->last_sort_refine_rounds = 0;
    if (n == 0) return Status{};
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    RowsetSort rs;
    YTGPU_TRY(rs.run(ctx, in, spec));

    JoinPrefix P{};
    const u32 prefix_bytes = rs.long_keys ? 0 : (join_cols >= rs.L.ncols ? rs.L.total_bytes : rs.L.col[join_cols].byte_offset);
    for (u32 c = 0; !rs.long_keys && c < rs.L.nchunks; ++c) P.chunk[c] = rs.chunks.cptrs[c];
    P.full_chunks = prefix_bytes / 8;
    const u32 rem = prefix_bytes % 8;
    P.tail_mask = rem ? ~0ull << (8 * (8 - rem)) : 0;

    DevBuf<u64> head, keep, sums, totals;
    DevBuf<u8> has_primary;
    OutBuf<u32> dst;
    YTGPU_TRY(head.allocate(ctx, n));
    YTGPU_TRY(keep.allocate(ctx, n));
    YTGPU_TRY(sums.allocate(ctx, scan_block_count(n)));
    YTGPU_TRY(totals.allocate(ctx, 2));
    YTGPU_TRY(has_primary.allocate(ctx, n));
    YTGPU_CUDA_TRY(cudaMemsetAsync(has_primary.p, 0, n, ctx->stream));
    const u32 threads = 256, blocks = (u32)((n + threads - 1) / threads);
    const SortPlan* plan = rs.perm.plan;
    const u32 *pa = rs.perm.idx[0], *pb = rs.perm.idx[1];
    YTGPU_TRY(dst.prepare(ctx, out_perm, n, out_mem));
    {
        KernelTimer t(ctx, KC_HISTOGRAM, 10);
        if (rs.long_keys) {
            KeyLayout JL = rs.L;
            JL.ncols = join_cols;
            join_heads_long_kernel<<<blocks, threads, 0, ctx->stream>>>(JL, rs.vals, rs.vc, rs.heap, plan, pa, pb, n, head.p);
        } else {
            join_heads_kernel<<<blocks, threads, 0, ctx->stream>>>(P, plan, pa, pb, n, head.p);
        }
        exclusive_scan_u64(ctx->stream, head.p, n, sums.p, totals.p);
        join_mark_kernel<<<blocks, threads, 0, ctx->stream>>>(plan, pa, pb, n, primary_rows, head.p, totals.p, has_primary.p);
        join_keep_kernel<<<blocks, threads, 0, ctx->stream>>>(plan, pa, pb, n, primary_rows, head.p, totals.p, has_primary.p, keep.p);
        exclusive_scan_u64(ctx->stream, keep.p, n, sums.p, totals.p + 1);
        join_compact_kernel<<<blocks, threads, 0, ctx->stream>>>(plan, pa, pb, n, keep.p, totals.p + 1, dst.p);
    }
    YTGPU_CUDA_TRY(cudaGetLastError());
    u64 count = 0;
    YTGPU_CUDA_TRY(cudaMemcpyAsync(&count, totals.p + 1, 8, cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    YTGPU_TRY(dst.download(ctx, count));
    if (out_mem == YTGPU_MEM_HOST && count) YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    *out_count = count;
    return Status{};
}

}  // namespace

namespace ytgpu {
Status sort_fixed_rows_impl(Context* ctx, const ytgpu_fixed_rows_view* in, const ytgpu_sort_spec* spec, u8* out_rows,
                            u32* out_perm, int out_mem) {
    if (!in || !spec || !spec->columns) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    const u64 n = in->row_count;
    const u32 rb = in->row_bytes;
    if (rb == 0 || rb % 16 != 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "row_bytes (%u) must be a positive multiple of 16", rb);
    KeyLayout L;
    YTGPU_TRY(build_key_layout(spec, /*fixed_rows*/ true, false, &L));
    for (u32 c = 0; c < L.ncols; ++c)
        if ((u64)L.col[c].index + L.col[c].payload_bytes > rb)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key column %u exceeds the row", c);
    if (n == 0) return Status{};
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));

    InBuf<u8> staged;
    OutBuf<u8> dst;
    YTGPU_TRY(staged.stage(ctx, in->rows, n * rb, in->mem));
    const u8* rows = staged.p;
    ChunkSet chunks;
    YTGPU_TRY(chunks.allocate(ctx, L.nchunks, n));
    SortScratch scratch;
    PermRef perm;
    if (out_rows) {
        YTGPU_TRY(dst.prepare(ctx, out_rows, n * rb, out_mem));
        // the sort may move the rows itself (three-pass schedule); then the permutation is written only if wanted
        scratch.gather.rows = rows;
        scratch.gather.out = dst.p;
        scratch.gather.row_bytes = rb;
        scratch.gather.want_perm = out_perm != nullptr;
    }
    YTGPU_TRY(prepare_histogram(ctx, (int)L.nchunks, &scratch));
    YTGPU_TRY(normalize_fixed_rows(ctx, L, rows, n, rb, chunks.ptrs, scratch.hist.p, &scratch.hist_precomputed));
    YTGPU_TRY(radix_sort_keys(ctx, chunks.cptrs, (int)L.nchunks, n, &scratch, &perm));
    if (out_rows) {
        if (!scratch.rows_gathered) YTGPU_TRY(gather_rows(ctx, rows, perm, dst.p, n, rb));
        YTGPU_TRY(dst.download(ctx, n * rb));
    }
    if (out_perm) {
        OutBuf<u32> perm_dst;
        YTGPU_TRY(perm_dst.prepare(ctx, out_perm, n, out_mem));
        YTGPU_TRY(materialize_perm(ctx, perm, n, perm_dst.p));
        YTGPU_TRY(perm_dst.download(ctx, n));
    }
    if (in->mem == YTGPU_MEM_HOST || out_mem == YTGPU_MEM_HOST) YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return Status{};
}
}  // namespace ytgpu

extern "C" {

int ytgpu_sort_rowset(ytgpu_context* h, const ytgpu_rowset_view* in, const ytgpu_sort_spec* spec, uint32_t* out_perm,
                      ytgpu_value* out_values, int out_mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, sort_rowset_impl(as_context(h), in, spec, out_perm, out_values, out_mem));
}

int ytgpu_sort_fixed_rows(ytgpu_context* h, const ytgpu_fixed_rows_view* in, const ytgpu_sort_spec* spec,
                          uint8_t* out_rows, uint32_t* out_perm, int out_mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, sort_fixed_rows_impl(as_context(h), in, spec, out_rows, out_perm, out_mem));
}

// The k-way merge with ties broken by (run index, position).  Few runs: pairwise merge-path rounds over the normalised
// keys (merge.cu).  Many runs, or a run that is not sorted: a stable sort of the concatenated runs, which IS that merge
// when the runs are sorted (rows of run r precede rows of run r+1 in the input, equal keys keep input order).
namespace {
Status merge_sorted_runs_impl(Context* ctx, const ytgpu_rowset_view* in, const ytgpu_sort_spec* spec, const u64* run_offsets,
                              u32 run_count, u32* out_perm, int out_mem) {
    if (!spec || !spec->columns || !out_perm) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    if (spec->column_count == 0 || spec->column_count > (u32)kMaxKeyColumns)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key column count must be in [1, %d]", kMaxKeyColumns);
    ctx->last_sort_refine_rounds = 0;
    const u64 n = in->row_count;
    if (n == 0) return Status{};
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    RowsetSort rs;
    YTGPU_TRY(rs.prepare(ctx, in, spec));
    OutBuf<u32> dst;
    YTGPU_TRY(dst.prepare(ctx, out_perm, n, out_mem));
    bool merged = false;
    if (ctx->opt_merge_path != 0 && !rs.long_keys)  // merge path compares normalised key chunks
        YTGPU_TRY(merge_sorted_key_runs(ctx, rs.chunks.cptrs, (int)rs.L.nchunks, n, run_offsets, run_count, dst.p, &merged));
    ctx->last_merge_used_merge_path = merged;
    if (!merged) {
        YTGPU_TRY(rs.sort(ctx, n));
        YTGPU_TRY(materialize_perm(ctx, rs.perm, n, dst.p));
    }
    if (out_mem == YTGPU_MEM_HOST) {
        YTGPU_TRY(dst.download(ctx, n));
        YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    }
    return Status{};
}
}  // namespace

int ytgpu_merge_sorted_runs(ytgpu_context* h, const ytgpu_rowset_view* in, const ytgpu_sort_spec* spec,
                            const uint64_t* run_offsets, uint32_t run_count, uint32_t* out_perm, int out_mem,
                            ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    if (!in || !run_offsets) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument"));
    if (run_offsets[0] != 0 || run_offsets[run_count] != in->row_count)
        return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "run offsets must cover [0, row_count]"));
    for (uint32_t r = 0; r < run_count; ++r)
        if (run_offsets[r] > run_offsets[r + 1])
            return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "run offsets must be non-decreasing"));
    return fill_error(err, merge_sorted_runs_impl(as_context(h), in, spec, run_offsets, run_count, out_perm, out_mem));
}

// TSortedJoiningReader (sorted_merging_reader.cpp:566-760): merge of the primary stream (run 0) with the foreign
// streams; a foreign row survives iff its join key occurs in the primary stream.
int ytgpu_join_sorted_runs(ytgpu_context* h, const ytgpu_rowset_view* in, const ytgpu_sort_spec* spec,
                           uint32_t join_key_column_count, const uint64_t* run_offsets, uint32_t run_count,
                           uint32_t* out_perm, uint64_t* out_row_count, int out_mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    if (!in || !spec || !spec->columns || !run_offsets || !out_perm || !out_row_count || run_count == 0)
        return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument"));
    if (spec->column_count == 0 || spec->column_count > (u32)kMaxKeyColumns || join_key_column_count == 0 ||
        join_key_column_count > spec->column_count)
        return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "join key column count must be in [1, key column count]"));
    if (run_offsets[0] != 0 || run_offsets[run_count] != in->row_count)
        return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "run offsets must cover [0, row_count]"));
    for (uint32_t r = 0; r < run_count; ++r)
        if (run_offsets[r] > run_offsets[r + 1])
            return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "run offsets must be non-decreasing"));
    return fill_error(err, join_sorted_impl(as_context(h), in, spec, join_key_column_count, run_offsets[1], out_perm,
                                            out_row_count, out_mem));
}

}  // extern "C"

// ---- ORDER BY ... OFFSET ... LIMIT over typed columns (ytgpu_order_rows) ----
// The rows to order are written as a device rowset, one 16-byte value per item, and sorted by RowsetSort: the order, the
// string widths, the packed / hybrid schedules and the long-key refinement are those of ytgpu_sort_rowset.
namespace {

constexpr u64 kMaxOrderRows = 1ull << 30;  // the radix sort's bound

struct OrderItemDev {
    ColumnDev col;          // numeric item
    const u64* starts;      // string item
    const u32* lengths;
    const u8* nulls;        // nullable
    u64 heap_base;          // offset of the column's heap in the concatenated heap
    u64 heap_bytes;
    u8 is_string;
    u8 type;                // the declared type of the sort key
};

// Position i of the rowset holds row rows[i] (or i): value k is item k of that row, NULL when the row's value is NULL.
// A row index past the columns writes NULLs and flags DE_ROW_OUT_OF_RANGE; a string past its heap, DE_STRING_OUT_OF_HEAP.
__global__ void __launch_bounds__(256) order_materialize_kernel(const OrderItemDev* __restrict__ items, u32 item_count, u64 column_rows,
                                                                const u32* __restrict__ rows, u64 count, ytgpu_value* __restrict__ out,
                                                                u32* err_word) {
    u32 err = 0;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (u64)gridDim.x * blockDim.x) {
        const u64 r = rows ? rows[i] : i;
        const bool bad = r >= column_rows;
        if (bad) err |= DE_ROW_OUT_OF_RANGE;
        for (u32 k = 0; k < item_count; ++k) {
            const OrderItemDev& it = items[k];
            ytgpu_value v{};
            v.id = (u16)k;
            v.type = YTGPU_TYPE_NULL;
            if (!bad) {
                if (it.is_string) {
                    if (!(it.nulls && it.nulls[r])) {
                        const u64 s = it.starts[r];
                        const u32 len = it.lengths[r];
                        if (s > it.heap_bytes || len > it.heap_bytes - s) {
                            err |= DE_STRING_OUT_OF_HEAP;
                        } else {
                            v.type = YTGPU_TYPE_STRING;
                            v.length = len;
                            v.data = it.heap_base + s;
                        }
                    }
                } else {
                    bool nul = false;
                    const u64 x = decode_at(it.col, (i64)r, &nul);
                    if (!nul) {
                        v.type = it.type;
                        v.data = it.type == YTGPU_TYPE_BOOLEAN ? (x != 0) : x;
                    }
                }
            }
            out[i * item_count + k] = v;
        }
    }
    if (err) atomicOr(err_word, err);
}

// out[i] = the row at sorted position offset + i.
__global__ void __launch_bounds__(256) order_window_kernel(const SortPlan* plan, const u32* pa, const u32* pb, const u32* __restrict__ rows,
                                                           u64 offset, u64 count, u32* __restrict__ out) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (u64)gridDim.x * blockDim.x) {
        const u32 p = perm_at(plan, pa, pb, offset + i);
        out[i] = rows ? rows[p] : p;
    }
}

bool order_numeric_type(u8 t) { return t == YTGPU_TYPE_INT64 || t == YTGPU_TYPE_UINT64 || t == YTGPU_TYPE_DOUBLE || t == YTGPU_TYPE_BOOLEAN; }

Status order_rows_impl(Context* ctx, const ytgpu_column_view* columns, u32 column_count, const ytgpu_string_column* string_columns,
                       u32 string_column_count, const ytgpu_order_item* items, u32 item_count, const u32* rows, u64 row_count, u64 offset,
                       u64 limit, u32* out_rows, u64* out_count, int out_mem) {
    if (row_count >= kMaxOrderRows)
        return make_status(YTGPU_ERR_UNSUPPORTED, "at most 2^30 - 1 rows are ordered (the radix sort's bound), got %llu",
                           (unsigned long long)row_count);
    if (!out_count) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null out_count");
    if (!items || item_count == 0 || item_count > (u32)kMaxKeyColumns)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "item count must be in [1, %d]", kMaxKeyColumns);
    if (out_mem != YTGPU_MEM_DEVICE && out_mem != YTGPU_MEM_HOST)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "out_mem must be YTGPU_MEM_DEVICE or YTGPU_MEM_HOST");
    i64 column_rows = -1;
    for (u32 k = 0; k < item_count; ++k) {
        const ytgpu_order_item& it = items[k];
        if (it.reserved != 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "item %u: reserved must be 0", k);
        i64 len;
        if (it.is_string) {
            if (!string_columns || it.column >= string_column_count)
                return make_status(YTGPU_ERR_INVALID_ARGUMENT, "item %u: no string column %u", k, it.column);
            const ytgpu_string_column& s = string_columns[it.column];
            if (s.mem != YTGPU_MEM_DEVICE && s.mem != YTGPU_MEM_HOST)
                return make_status(YTGPU_ERR_INVALID_ARGUMENT, "item %u: string column mem must be YTGPU_MEM_DEVICE or YTGPU_MEM_HOST", k);
            if (s.row_count && (!s.starts || !s.lengths))
                return make_status(YTGPU_ERR_INVALID_ARGUMENT, "item %u: null starts or lengths", k);
            if (s.heap_bytes && !s.heap) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "item %u: null heap", k);
            len = (i64)s.row_count;
        } else {
            if (!columns || it.column >= column_count) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "item %u: no column %u", k, it.column);
            const ytgpu_column_view& c = columns[it.column];
            if (!order_numeric_type(c.value_type))
                return make_status(YTGPU_ERR_UNSUPPORTED, "item %u: value type 0x%x is not INT64, UINT64, DOUBLE or BOOLEAN", k, c.value_type);
            if (c.value_count < 0 || c.start_index < 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "item %u: negative column range", k);
            len = c.value_count;
        }
        if (column_rows >= 0 && len != column_rows) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "item columns differ in length");
        column_rows = len;
    }
    if (!rows && row_count > (u64)column_rows)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "without rows, row_count (%llu) exceeds the columns' length (%lld)",
                           (unsigned long long)row_count, (long long)column_rows);
    const u64 n = row_count;
    const u64 window = std::min(limit, n - std::min(offset, n));
    *out_count = window;
    if (!out_rows || window == 0) return Status{};
    ctx->last_sort_refine_rounds = 0;
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));

    InBuf<u32> staged_rows;
    YTGPU_TRY(staged_rows.stage(ctx, rows, n, out_mem));
    const u32* drows = staged_rows.p;
    // the item columns on the device; each string heap at its offset in one concatenated heap
    std::vector<StagedColumn> staged(item_count);
    std::vector<InBuf<u64>> sstarts(item_count);
    std::vector<InBuf<u32>> slengths(item_count);
    std::vector<InBuf<u8>> snulls(item_count);
    std::vector<OrderItemDev> host_items(item_count);
    std::vector<ytgpu_key_column> keys(item_count);
    u64 heap_total = 0;
    for (u32 k = 0; k < item_count; ++k) {
        OrderItemDev& d = host_items[k];
        d = OrderItemDev{};
        keys[k] = ytgpu_key_column{k, 0, 0, items[k].descending ? (u8)1 : (u8)0, 0, 0};
        if (!items[k].is_string) {
            YTGPU_TRY(stage_column(ctx, &columns[items[k].column], &staged[k]));
            d.col = staged[k].dev;
            d.type = columns[items[k].column].value_type;
            keys[k].type = d.type;
            continue;
        }
        const ytgpu_string_column& s = string_columns[items[k].column];
        d.is_string = 1;
        d.type = YTGPU_TYPE_STRING;
        keys[k].type = YTGPU_TYPE_STRING;
        d.heap_base = heap_total;
        d.heap_bytes = s.heap_bytes;
        heap_total += s.heap_bytes;
        const int mem = s.row_count ? s.mem : YTGPU_MEM_DEVICE;  // no rows: the caller's pointers stay
        YTGPU_TRY(sstarts[k].stage(ctx, s.starts, s.row_count, mem));
        YTGPU_TRY(slengths[k].stage(ctx, s.lengths, s.row_count, mem));
        YTGPU_TRY(snulls[k].stage(ctx, s.null_bytemap, s.row_count, mem));
        d.starts = sstarts[k].p;
        d.lengths = slengths[k].p;
        d.nulls = snulls[k].p;
    }
    DevBuf<u8> heap;
    YTGPU_TRY(heap.allocate(ctx, heap_total));
    for (u32 k = 0; k < item_count; ++k)  // each heap lands at its offset in the one sort heap, from either memory space
        if (host_items[k].is_string)
            YTGPU_TRY(copy_in(ctx, heap.p + host_items[k].heap_base, string_columns[items[k].column].heap, host_items[k].heap_bytes,
                              string_columns[items[k].column].mem));
    InBuf<OrderItemDev> dev_items;
    YTGPU_TRY(dev_items.stage(ctx, host_items.data(), item_count, YTGPU_MEM_HOST));
    DevBuf<ytgpu_value> values;
    YTGPU_TRY(values.allocate(ctx, n * item_count));
    {
        KernelTimer t(ctx, KC_EXTRACT);
        order_materialize_kernel<<<blocks_for(n, 256, 16), 256, 0, ctx->stream>>>(dev_items.p, item_count, (u64)column_rows, drows, n,
                                                                                   values.p, ctx->dev_err);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_TRY(check_device_errors(ctx));  // synchronises

    const ytgpu_rowset_view view{values.p, n, item_count, 0, heap.p, heap_total, YTGPU_MEM_DEVICE};
    const ytgpu_sort_spec spec{keys.data(), item_count};
    RowsetSort rs;
    YTGPU_TRY(rs.run(ctx, &view, &spec));

    OutBuf<u32> dst;
    YTGPU_TRY(dst.prepare(ctx, out_rows, window, out_mem));
    {
        KernelTimer t(ctx, KC_GATHER);
        order_window_kernel<<<blocks_for(window, 256, 16), 256, 0, ctx->stream>>>(rs.perm.plan, rs.perm.idx[0], rs.perm.idx[1], drows,
                                                                                  std::min(offset, n), window, dst.p);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_TRY(dst.download(ctx, window));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return Status{};
}

}  // namespace

extern "C" int ytgpu_order_rows(ytgpu_context* h, const ytgpu_column_view* columns, uint32_t column_count,
                                const ytgpu_string_column* string_columns, uint32_t string_column_count, const ytgpu_order_item* items,
                                uint32_t item_count, const uint32_t* rows, uint64_t row_count, uint64_t offset, uint64_t limit,
                                uint32_t* out_rows, uint64_t* out_count, int out_mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, order_rows_impl(as_context(h), columns, column_count, string_columns, string_column_count, items, item_count,
                                           rows, row_count, offset, limit, out_rows, out_count, out_mem));
}
