// groupby_multi.cu — GROUP BY over several key columns with several aggregates (the general form of the hashed path).
//
// Replaces, for tuple keys and aggregate lists, the same reference code as ytgpu_scan_filter_groupby:
//   YT QL   GroupOpHelper / InsertGroupRow (library/query/engine/cg_routines/registry.cpp:1571-1655,1783-1920) with the
//           aggregates of builtin_function_types.cpp:201-254 — sum / min / max (engine/udf/sum.c, min.c, max.c), avg and
//           argmin / argmax (builtin_function_profiler.cpp:1300-1600), first (registry.cpp:3633-3693), count;
//   CHYT    DB::Aggregator with a keys128 / serialized key and a list of aggregate functions;
//   YQL     BlockCombineHashed over tuple keys (mkql_block_agg.cpp:1234-1400).
// Three steps instead of one fused kernel (the single-key SUM/COUNT fast path stays in columnar.cu):
//   1. assign: every row that passes the predicate finds or claims the slot of its key tuple in an open-addressing
//      table.  A slot stores the index of the row that claimed it; tuples are compared by decoding that row's key
//      columns again (the inputs are immutable), so any number of key columns needs no lock and no key storage.
//      COUNT(*) and the group's first row are updated here; the slot of every row is kept (4 bytes per row).
//   2. accumulate: one pass per aggregate over its value column, atomics on per-slot state.  min / max move one way, so a
//      plain read that already bounds the value skips the atomic; argmin / argmax / first select a ROW (atomicMin of the
//      row index among the rows that attain the bound), the value is gathered at the end — exactly the reference's
//      "the first row wins a tie" (strict comparison in UpdateAggregateValue).  An aggregate over a string column (or
//      argmin / argmax by one) takes mg_accumulate_strings_kernel instead: it selects the row lock-free with a CAS on
//      the slot's row, comparing strings by the width-free key words of keys.cuh.
//   3. emit: occupied slots are compacted and ordered by first row == QL's first-seen order (InsertGroupRow appends new
//      groups), keys are decoded from the group's first row, states are finalised (avg = sum / count as double).
#include <vector>

#include "columnar.cuh"
#include "context.cuh"
#include "groupby_agg.cuh"
#include "key_tuple.cuh"
#include "keys.cuh"
#include "radix_sort.cuh"
#include "strings.cuh"

using namespace ytgpu;

namespace {

// Step 3b: keys, COUNT(*) and first rows in output order.
struct KeyOutputs {
    u64* keys[kMaxGroupKeys];
    u8* key_null[kMaxGroupKeys];
};
__global__ void __launch_bounds__(256) mg_emit_keys_kernel(const KeyColumns K, const SortPlan* plan, const u32* pa, const u32* pb, u64 g,
                                                           const u32* slots, const unsigned long long* first,
                                                           const unsigned long long* counts, KeyOutputs O, u64* out_counts,
                                                           u64* out_first, u32* out_slot_sorted) {
    const u64 o = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= g) return;
    const u32 slot = slots[perm_at(plan, pa, pb, o)];
    out_slot_sorted[o] = slot;
    const u64 row = first[slot];
    const KeyTuple t = load_tuple(K, row);
#pragma unroll
    for (u32 k = 0; k < (u32)kMaxGroupKeys; ++k)
        if (k < K.count) {
            O.keys[k][o] = t.w[k];
            O.key_null[k][o] = (t.nulls >> k) & 1;
        }
    if (out_counts) out_counts[o] = counts[slot];
    if (out_first) out_first[o] = row;
}


Status groupby_multi_impl(Context* ctx, const ytgpu_column_view* key_columns, u32 key_count, const ytgpu_column_view* value_columns,
                          u32 value_count, const ytgpu_aggregate* aggregates, u32 aggregate_count, const ytgpu_predicate* pred,
                          int32_t pred_column, u64 hint, ytgpu_groupby_multi_result* out, int out_mem,
                          const ytgpu_string_column* string_columns, u32 string_count) {
    if (!key_columns || !out || (aggregate_count && !aggregates) || (value_count && !value_columns) || (string_count && !string_columns))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    // aggregate arguments index value_columns ++ string_columns
    const u64 columns_total = (u64)value_count + string_count;
    auto is_string = [&](int32_t c) { return (u32)c >= value_count; };
    if (key_count == 0 || key_count > (u32)kMaxGroupKeys)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key column count must be in [1, %d]", kMaxGroupKeys);
    if (aggregate_count > (u32)kMaxAggregates) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "at most %d aggregates", kMaxAggregates);
    if (!out->keys || !out->key_null || (aggregate_count && (!out->values || !out->value_null)))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null output array");
    const u64 n = (u64)key_columns[0].value_count;
    for (u32 k = 0; k < key_count; ++k)
        if ((u64)key_columns[k].value_count != n) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key columns differ in length");
    for (u32 v = 0; v < value_count; ++v)
        if ((u64)value_columns[v].value_count != n) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "value column %u differs in length", v);
    for (u32 s = 0; s < string_count; ++s) {
        const ytgpu_string_column& S = string_columns[s];
        if (S.row_count != n) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string column %u differs in length", s);
        if ((S.heap_bytes && !S.heap) || !S.starts || !S.lengths)  // an empty heap (all "" / NULL) is never read
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string column %u: null heap, starts or lengths", s);
        if (S.mem != YTGPU_MEM_DEVICE && S.mem != YTGPU_MEM_HOST)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string column %u: mem must be YTGPU_MEM_DEVICE or YTGPU_MEM_HOST", s);
    }
    if (n > (1ull << 30)) return make_status(YTGPU_ERR_UNSUPPORTED, "at most 2^30 rows per call (slots and rows are 32-bit)");
    const int op = pred ? pred->op : YTGPU_CMP_NONE;
    if (op != YTGPU_CMP_NONE && (pred_column < 0 || (u32)pred_column >= value_count))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "predicate column %d out of range", (int)pred_column);
    for (u32 a = 0; a < aggregate_count; ++a) {
        const ytgpu_aggregate& A = aggregates[a];
        if (A.op < YTGPU_AGG_SUM || A.op > YTGPU_AGG_FIRST) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "aggregate %u: unknown op %d", a, A.op);
        if (A.column < 0 || (u64)A.column >= columns_total) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "aggregate %u: column out of range", a);
        if (is_string(A.column)) {
            if (A.op == YTGPU_AGG_SUM || A.op == YTGPU_AGG_AVG)
                return make_status(YTGPU_ERR_UNSUPPORTED, "aggregate %u: sum / avg over a string column", a);
        } else {
            const u8 t = value_columns[A.column].value_type;
            if (!aggregatable_type(t)) return make_status(YTGPU_ERR_UNSUPPORTED, "aggregate %u: value type 0x%x is not a fixed-width scalar", a, t);
            if ((A.op == YTGPU_AGG_SUM || A.op == YTGPU_AGG_AVG) && t == YTGPU_TYPE_BOOLEAN)
                return make_status(YTGPU_ERR_UNSUPPORTED, "aggregate %u: sum / avg need int64, uint64 or double", a);
        }
        if (A.op == YTGPU_AGG_ARGMIN || A.op == YTGPU_AGG_ARGMAX) {
            if (A.by_column < 0 || (u64)A.by_column >= columns_total)
                return make_status(YTGPU_ERR_INVALID_ARGUMENT, "aggregate %u: by_column out of range", a);
            if (!is_string(A.by_column) && !aggregatable_type(value_columns[A.by_column].value_type))
                return make_status(YTGPU_ERR_UNSUPPORTED, "aggregate %u: by_column is not a fixed-width scalar", a);
        }
    }
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    out->group_count = 0;
    if (n == 0) return Status{};

    std::vector<StagedColumn> sk(key_count), sv(value_count);
    KeyColumns K{};
    K.count = key_count;
    for (u32 k = 0; k < key_count; ++k) {
        YTGPU_TRY(stage_column(ctx, &key_columns[k], &sk[k]));
        K.col[k] = sk[k].dev;
    }
    for (u32 v = 0; v < value_count; ++v) YTGPU_TRY(stage_column(ctx, &value_columns[v], &sv[v]));
    std::vector<StagedStrings> ss(string_count);
    for (u32 s = 0; s < string_count; ++s) YTGPU_TRY(stage_strings(ctx, string_columns[s], &ss[s]));
    bool keys_direct = true;  // plain 64-bit key vectors: the probe compares with one load per column
    for (u32 k = 0; k < key_count; ++k)
        keys_direct = keys_direct && is_direct64(sk[k].dev) && sk[k].dev.base == 0 && !sk[k].dev.zigzag;
    const ColumnDev pred_dev = op != YTGPU_CMP_NONE ? sv[pred_column].dev : ColumnDev{};
    const u64 constant = pred ? pred->constant : 0;

    // step 1
    KeyTable T;
    YTGPU_TRY(assign_key_slots(ctx, KC_GROUPBY, K, keys_direct, pred_dev, op, constant, n, hint, &T));
    const u64 cap = T.cap;
    DevBuf<u32> counter;
    YTGPU_TRY(counter.allocate(ctx, 1));
    const u32 threads = 256;
    const u32 all_rows_blocks = (u32)((n + threads - 1) / threads);

    // step 2
    std::vector<DevBuf<unsigned long long>> acc(aggregate_count), nn(aggregate_count), rows(aggregate_count);
    std::vector<AggState> states(aggregate_count);
    bool any_strings = false;
    for (u32 a = 0; a < aggregate_count; ++a) {
        const ytgpu_aggregate& A = aggregates[a];
        const bool arg = A.op == YTGPU_AGG_ARGMIN || A.op == YTGPU_AGG_ARGMAX;
        if (is_string(A.column) || (arg && is_string(A.by_column))) {
            // string state: the selected row, or the non-NULL count
            AggState S{nullptr, nullptr, nullptr};
            if (A.op == YTGPU_AGG_COUNT) {
                YTGPU_TRY(nn[a].allocate(ctx, cap));
                YTGPU_CUDA_TRY(cudaMemsetAsync(nn[a].p, 0, cap * 8, ctx->stream));
                S.nn = nn[a].p;
            } else {
                YTGPU_TRY(rows[a].allocate(ctx, cap));
                YTGPU_CUDA_TRY(cudaMemsetAsync(rows[a].p, 0xff, cap * 8, ctx->stream));
                S.row = rows[a].p;
            }
            states[a] = S;
            const bool col_str = is_string(A.column), by_str = arg && is_string(A.by_column);
            const ColumnDev col = col_str ? ColumnDev{} : sv[A.column].dev;
            const StringDev cs = col_str ? ss[A.column - value_count].dev : StringDev{};
            const ColumnDev by = arg && !by_str ? sv[A.by_column].dev : ColumnDev{};
            const StringDev bs = by_str ? ss[A.by_column - value_count].dev : StringDev{};
            KernelTimer t(ctx, KC_GROUPBY);
            mg_accumulate_strings_kernel<<<all_rows_blocks, threads, 0, ctx->stream>>>(A.op, col, cs, by, bs, n, T.slot_of_row.p, S,
                                                                                      ctx->dev_err);
            YTGPU_CUDA_TRY(cudaGetLastError());
            any_strings = true;
            continue;
        }
        YTGPU_TRY(accumulate_scalar(ctx, A.op, sv[A.column].dev, arg ? sv[A.by_column].dev : ColumnDev{}, n, cap, T.slot_of_row.p, &acc[a],
                                    &nn[a], &rows[a], &states[a]));
    }
    if (any_strings) YTGPU_TRY(check_device_errors(ctx));  // a string that leaves its heap

    // step 3
    const u64 max_groups = std::min<u64>(n, cap);
    DevBuf<u64> cfirst;
    DevBuf<u32> cslot, slot_sorted;
    YTGPU_TRY(cfirst.allocate(ctx, max_groups));
    YTGPU_TRY(cslot.allocate(ctx, max_groups));
    YTGPU_CUDA_TRY(cudaMemsetAsync(counter.p, 0, 4, ctx->stream));
    mg_compact_kernel<<<blocks_for(cap, 256, 8), 256, 0, ctx->stream>>>(T.rep.p, cap, T.first.p, cfirst.p, cslot.p, counter.p);
    ctx->count_launch();
    u32 g32 = 0;
    YTGPU_CUDA_TRY(cudaMemcpyAsync(&g32, counter.p, 4, cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    const u64 g = g32;
    out->group_count = g;
    if (g > out->capacity)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "result has %llu groups, capacity is %llu", (unsigned long long)g,
                           (unsigned long long)out->capacity);
    if (g == 0) return Status{};

    SortScratch scratch;
    PermRef perm;
    const u64* cptr[1] = {cfirst.p};
    YTGPU_TRY(radix_sort_chunks(ctx, cptr, 1, g, &scratch, &perm));
    YTGPU_TRY(slot_sorted.allocate(ctx, g));

    std::vector<OutBuf<u64>> tk(key_count), tv(aggregate_count);
    std::vector<OutBuf<u8>> tkn(key_count), tvn(aggregate_count);
    OutBuf<u64> tcounts, tfirst;
    KeyOutputs O{};
    for (u32 k = 0; k < key_count; ++k) {
        if (!out->keys[k] || !out->key_null[k]) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null key output %u", k);
        YTGPU_TRY(tk[k].prepare(ctx, out->keys[k], g, out_mem));
        YTGPU_TRY(tkn[k].prepare(ctx, out->key_null[k], g, out_mem));
        O.keys[k] = tk[k].p;
        O.key_null[k] = tkn[k].p;
    }
    YTGPU_TRY(tcounts.prepare(ctx, out->counts, g, out_mem));
    YTGPU_TRY(tfirst.prepare(ctx, out->first_rows, g, out_mem));
    const u32 gblocks = (u32)((g + threads - 1) / threads);
    mg_emit_keys_kernel<<<gblocks, threads, 0, ctx->stream>>>(K, perm.plan, perm.idx[0], perm.idx[1], g, cslot.p, T.first.p, T.counts.p, O, tcounts.p,
                                                             tfirst.p, slot_sorted.p);
    ctx->count_launch();
    for (u32 a = 0; a < aggregate_count; ++a) {
        if (!out->values[a] || !out->value_null[a]) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null aggregate output %u", a);
        YTGPU_TRY(tv[a].prepare(ctx, out->values[a], g, out_mem));
        YTGPU_TRY(tvn[a].prepare(ctx, out->value_null[a], g, out_mem));
        const ytgpu_aggregate& A = aggregates[a];
        const bool row_result = is_string(A.column) && A.op != YTGPU_AGG_COUNT;
        const ColumnDev col = is_string(A.column) ? ColumnDev{} : sv[A.column].dev;
        mg_finalize_kernel<<<gblocks, threads, 0, ctx->stream>>>(A.op, col, 0, g, slot_sorted.p, states[a], tv[a].p, tvn[a].p, row_result);
        ctx->count_launch();
        YTGPU_TRY(tv[a].download(ctx, g));
        YTGPU_TRY(tvn[a].download(ctx, g));
    }
    YTGPU_CUDA_TRY(cudaGetLastError());
    for (u32 k = 0; k < key_count; ++k) {
        YTGPU_TRY(tk[k].download(ctx, g));
        YTGPU_TRY(tkn[k].download(ctx, g));
    }
    YTGPU_TRY(tcounts.download(ctx, g));
    YTGPU_TRY(tfirst.download(ctx, g));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return Status{};
}

}  // namespace

extern "C" {

int ytgpu_scan_filter_groupby_multi(ytgpu_context* h, const ytgpu_column_view* key_columns, uint32_t key_count,
                                    const ytgpu_column_view* value_columns, uint32_t value_count, const ytgpu_aggregate* aggregates,
                                    uint32_t aggregate_count, const ytgpu_predicate* predicate, int32_t predicate_column,
                                    uint64_t group_count_hint, ytgpu_groupby_multi_result* out, int out_mem, ytgpu_error* err) {
    return ytgpu_scan_filter_groupby_multi_strings(h, key_columns, key_count, value_columns, value_count, aggregates, aggregate_count,
                                                   predicate, predicate_column, group_count_hint, out, out_mem, nullptr, 0, err);
}

int ytgpu_scan_filter_groupby_multi_strings(ytgpu_context* h, const ytgpu_column_view* key_columns, uint32_t key_count,
                                            const ytgpu_column_view* value_columns, uint32_t value_count,
                                            const ytgpu_aggregate* aggregates, uint32_t aggregate_count,
                                            const ytgpu_predicate* predicate, int32_t predicate_column, uint64_t group_count_hint,
                                            ytgpu_groupby_multi_result* out, int out_mem, const ytgpu_string_column* string_columns,
                                            uint32_t string_count, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, groupby_multi_impl(as_context(h), key_columns, key_count, value_columns, value_count, aggregates,
                                              aggregate_count, predicate, predicate_column, group_count_hint, out, out_mem,
                                              string_columns, string_count));
}

}  // extern "C"
