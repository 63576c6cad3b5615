// join.cu — hash JOIN: the join table (built once from the foreign keys, probed any number of times) with inner, left,
// left semi and left only joins over key tuples, the one-shot ytgpu_hash_join over it, and the gathers that turn its pairs
// into columns.
//
// Replaces the row-by-row hash lookup of YT QL's JoinOpHelper (library/query/engine/cg_routines/registry.cpp): the foreign
// rows are built into a table keyed on the join key, every primary row looks its key up there.  The build (steps 0-2)
// depends on the foreign side only; a probe (steps 3-5) on the table and one set of primary rows:
//   0. decode: the foreign key tuples, decoded to 64-bit payloads plus a null mask per row, into the table's own memory: a
//      probe compares against them with one plain load per column, and never reads the caller's foreign columns.
//   1. assign: the GROUP BY assign step (key_tuple.cuh) over the foreign keys, sized for the foreign row count: rep[slot] =
//      a foreign row holding the tuple, counts[slot] = the foreign rows of the tuple, slot_of_row[f] = f's slot.  Under
//      the SQL NULL rule the assign step's predicate (null mask == 0) keeps the rows with a NULL component out.
//   2. per-key lists: the counts, scanned, give each slot's start; one stable radix sort of the foreign rows by slot lists
//      every slot's rows in ascending order (an atomic scatter would not be stable, and the order is part of the result).
//   3. probe: each primary row loads and hashes its tuple with the same hash_tuple, walks the table comparing against the
//      table's decoded tuples at the slot's row and stops at an empty slot: its slot, and its pair count.  SEMI / ANTI
//      run the existence probe instead: one flag per primary row, no slot and no count.
//   4. offsets: the pair counts (or flags), scanned; the total is read back (a count query ends here).  SEMI / ANTI list
//      the flagged rows through the scanned flags.
//   5. write: each CTA owns a fixed range of output positions, finds its first primary row by binary search over the
//      offsets and walks the rows and their slot lists from there, galloping over rows without pairs.  So a key with 10^6
//      foreign rows spreads over about 245 CTAs, and a run of r unmatched rows costs a thread about 2 log2(r) loads:
//      neither serialises on one thread.
// String key components become UINT64 id columns before step 0 and step 3, and the steps above run on them unchanged.  The
// build keeps a string dictionary per string key (string_dict.cuh): a compacted copy of the foreign values and the hash
// table of their first rows.  A foreign value's id is the first foreign row holding its bytes; a primary value's id is what
// the dictionary lookup finds, or kStringDictMiss, which no foreign id equals.  NULL stays NULL.
#include <algorithm>
#include <new>
#include <vector>

#include "columnar.cuh"
#include "context.cuh"
#include "key_tuple.cuh"
#include "radix_sort.cuh"
#include "scan.cuh"
#include "string_dict.cuh"

using namespace ytgpu;

namespace {

constexpr u32 kNoRow = YTGPU_JOIN_NO_ROW;
// Rows per side: slots and rows are 32-bit.  The foreign side is also sorted by slot, and the radix sort takes fewer than
// 2^30 rows (its look-back words carry 30-bit counts).
constexpr u64 kMaxPrimaryRows = 1ull << 30;
constexpr u64 kMaxForeignRows = (1ull << 30) - 1;

// The table's own copy of the foreign key tuples (step 0): payload of key k of row f at w[k * rows + f], NULL as 0.
struct TableKeys {
    const u64* w;
    const u8* nulls;  // bit k: key k of the row is NULL; nullptr when no row in the table has a NULL component
    u64 rows;
};

template <int NK>
__device__ __forceinline__ KeyTuple load_table_tuple(const TableKeys& F, u32 count, u32 row) {
    KeyTuple t;
    t.nulls = F.nulls ? F.nulls[row] : 0u;
#pragma unroll
    for (u32 k = 0; k < (u32)(NK ? NK : kMaxGroupKeys); ++k) t.w[k] = (NK || k < count) ? F.w[(u64)k * F.rows + row] : 0;
    return t;
}

// Step 0: every foreign row's tuple, decoded once.  DIRECT: every key column is a plain 64-bit vector.
template <bool DIRECT>
__global__ void __launch_bounds__(256) hj_decode_keys_kernel(const KeyColumns K, u64 n, u64* __restrict__ w, u8* __restrict__ nulls) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        u32 m = 0;
#pragma unroll 1
        for (u32 k = 0; k < K.count; ++k) {
            bool nul = false;
            const u64 v = DIRECT ? reinterpret_cast<const u64*>(K.col[k].values)[(u64)K.col[k].start + i] : decode_at(K.col[k], (i64)i, &nul);
            w[(u64)k * n + i] = nul ? 0 : v;
            m |= (u32)nul << k;
        }
        nulls[i] = (u8)m;
    }
}

// Step 3, with the two-rows-in-flight structure of mg_assign_kernel: the probe is a chain of dependent loads (key -> slot ->
// the foreign row's key), so both rows' loads are issued before either is used.  DIRECT: every primary key column is a
// plain 64-bit vector (the foreign side is always the table's decoded copy); NK: 1, 2 or 0 (P.count columns).  emit(row,
// slot) runs once per primary row, slot = kNoSlot without a match.  never_match: a primary tuple with a NULL component
// matches nothing (the SQL rule) and does not touch the table.
template <bool DIRECT, int NK, class Emit>
__device__ __forceinline__ void probe_rows(const KeyColumns& P, const TableKeys& F, u64 n, const u32* __restrict__ rep, u64 mask,
                                           bool never_match, Emit emit) {
    constexpr int R = NK ? 2 : 1;  // 3+ key columns: four 8-word tuples in flight would cost the occupancy
    const u64 stride = (u64)gridDim.x * blockDim.x;
    u64 base = (u64)blockIdx.x * blockDim.x + threadIdx.x;
    KeyTuple ahead[R];
#pragma unroll
    for (int j = 0; j < R; ++j)
        if (base + (u64)j * stride < n) ahead[j] = load_tuple<DIRECT, NK>(P, base + (u64)j * stride);
    for (; base < n; base += stride * R) {
        u64 row[R], b[R];
        u32 r[R], slot[R];
        bool valid[R], look[R];
        KeyTuple mine[R], cand[R];
#pragma unroll
        for (int j = 0; j < R; ++j) {
            mine[j] = ahead[j];
            const u64 nxt = base + stride * R + (u64)j * stride;
            if (nxt < n) ahead[j] = load_tuple<DIRECT, NK>(P, nxt);
        }
#pragma unroll
        for (int j = 0; j < R; ++j) {
            row[j] = base + (u64)j * stride;
            valid[j] = row[j] < n;
            look[j] = valid[j] && !(never_match && mine[j].nulls);
            slot[j] = kNoSlot;
            b[j] = look[j] ? hash_tuple<NK>(P, mine[j]) & mask : 0;
            r[j] = look[j] ? rep[b[j]] : kNoSlot;
        }
#pragma unroll
        for (int j = 0; j < R; ++j)
            if (r[j] != kNoSlot) cand[j] = load_table_tuple<NK>(F, P.count, r[j]);
#pragma unroll
        for (int j = 0; j < R; ++j) {
            if (!look[j]) continue;
            u32 rr = r[j];
            bool have = true;  // cand[j] holds the key of foreign row rr
            u64 bb = b[j];
            for (u64 probes = 0; probes <= mask && rr != kNoSlot; ++probes) {
                if (same_tuple<NK>(P, mine[j], have ? cand[j] : load_table_tuple<NK>(F, P.count, rr))) {
                    slot[j] = (u32)bb;
                    break;
                }
                bb = (bb + 1) & mask;
                rr = rep[bb];
                have = false;
            }
        }
#pragma unroll
        for (int j = 0; j < R; ++j)
            if (valid[j]) emit(row[j], slot[j]);
    }
}

// Step 3 of INNER / LEFT: the slot and the pair count of every primary row.
template <bool DIRECT, int NK>
__global__ void __launch_bounds__(256) hj_probe_kernel(const KeyColumns P, const TableKeys F, u64 n, const u32* __restrict__ rep, u64 mask,
                                                       const unsigned long long* __restrict__ counts, int left, int never_match,
                                                       u32* __restrict__ probe_slot, u64* __restrict__ pair_counts) {
    probe_rows<DIRECT, NK>(P, F, n, rep, mask, never_match, [&](u64 row, u32 slot) {
        probe_slot[row] = slot;
        pair_counts[row] = slot != kNoSlot ? (u64)counts[slot] : (left ? 1 : 0);
    });
}

// Step 3 of SEMI / ANTI, the existence probe: it stops at the first match, reads neither the counts nor the per-key lists,
// and writes one flag per primary row: 1 when the row is listed (SEMI: it has a match; ANTI: it has none).
template <bool DIRECT, int NK>
__global__ void __launch_bounds__(256) hj_exists_kernel(const KeyColumns P, const TableKeys F, u64 n, const u32* __restrict__ rep, u64 mask,
                                                        int never_match, int anti, u64* __restrict__ flags) {
    probe_rows<DIRECT, NK>(P, F, n, rep, mask, never_match, [&](u64 row, u32 slot) { flags[row] = (slot != kNoSlot) != (anti != 0); });
}

// Step 4 of SEMI / ANTI: the scanned flags -> the ascending list of flagged rows.
__global__ void __launch_bounds__(256) hj_list_rows_kernel(const u64* __restrict__ offsets, u64 n, const u64* __restrict__ total,
                                                           u32* __restrict__ out) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        const u64 end = i + 1 < n ? offsets[i + 1] : *total;
        if (end != offsets[i]) out[offsets[i]] = (u32)i;
    }
}

// The sort key of step 2: a foreign row's slot.
__global__ void __launch_bounds__(256) hj_slot_keys_kernel(const u32* __restrict__ slot_of_row, u64 n, u64* __restrict__ keys) {
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) keys[i] = slot_of_row[i];
}

// Step 5: CTA c writes output positions [c * kWriteTile, (c + 1) * kWriteTile), thread t the kWriteItems consecutive ones
// from c * kWriteTile + t * kWriteItems, into shared memory first so that the global stores are coalesced.
constexpr int kWriteThreads = 256;
constexpr int kWriteItems = 16;
constexpr int kWriteTile = kWriteThreads * kWriteItems;
__device__ __forceinline__ u32 tile_index(u32 i) { return i + i / kWriteItems; }  // one pad word per thread: no bank conflicts

__global__ void __launch_bounds__(kWriteThreads) hj_write_pairs_kernel(const u64* __restrict__ offsets, u64 n, u64 total,
                                                                       const u32* __restrict__ probe_slot, const u64* __restrict__ slot_start,
                                                                       const u32* __restrict__ rows_by_slot, u32* __restrict__ out_primary,
                                                                       u32* __restrict__ out_foreign) {
    __shared__ u32 s_p[kWriteTile + kWriteThreads], s_f[kWriteTile + kWriteThreads];
    const u64 tile0 = (u64)blockIdx.x * kWriteTile;
    const u64 first = tile0 + (u64)threadIdx.x * kWriteItems;
    if (first < total) {
        u64 lo = 0, hi = n;  // the last row p with offsets[p] <= first (offsets[0] = 0): it has a pair there
        while (hi - lo > 1) {
            const u64 mid = (lo + hi) >> 1;
            if (offsets[mid] <= first) lo = mid;
            else hi = mid;
        }
        u64 p = lo, start = offsets[p], end = p + 1 < n ? offsets[p + 1] : total;
#pragma unroll 1
        for (u32 k = 0; k < (u32)kWriteItems; ++k) {
            const u64 o = first + k;
            if (o >= total) break;
            if (o >= end) {
                const u64 next_end = p + 2 < n ? offsets[p + 2] : total;
                if (o < next_end) {  // the next row: the common case, one load
                    ++p;
                    start = end;
                    end = next_end;
                } else {
                    // A run of rows without pairs (INNER misses; a sorted primary table against a dimension that covers
                    // part of its key range): the last q with offsets[q] <= o by a gallop from p + 2 (offsets[p + 2] =
                    // next_end <= o) and a binary search inside the last step, O(log run) loads rather than one per row,
                    // so no thread does more than kWriteItems such searches.
                    u64 q = p + 2, step = 1;
                    while (q + step < n && offsets[q + step] <= o) {
                        q += step;
                        step <<= 1;
                    }
                    u64 qe = q + step < n ? q + step : n;  // offsets[qe] > o, or qe == n
                    while (qe - q > 1) {
                        const u64 mid = (q + qe) >> 1;
                        if (offsets[mid] <= o) q = mid;
                        else qe = mid;
                    }
                    p = q;
                    start = offsets[p];
                    end = p + 1 < n ? offsets[p + 1] : total;
                }
            }
            const u32 s = probe_slot[p];
            const u32 i = tile_index(threadIdx.x * kWriteItems + k);
            s_p[i] = (u32)p;
            s_f[i] = s == kNoSlot ? kNoRow : rows_by_slot[slot_start[s] + (o - start)];
        }
    }
    __syncthreads();
    const u32 m = (u32)std::min<u64>((u64)kWriteTile, total - tile0);
    for (u32 i = threadIdx.x; i < m; i += kWriteThreads) {
        out_primary[tile0 + i] = s_p[tile_index(i)];
        out_foreign[tile0 + i] = s_f[tile_index(i)];
    }
}

// ytgpu_gather_column: one row per thread; each warp writes its 32 null bits as one word.  The grid covers whole 64-row
// words, so the bits past `count` are written as zeros.
__global__ void __launch_bounds__(256) hj_gather_kernel(const ColumnDev c, u64 column_rows, const u32* __restrict__ rows, u64 count,
                                                        u64* __restrict__ out, u32* __restrict__ out_bits, unsigned long long* null_count,
                                                        u32* err_word) {
    const u64 padded = (count + 63) / 64 * 64;
    u32 bad = 0, nulls = 0;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < padded; i += (u64)gridDim.x * blockDim.x) {
        bool nul = false;
        if (i < count) {
            const u32 r = rows[i];
            u64 v = 0;
            if (r == kNoRow) {
                nul = true;
            } else if ((u64)r >= column_rows) {
                bad = 1;
                nul = true;
            } else {
                v = decode_at(c, (i64)r, &nul);
            }
            out[i] = nul ? 0 : v;
        }
        const u32 m = __ballot_sync(0xffffffffu, nul);
        if ((threadIdx.x & 31) == 0) {
            out_bits[i >> 5] = m;
            nulls += __popc(m);
        }
    }
    if (bad) atomicOr(err_word, (u32)DE_ROW_OUT_OF_RANGE);
    if ((threadIdx.x & 31) == 0 && nulls) atomicAdd(null_count, (unsigned long long)nulls);
}

__global__ void __launch_bounds__(256) hj_gather_strings_kernel(const u64* __restrict__ starts, const u32* __restrict__ lengths,
                                                                const u8* __restrict__ nulls, u64 column_rows, const u32* __restrict__ rows,
                                                                u64 count, u64* __restrict__ out_starts, u32* __restrict__ out_lengths,
                                                                u8* __restrict__ out_nulls, u32* err_word) {
    u32 bad = 0;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (u64)gridDim.x * blockDim.x) {
        const u32 r = rows[i];
        bool nul = r == kNoRow;
        if (!nul && (u64)r >= column_rows) {
            bad = 1;
            nul = true;
        }
        nul = nul || (nulls && nulls[r]);
        out_starts[i] = nul ? 0 : starts[r];
        out_lengths[i] = nul ? 0 : lengths[r];
        out_nulls[i] = nul ? 1 : 0;
    }
    if (bad) atomicOr(err_word, (u32)DE_ROW_OUT_OF_RANGE);
}

bool join_key_type(u8 t) { return t == YTGPU_TYPE_INT64 || t == YTGPU_TYPE_UINT64 || t == YTGPU_TYPE_DOUBLE || t == YTGPU_TYPE_BOOLEAN; }

Status check_side(const ytgpu_column_view* keys, u32 key_count, const char* side, u64 max_rows, u64* rows) {
    for (u32 k = 0; k < key_count; ++k) {
        if (keys[k].value_count < 0 || keys[k].start_index < 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "%s key %u: negative column range", side, k);
        if (keys[k].value_count != keys[0].value_count)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "%s key columns differ in length", side);
        if (!join_key_type(keys[k].value_type))
            return make_status(YTGPU_ERR_UNSUPPORTED, "%s key %u: value type 0x%x is not INT64, UINT64, DOUBLE or BOOLEAN", side, k,
                               keys[k].value_type);
    }
    *rows = (u64)keys[0].value_count;
    if (*rows > max_rows)
        return make_status(YTGPU_ERR_UNSUPPORTED, "%s side: at most %llu rows (slots and rows are 32-bit)", side, (unsigned long long)max_rows);
    return Status{};
}

// The string keys of one side: one length, which is the numeric keys' when there are any (have_rows: *rows holds it).
Status check_string_side(const ytgpu_string_column* strings, u32 count, bool have_rows, const char* side, u64 max_rows, u64* rows) {
    for (u32 s = 0; s < count; ++s) {
        const ytgpu_string_column& c = strings[s];
        if (s == 0 && !have_rows) *rows = c.row_count;
        if (c.row_count != *rows) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "%s string key %u differs in length from the other keys", side, s);
        if (c.mem != YTGPU_MEM_DEVICE && c.mem != YTGPU_MEM_HOST)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "%s string key %u: mem must be YTGPU_MEM_DEVICE or YTGPU_MEM_HOST", side, s);
        if ((c.row_count && (!c.starts || !c.lengths)) || (c.heap_bytes && !c.heap))  // an empty heap (all "" / NULL) is never read
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "%s string key %u: null heap, starts or lengths", side, s);
    }
    if (*rows > max_rows)
        return make_status(YTGPU_ERR_UNSUPPORTED, "%s side: at most %llu rows (slots and rows are 32-bit)", side, (unsigned long long)max_rows);
    return Status{};
}

bool known_kind(int kind) {
    return kind == YTGPU_JOIN_INNER || kind == YTGPU_JOIN_LEFT || kind == YTGPU_JOIN_SEMI || kind == YTGPU_JOIN_ANTI;
}

// A built table (ytgpu_join_table): the foreign side after steps 0-2.  Immutable once built; its buffers are the
// context's stream-ordered memory.
struct JoinTable {
    Context* ctx = nullptr;
    u32 key_count = 0;           // the tuple's components: the numeric keys, then string_count string keys
    u32 string_count = 0;
    u8 types[kMaxGroupKeys] = {};
    int nulls = YTGPU_JOIN_NULLS_EQUAL;
    u64 rows = 0;                // foreign rows
    bool null_keys = false;      // a row in the table may have a NULL component: the probe loads the null masks
    bool listed = false;         // step 2 ran (a one-shot count query skips it: it writes no pairs)
    DevBuf<u64> keys;            // step 0: key_count * rows payloads, column by column
    DevBuf<u8> null_mask;        // step 0: bit k = key k of the row is NULL
    KeyTable T;                  // step 1: rep and counts (slot_of_row and first are released after step 2)
    DevBuf<u64> slot_start;      // step 2: exclusive scan of counts
    DevBuf<u32> rows_by_slot;    // step 2: the foreign rows stable-sorted by slot, slot s at [slot_start[s], + counts[s])
    StringDict dicts[kMaxGroupKeys];  // string key s: dicts[s]

    TableKeys dev() const { return TableKeys{keys.p, null_keys ? null_mask.p : nullptr, rows}; }
};

// Steps 0-2 over the staged foreign key columns KF (nf rows).  list_rows = false skips step 2: the table then answers
// counts and SEMI / ANTI probes, not INNER / LEFT pair writes.  Synchronises once for the assign step's error word (more
// when a full table doubles), and the sort reads its plan back once from 2^18 rows.
Status build_table(Context* ctx, const KeyColumns& KF, bool foreign_direct, u64 nf, int nulls, bool list_rows, JoinTable* J) {
    J->ctx = ctx;
    J->key_count = KF.count;
    for (u32 k = 0; k < KF.count; ++k) J->types[k] = KF.col[k].value_type;
    J->nulls = nulls;
    J->rows = nf;
    const bool never_match = nulls == YTGPU_JOIN_NULLS_NEVER_MATCH;
    // under the SQL rule no row with a NULL component enters the table; plain 64-bit columns have no NULLs at all
    J->null_keys = !never_match && !foreign_direct;
    YTGPU_TRY(J->keys.allocate(ctx, nf * KF.count));
    YTGPU_TRY(J->null_mask.allocate(ctx, nf));
    if (nf == 0) {  // a one-slot empty table: every probe ends at once
        J->T.cap = 1;
        YTGPU_TRY(J->T.rep.allocate(ctx, 1));
        YTGPU_TRY(J->T.counts.allocate(ctx, 1));
        YTGPU_CUDA_TRY(cudaMemsetAsync(J->T.rep.p, 0xff, 4, ctx->stream));
        YTGPU_CUDA_TRY(cudaMemsetAsync(J->T.counts.p, 0, 8, ctx->stream));
        J->listed = true;
        return Status{};
    }
    {  // step 0
        KernelTimer t(ctx, KC_JOIN);
        const u32 blocks = blocks_for(nf, 256, 8);
        if (foreign_direct) hj_decode_keys_kernel<true><<<blocks, 256, 0, ctx->stream>>>(KF, nf, J->keys.p, J->null_mask.p);
        else hj_decode_keys_kernel<false><<<blocks, 256, 0, ctx->stream>>>(KF, nf, J->keys.p, J->null_mask.p);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    // step 1; the SQL rule keeps the rows whose null mask is not 0 out through the assign step's predicate
    ColumnDev mask_col{};
    int op = YTGPU_CMP_NONE;
    if (never_match) {
        mask_col.count = (i64)nf;
        mask_col.values = J->null_mask.p;
        mask_col.values_count = nf;
        mask_col.bit_width = 8;
        mask_col.has_values = 1;
        mask_col.value_type = YTGPU_TYPE_UINT64;
        op = YTGPU_CMP_EQ;
    }
    YTGPU_TRY(assign_key_slots(ctx, KC_JOIN, KF, foreign_direct, mask_col, op, 0, nf, nf, &J->T));
    J->T.first.reset();
    if (!list_rows) return Status{};

    // step 2 (rows kept out by the SQL rule have slot kNoSlot: they sort behind every listed row)
    DevBuf<u64> sort_keys, scan_sums, total;
    YTGPU_TRY(J->slot_start.allocate(ctx, J->T.cap));
    YTGPU_TRY(scan_sums.allocate(ctx, scan_block_count(J->T.cap)));
    YTGPU_TRY(total.allocate(ctx, 1));
    YTGPU_CUDA_TRY(cudaMemcpyAsync(J->slot_start.p, J->T.counts.p, J->T.cap * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    YTGPU_TRY(sort_keys.allocate(ctx, nf));
    {
        KernelTimer t(ctx, KC_JOIN, 4);
        exclusive_scan_u64(ctx->stream, J->slot_start.p, J->T.cap, scan_sums.p, total.p);
        hj_slot_keys_kernel<<<blocks_for(nf, 256, 8), 256, 0, ctx->stream>>>(J->T.slot_of_row.p, nf, sort_keys.p);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    J->T.slot_of_row.reset();
    SortScratch scratch;
    PermRef perm;
    const u64* chunk[1] = {sort_keys.p};
    YTGPU_TRY(radix_sort_chunks(ctx, chunk, 1, nf, &scratch, &perm));
    YTGPU_TRY(J->rows_by_slot.allocate(ctx, nf));
    YTGPU_TRY(materialize_perm(ctx, perm, nf, J->rows_by_slot.p));
    J->listed = true;
    return Status{};
}

// Steps 3-5 of one probe: the staged primary key columns KP (np >= 1 rows) against table J.  The caller has checked the
// arguments and written *out_count = 0.
// read_errors: the device error word is read with the count (the string lookups' bounds checks).
Status probe_table(Context* ctx, const JoinTable& J, const KeyColumns& KP, bool primary_direct, u64 np, int kind, u32* out_primary,
                   u32* out_foreign, u64 capacity, u64* out_count, int out_mem, bool read_errors = false) {
    const TableKeys F = J.dev();
    const u64 mask = J.T.cap - 1;
    const int never_match = J.nulls == YTGPU_JOIN_NULLS_NEVER_MATCH;
    const u32 key_count = KP.count;
    const u32 blocks = blocks_for((np + 1) / 2, 256, 16);
    const bool host = out_mem == YTGPU_MEM_HOST;
    DevBuf<u64> offsets, scan_sums, total;
    YTGPU_TRY(offsets.allocate(ctx, np));
    YTGPU_TRY(scan_sums.allocate(ctx, scan_block_count(np)));
    YTGPU_TRY(total.allocate(ctx, 1));
#define YTGPU_HJ_DISPATCH(LAUNCH)                           \
    if (primary_direct && key_count == 1) LAUNCH(true, 1);  \
    else if (primary_direct && key_count == 2) LAUNCH(true, 2); \
    else if (primary_direct) LAUNCH(true, 0);               \
    else if (key_count == 1) LAUNCH(false, 1);              \
    else if (key_count == 2) LAUNCH(false, 2);              \
    else LAUNCH(false, 0)

    if (kind == YTGPU_JOIN_SEMI || kind == YTGPU_JOIN_ANTI) {
        {  // steps 3 and 4: flags, their scan, and the list of flagged rows
            KernelTimer t(ctx, KC_JOIN, out_primary ? 5 : 4);
            const int anti = kind == YTGPU_JOIN_ANTI;
#define YTGPU_HJ_EXISTS(D, N) \
    hj_exists_kernel<D, N><<<blocks, 256, 0, ctx->stream>>>(KP, F, np, J.T.rep.p, mask, never_match, anti, offsets.p)
            YTGPU_HJ_DISPATCH(YTGPU_HJ_EXISTS);
#undef YTGPU_HJ_EXISTS
            exclusive_scan_u64(ctx->stream, offsets.p, np, scan_sums.p, total.p);
            YTGPU_CUDA_TRY(cudaGetLastError());
        }
        // the list has at most np rows: with that much DEVICE capacity it goes straight to the output, and the count is
        // the one read-back; with less, it is staged and copied out once its length is known, in either memory space
        DevBuf<u32> staged;
        u32* dst = out_primary;
        if (out_primary && (host || capacity < np)) {
            YTGPU_TRY(staged.allocate(ctx, np));
            dst = staged.p;
        }
        if (out_primary) {
            hj_list_rows_kernel<<<blocks_for(np, 256, 16), 256, 0, ctx->stream>>>(offsets.p, np, total.p, dst);
            YTGPU_CUDA_TRY(cudaGetLastError());
        }
        u64 rows = 0;
        YTGPU_CUDA_TRY(cudaMemcpyAsync(&rows, total.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
        if (read_errors) YTGPU_TRY(check_device_errors(ctx));  // synchronises
        else YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
        *out_count = rows;
        if (!out_primary) return Status{};
        if (rows > capacity)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "the join lists %llu rows, capacity is %llu", (unsigned long long)rows,
                               (unsigned long long)capacity);
        if (dst != out_primary && rows) {
            YTGPU_TRY(copy_out(ctx, out_primary, dst, rows * 4, out_mem));
            YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
        }
        return Status{};
    }

    // step 3
    DevBuf<u32> probe_slot;
    YTGPU_TRY(probe_slot.allocate(ctx, np));
    {
        KernelTimer t(ctx, KC_JOIN);
        const int left = kind == YTGPU_JOIN_LEFT;
#define YTGPU_HJ_PROBE(D, N)                                                                                                    \
    hj_probe_kernel<D, N><<<blocks, 256, 0, ctx->stream>>>(KP, F, np, J.T.rep.p, mask, J.T.counts.p, left, never_match, probe_slot.p, \
                                                           offsets.p)
        YTGPU_HJ_DISPATCH(YTGPU_HJ_PROBE);
#undef YTGPU_HJ_PROBE
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
#undef YTGPU_HJ_DISPATCH
    // step 4
    {
        KernelTimer t(ctx, KC_JOIN, 3);
        exclusive_scan_u64(ctx->stream, offsets.p, np, scan_sums.p, total.p);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    u64 pairs = 0;
    YTGPU_CUDA_TRY(cudaMemcpyAsync(&pairs, total.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (read_errors) YTGPU_TRY(check_device_errors(ctx));  // synchronises
    else YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    *out_count = pairs;
    if (!out_primary) return Status{};
    if (pairs > capacity)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "the join has %llu pairs, pairs_capacity is %llu", (unsigned long long)pairs,
                           (unsigned long long)capacity);
    if (pairs == 0) return Status{};
    if (!J.listed) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "the table was built without its per-key row lists");

    // step 5
    OutBuf<u32> dp, df;
    YTGPU_TRY(dp.prepare(ctx, out_primary, pairs, out_mem));
    YTGPU_TRY(df.prepare(ctx, out_foreign, pairs, out_mem));
    {
        KernelTimer t(ctx, KC_JOIN);
        const u64 tiles = (pairs + kWriteTile - 1) / kWriteTile;
        hj_write_pairs_kernel<<<(u32)tiles, kWriteThreads, 0, ctx->stream>>>(offsets.p, np, pairs, probe_slot.p, J.slot_start.p,
                                                                             J.rows_by_slot.p, dp.p, df.p);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_TRY(dp.download(ctx, pairs));
    YTGPU_TRY(df.download(ctx, pairs));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return Status{};
}

// Stages key_count columns into staged (key_count entries) and reports whether each is a plain 64-bit vector without base
// or zig-zag.
Status stage_keys(Context* ctx, const ytgpu_column_view* keys, u32 key_count, std::vector<StagedColumn>* staged, KeyColumns* K,
                  bool* direct) {
    *K = KeyColumns{};
    K->count = key_count;
    *direct = true;
    for (u32 k = 0; k < key_count; ++k) {
        YTGPU_TRY(stage_column(ctx, &keys[k], &(*staged)[k]));
        K->col[k] = (*staged)[k].dev;
        *direct = *direct && is_direct64(K->col[k]) && K->col[k].base == 0 && !K->col[k].zigzag;
    }
    return Status{};
}

Status hash_join_impl(Context* ctx, const ytgpu_column_view* primary_keys, const ytgpu_column_view* foreign_keys, u32 key_count, int kind,
                      u32* out_primary, u32* out_foreign, u64 pairs_capacity, u64* out_pair_count, int out_mem) {
    if (!primary_keys || !foreign_keys || !out_pair_count) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    if (key_count == 0 || key_count > (u32)YTGPU_JOIN_MAX_KEYS)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key column count must be in [1, %d]", YTGPU_JOIN_MAX_KEYS);
    if (kind != YTGPU_JOIN_INNER && kind != YTGPU_JOIN_LEFT) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "unknown join kind %d", kind);
    if ((out_primary == nullptr) != (out_foreign == nullptr))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "both outputs or neither (a count query) must be given");
    if (out_mem != YTGPU_MEM_DEVICE && out_mem != YTGPU_MEM_HOST)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "out_mem must be YTGPU_MEM_DEVICE or YTGPU_MEM_HOST");
    u64 np = 0, nf = 0;
    YTGPU_TRY(check_side(primary_keys, key_count, "primary", kMaxPrimaryRows, &np));
    YTGPU_TRY(check_side(foreign_keys, key_count, "foreign", kMaxForeignRows, &nf));
    for (u32 k = 0; k < key_count; ++k)
        if (primary_keys[k].value_type != foreign_keys[k].value_type)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key %u: primary type 0x%x differs from foreign type 0x%x (no implicit widening)", k,
                               primary_keys[k].value_type, foreign_keys[k].value_type);
    *out_pair_count = 0;
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    if (np == 0) return Status{};

    // both sides staged (and their column checks made) before the first launch; then one build, one probe
    std::vector<StagedColumn> sp(key_count), sf(key_count);
    KeyColumns KP, KF;
    bool primary_direct = false, foreign_direct = false;
    YTGPU_TRY(stage_keys(ctx, primary_keys, key_count, &sp, &KP, &primary_direct));
    YTGPU_TRY(stage_keys(ctx, foreign_keys, key_count, &sf, &KF, &foreign_direct));
    JoinTable J;
    YTGPU_TRY(build_table(ctx, KF, foreign_direct, nf, YTGPU_JOIN_NULLS_EQUAL, out_primary != nullptr, &J));
    return probe_table(ctx, J, KP, primary_direct, np, kind, out_primary, out_foreign, pairs_capacity, out_pair_count, out_mem);
}

Status join_table_build_impl(Context* ctx, const ytgpu_column_view* foreign_keys, u32 key_count, const ytgpu_string_column* strings,
                             u32 string_count, int nulls, JoinTable** out) {
    if ((key_count && !foreign_keys) || (string_count && !strings) || !out) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    *out = nullptr;
    const u64 total = (u64)key_count + string_count;
    if (total == 0 || total > (u64)YTGPU_JOIN_MAX_KEYS)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key column count must be in [1, %d]", YTGPU_JOIN_MAX_KEYS);
    if (nulls != YTGPU_JOIN_NULLS_EQUAL && nulls != YTGPU_JOIN_NULLS_NEVER_MATCH)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "unknown NULL rule %d", nulls);
    u64 nf = 0;
    if (key_count) YTGPU_TRY(check_side(foreign_keys, key_count, "foreign", kMaxForeignRows, &nf));
    YTGPU_TRY(check_string_side(strings, string_count, key_count != 0, "foreign", kMaxForeignRows, &nf));
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    std::vector<StagedColumn> sf(key_count);
    KeyColumns KF;
    bool foreign_direct = false;
    YTGPU_TRY(stage_keys(ctx, foreign_keys, key_count, &sf, &KF, &foreign_direct));
    JoinTable* J = new (std::nothrow) JoinTable();
    if (!J) return make_status(YTGPU_ERR_OUT_OF_MEMORY, "host allocation failed");
    // the string keys' ids: read by step 0 only, so they are freed when the build returns
    DevBuf<u64> ids[kMaxGroupKeys];
    DevBuf<u32> null_bits[kMaxGroupKeys];
    Status s = string_dicts_build(ctx, strings, string_count, nf, J->dicts, ids, null_bits);
    if (s.code == YTGPU_OK) {
        KF.count = (u32)total;
        for (u32 c = 0; c < string_count; ++c) {
            KF.col[key_count + c] = id_column(ids[c].p, null_bits[c].p, nf);
            foreign_direct = foreign_direct && !strings[c].null_bytemap;
        }
        s = build_table(ctx, KF, foreign_direct, nf, nulls, true, J);
    }
    if (s.code == YTGPU_OK) {
        J->string_count = string_count;
        for (u32 c = 0; c < string_count; ++c) J->types[key_count + c] = YTGPU_TYPE_STRING;
        const cudaError_t e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) s = cuda_status(e, "cudaStreamSynchronize");
    }
    if (s.code != YTGPU_OK) {
        delete J;
        return s;
    }
    *out = J;
    return Status{};
}

Status join_table_probe_impl(Context* ctx, const JoinTable* J, const ytgpu_column_view* primary_keys, u32 key_count,
                             const ytgpu_string_column* strings, u32 string_count, int kind, u32* out_primary, u32* out_foreign, u64 capacity,
                             u64* out_count, int out_mem) {
    if (!J || (key_count && !primary_keys) || (string_count && !strings) || !out_count)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    if (J->ctx != ctx) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "the table was built on another context");
    const u32 table_numeric = J->key_count - J->string_count;
    if (key_count != table_numeric)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "%u key columns, the table has %u", key_count, table_numeric);
    if (string_count != J->string_count)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "%u string key columns, the table has %u", string_count, J->string_count);
    if (!known_kind(kind)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "unknown join kind %d", kind);
    const bool rows_only = kind == YTGPU_JOIN_SEMI || kind == YTGPU_JOIN_ANTI;
    if (rows_only && out_foreign)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "a SEMI or ANTI join lists primary rows only: out_foreign_rows must be NULL");
    if (!rows_only && (out_primary == nullptr) != (out_foreign == nullptr))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "both outputs or neither (a count query) must be given");
    if (out_mem != YTGPU_MEM_DEVICE && out_mem != YTGPU_MEM_HOST)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "out_mem must be YTGPU_MEM_DEVICE or YTGPU_MEM_HOST");
    u64 np = 0;
    if (key_count) YTGPU_TRY(check_side(primary_keys, key_count, "primary", kMaxPrimaryRows, &np));
    YTGPU_TRY(check_string_side(strings, string_count, key_count != 0, "primary", kMaxPrimaryRows, &np));
    for (u32 k = 0; k < key_count; ++k)
        if (primary_keys[k].value_type != J->types[k])
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key %u: primary type 0x%x differs from the table's type 0x%x (no implicit widening)",
                               k, primary_keys[k].value_type, J->types[k]);
    *out_count = 0;
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    if (np == 0) return Status{};
    std::vector<StagedColumn> sp(key_count);
    KeyColumns KP;
    bool primary_direct = false;
    YTGPU_TRY(stage_keys(ctx, primary_keys, key_count, &sp, &KP, &primary_direct));
    DevBuf<u64> ids[kMaxGroupKeys];
    DevBuf<u32> null_bits[kMaxGroupKeys];
    KP.count = key_count + string_count;
    for (u32 c = 0; c < string_count; ++c) {
        YTGPU_TRY(ids[c].allocate(ctx, np));
        if (strings[c].null_bytemap) YTGPU_TRY(null_bits[c].allocate(ctx, (np + 31) / 32));
        YTGPU_TRY(string_dict_lookup(ctx, J->dicts[c], strings[c], np, ids[c].p, null_bits[c].p));
        KP.col[key_count + c] = id_column(ids[c].p, null_bits[c].p, np);
        primary_direct = primary_direct && !strings[c].null_bytemap;
    }
    return probe_table(ctx, *J, KP, primary_direct, np, kind, out_primary, out_foreign, capacity, out_count, out_mem, string_count != 0);
}

Status gather_column_impl(Context* ctx, const ytgpu_column_view* column, const u32* rows, u64 count, u64* out_values, u8* out_null_bitmap,
                          u64* out_null_count, int out_mem) {
    if (!column) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null column");
    if (out_mem != YTGPU_MEM_DEVICE && out_mem != YTGPU_MEM_HOST)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "out_mem must be YTGPU_MEM_DEVICE or YTGPU_MEM_HOST");
    if (count && (!rows || !out_values || !out_null_bitmap)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null rows or output");
    if (!join_key_type(column->value_type))
        return make_status(YTGPU_ERR_UNSUPPORTED, "value type 0x%x is not INT64, UINT64, DOUBLE or BOOLEAN", column->value_type);
    if (out_null_count) *out_null_count = 0;
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    if (count == 0) return Status{};
    StagedColumn sc;
    YTGPU_TRY(stage_column(ctx, column, &sc));
    InBuf<u32> drows;
    YTGPU_TRY(drows.stage(ctx, rows, count, out_mem));  // the row indexes live in out_mem
    const u64 words = (count + 63) / 64;
    OutBuf<u64> dv, db;
    DevBuf<unsigned long long> nulls;
    YTGPU_TRY(dv.prepare(ctx, out_values, count, out_mem));
    YTGPU_TRY(db.prepare(ctx, reinterpret_cast<u64*>(out_null_bitmap), words, out_mem));
    YTGPU_TRY(nulls.allocate(ctx, 1));
    YTGPU_CUDA_TRY(cudaMemsetAsync(nulls.p, 0, 8, ctx->stream));
    {
        KernelTimer t(ctx, KC_JOIN);
        hj_gather_kernel<<<blocks_for(words * 64, 256, 16), 256, 0, ctx->stream>>>(sc.dev, (u64)column->value_count, drows.p, count, dv.p,
                                                                                   reinterpret_cast<u32*>(db.p), nulls.p, ctx->dev_err);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_TRY(dv.download(ctx, count));
    YTGPU_TRY(db.download(ctx, words));
    unsigned long long null_count = 0;
    YTGPU_CUDA_TRY(cudaMemcpyAsync(&null_count, nulls.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_TRY(check_device_errors(ctx));  // synchronises
    if (out_null_count) *out_null_count = null_count;
    return Status{};
}

Status gather_string_column_impl(Context* ctx, const ytgpu_string_column* column, const u32* rows, u64 count, u64* out_starts,
                                 u32* out_lengths, u8* out_null_bytemap, int out_mem) {
    if (!column) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null column");
    if (out_mem != YTGPU_MEM_DEVICE && out_mem != YTGPU_MEM_HOST)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "out_mem must be YTGPU_MEM_DEVICE or YTGPU_MEM_HOST");
    if (column->mem != YTGPU_MEM_DEVICE && column->mem != YTGPU_MEM_HOST)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "column mem must be YTGPU_MEM_DEVICE or YTGPU_MEM_HOST");
    const u64 n = column->row_count;
    if (n && (!column->starts || !column->lengths)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null starts or lengths");
    if (count && (!rows || !out_starts || !out_lengths || !out_null_bytemap))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null rows or output");
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    if (count == 0) return Status{};
    // the heap is never read: only starts, lengths and the null bytemap move
    InBuf<u64> ds;
    InBuf<u32> dl;
    InBuf<u8> dn;
    const int mem = n ? column->mem : YTGPU_MEM_DEVICE;  // no rows: the caller's pointers stay
    YTGPU_TRY(ds.stage(ctx, column->starts, n, mem));
    YTGPU_TRY(dl.stage(ctx, column->lengths, n, mem));
    YTGPU_TRY(dn.stage(ctx, column->null_bytemap, n, mem));
    InBuf<u32> drows;
    YTGPU_TRY(drows.stage(ctx, rows, count, out_mem));  // the row indexes live in out_mem
    OutBuf<u64> os;
    OutBuf<u32> ol;
    OutBuf<u8> on;
    YTGPU_TRY(os.prepare(ctx, out_starts, count, out_mem));
    YTGPU_TRY(ol.prepare(ctx, out_lengths, count, out_mem));
    YTGPU_TRY(on.prepare(ctx, out_null_bytemap, count, out_mem));
    {
        KernelTimer t(ctx, KC_JOIN);
        hj_gather_strings_kernel<<<blocks_for(count, 256, 16), 256, 0, ctx->stream>>>(ds.p, dl.p, dn.p, n, drows.p, count, os.p, ol.p, on.p,
                                                                                       ctx->dev_err);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_TRY(os.download(ctx, count));
    YTGPU_TRY(ol.download(ctx, count));
    YTGPU_TRY(on.download(ctx, count));
    return check_device_errors(ctx);  // synchronises
}

}  // namespace

extern "C" {

int ytgpu_hash_join(ytgpu_context* h, const ytgpu_column_view* primary_keys, const ytgpu_column_view* foreign_keys, uint32_t key_count,
                    int kind, uint32_t* out_primary_rows, uint32_t* out_foreign_rows, uint64_t pairs_capacity, uint64_t* out_pair_count,
                    int out_mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, hash_join_impl(as_context(h), primary_keys, foreign_keys, key_count, kind, out_primary_rows, out_foreign_rows,
                                          pairs_capacity, out_pair_count, out_mem));
}

int ytgpu_join_table_build(ytgpu_context* h, const ytgpu_column_view* foreign_keys, uint32_t key_count, int nulls, ytgpu_join_table** out,
                           ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    JoinTable* t = nullptr;
    const int code = fill_error(err, join_table_build_impl(as_context(h), foreign_keys, key_count, nullptr, 0, nulls, &t));
    if (out) *out = reinterpret_cast<ytgpu_join_table*>(t);
    return code;
}

int ytgpu_join_table_probe(ytgpu_context* h, const ytgpu_join_table* table, const ytgpu_column_view* primary_keys, uint32_t key_count,
                           int kind, uint32_t* out_primary_rows, uint32_t* out_foreign_rows, uint64_t capacity, uint64_t* out_count,
                           int out_mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, join_table_probe_impl(as_context(h), reinterpret_cast<const JoinTable*>(table), primary_keys, key_count, nullptr, 0,
                                                 kind, out_primary_rows, out_foreign_rows, capacity, out_count, out_mem));
}

int ytgpu_join_table_build_strings(ytgpu_context* h, const ytgpu_column_view* foreign_keys, uint32_t key_count,
                                   const ytgpu_string_column* foreign_string_keys, uint32_t string_key_count, int nulls,
                                   ytgpu_join_table** out, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    JoinTable* t = nullptr;
    const int code = fill_error(err, join_table_build_impl(as_context(h), foreign_keys, key_count, foreign_string_keys, string_key_count,
                                                           nulls, &t));
    if (out) *out = reinterpret_cast<ytgpu_join_table*>(t);
    return code;
}

int ytgpu_join_table_probe_strings(ytgpu_context* h, const ytgpu_join_table* table, const ytgpu_column_view* primary_keys,
                                   uint32_t key_count, const ytgpu_string_column* primary_string_keys, uint32_t string_key_count,
                                   int kind, uint32_t* out_primary_rows, uint32_t* out_foreign_rows, uint64_t capacity,
                                   uint64_t* out_count, int out_mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, join_table_probe_impl(as_context(h), reinterpret_cast<const JoinTable*>(table), primary_keys, key_count,
                                                 primary_string_keys, string_key_count, kind, out_primary_rows, out_foreign_rows, capacity,
                                                 out_count, out_mem));
}

int ytgpu_join_table_destroy(ytgpu_join_table* table, ytgpu_error* err) {
    if (!table) return fill_error(err, Status{});
    JoinTable* t = reinterpret_cast<JoinTable*>(table);
    Context* ctx = t->ctx;
    std::unique_lock<std::mutex> lock(ctx->mu);
    const cudaError_t e = cudaSetDevice(ctx->device);
    delete t;  // stream-ordered frees on the context's stream
    return fill_error(err, e == cudaSuccess ? Status{} : cuda_status(e, "cudaSetDevice"));
}

int ytgpu_gather_column(ytgpu_context* h, const ytgpu_column_view* column, const uint32_t* rows, uint64_t count, uint64_t* out_values,
                        uint8_t* out_null_bitmap, uint64_t* out_null_count, int out_mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, gather_column_impl(as_context(h), column, rows, count, out_values, out_null_bitmap, out_null_count, out_mem));
}

int ytgpu_gather_string_column(ytgpu_context* h, const ytgpu_string_column* column, const uint32_t* rows, uint64_t count,
                               uint64_t* out_starts, uint32_t* out_lengths, uint8_t* out_null_bytemap, int out_mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, gather_string_column_impl(as_context(h), column, rows, count, out_starts, out_lengths, out_null_bytemap,
                                                     out_mem));
}

}  // extern "C"
