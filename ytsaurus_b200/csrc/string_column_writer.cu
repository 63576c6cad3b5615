// string_column_writer.cu — the unversioned string column writer, every segment of a column at once.
//
// Replaces TUnversionedStringColumnWriter<String> (yt/yt/ytlib/table_chunk_format/string_column_writer.cpp): CaptureValue
// :96-150 (first-seen dictionary), AddValues :689-705 (runs; a segment ends at max_values values or > 32 MB of bytes),
// GetSegmentSize :646-676 + DumpSegment :589-636 (the smallest of four layouts, first minimum in enum order), Dump* :152-229,
// :496-586 (parts; offsets as zig-zag differences from i * expected_length, core/misc/bit_packed_unsigned_vector.cpp:11-33).
//
// The reference walks the values on one core with a hash map string -> id.  Here:
//   0. lengths -> prefix sums; a single thread cuts the segments (binary searches over the prefix sums);
//   1. insert : one thread per row hashes its string and finds / claims the slot of its VALUE in the segment's
//               open-addressing table.  A slot is one 64-bit word (fingerprint, row): the string itself is compared through
//               the row the slot points at, atomicMin lowers the row, so the word converges to the FIRST row holding the
//               value — "first seen" without any order of execution (same scheme as the integer writer);
//   2. flags  : first occurrence / run start per row, three exclusive scans (counts, dictionary bytes, run bytes): a scan
//               value at a first occurrence is its dictionary id, at a run start its run index, the byte scans are the
//               offset vectors; dictionary entries and run starts are scattered to their ranks;
//   3. decide : per segment the four size estimates and the layout; the expected length of the chosen offsets vector; one
//               more pass over the rows finds the largest zig-zag difference (the bit width of the offsets); then part
//               sizes and data offsets (segments are laid out 8-byte aligned);
//   4. pack   : one thread per OUTPUT word of the bit-packed vectors / bitmaps; string bytes are copied by whole warps.
//
// The same insert, over a whole column as one segment, gives ytgpu_string_value_ids and the string dictionary of
// string_dict.cuh, which keeps its table and looks other strings up in it with the same hash and slot words.
#include <algorithm>
#include <vector>

#include "context.cuh"
#include "scan.cuh"
#include "string_dict.cuh"
#include "strings.cuh"

using namespace ytgpu;

namespace {

constexpr u32 kNone = 0xffffffffu;
constexpr u64 kEmptySlot = ~0ull;
constexpr u64 kRowsPerBlock = 2048;

__device__ __forceinline__ u32 width_of(u64 v) { return v == 0 ? 0u : 64u - (u32)__clzll((long long)v); }
__device__ __forceinline__ u64 packed_bytes(u64 max_value, u64 count) { return 8ull * (1ull + (((u64)width_of(max_value) * count + 63ull) >> 6)); }
__device__ __forceinline__ u32 zigzag32(i32 v) { return ((u32)v << 1) ^ (u32)(v >> 31); }
__device__ __forceinline__ u64 mix64(u64 x) {
    x ^= x >> 33;
    x *= 0xff51afd7ed558ccdull;
    x ^= x >> 33;
    return x;
}

struct Input {
    const u8* heap;
    const u64* starts;
    const u32* lengths;
    const u8* nulls;
    u64 n;
};

// A column staged by stage_strings, as the kernels here take it.
Input input_of(const StagedStrings& s, u64 n) { return Input{s.dev.heap, s.dev.starts, s.dev.lengths, s.dev.nulls, n}; }

__device__ __forceinline__ bool is_null(const Input& in, u64 g) { return in.nulls && in.nulls[g]; }

// 0a. non-null lengths (the sentinel at n makes scan[n] the grand total)
__global__ void __launch_bounds__(256) lengths_kernel(const Input in, u64* __restrict__ out) {
    for (u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x; g <= in.n; g += (u64)gridDim.x * blockDim.x)
        out[g] = (g < in.n && !is_null(in, g)) ? in.lengths[g] : 0;
}

// 0b. AddValues' segment rule, one thread: a segment ends after max_values values or with the value that lifts its
// bytes above max_buffer (string_column_writer.cpp:701-703).
__global__ void cut_kernel(const u64* __restrict__ P, u64 n, u32 max_values, u64 max_buffer, u64* __restrict__ seg_start, u32 capacity,
                           u32* __restrict__ nseg_out) {
    u64 s = 0;
    u32 k = 0;
    while (s < n && k < capacity) {
        seg_start[k++] = s;
        const u64 limit = P[s] + max_buffer;
        u64 lo = s + 1, hi = n + 1;  // smallest t in [s+1, n+1) with P[t] > limit, else n+1
        while (lo < hi) {
            const u64 mid = (lo + hi) >> 1;
            if (P[mid] > limit) hi = mid;
            else lo = mid + 1;
        }
        s = min(min(s + (u64)max_values, lo), n);
    }
    seg_start[k] = n;
    *nseg_out = s < n ? kNone : k;  // kNone: the capacity bound was wrong (cannot happen)
}

__global__ void __launch_bounds__(256) segment_of_row_kernel(const u64* __restrict__ seg_start, u32 nseg, u64 n, u32* __restrict__ seg_of_row) {
    for (u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x; g < n; g += (u64)gridDim.x * blockDim.x) {
        u32 lo = 0, hi = nseg;
        while (hi - lo > 1) {
            const u32 mid = (lo + hi) >> 1;
            if (seg_start[mid] <= g) lo = mid;
            else hi = mid;
        }
        seg_of_row[g] = lo;
    }
}

__device__ __forceinline__ bool same_bytes(const u8* pa, const u8* pb, u32 len) {
    for (u32 i = 0; i < len; ++i)
        if (pa[i] != pb[i]) return false;
    return true;
}

__device__ __forceinline__ bool same_string(const Input& in, u64 a, u64 b) {
    const u32 len = in.lengths[a];
    if (in.lengths[b] != len) return false;
    return same_bytes(in.heap + in.starts[a], in.heap + in.starts[b], len);
}

// The hash of a value's bytes: FNV-1a seeded with the length, then mix64.  Its top 32 bits are the value's fingerprint, its
// low bits under a table's mask the value's first slot.  The insert and the dictionary lookup both hash through here.
__device__ __forceinline__ u64 string_hash(const u8* p, u32 len) {
    u64 hsh = 0xcbf29ce484222325ull ^ len;
    for (u32 k = 0; k < len; ++k) hsh = (hsh ^ p[k]) * 0x100000001b3ull;
    return mix64(hsh);
}

// A slot word: the fingerprint, and the row (inside its segment) of the value the slot holds.
__device__ __forceinline__ u64 slot_word(u32 fp, u32 row) { return ((u64)fp << 32) | (u64)row; }

// Every segment has its own table: a power of two >= 2 x the segment's rows, at least 8 slots.  table_at[s] <- its slot
// count, and table_at[nseg] <- 0 so that the exclusive scan turns table_at into the first slots plus the total.  Sizing by
// the segment's own rows keeps a column cut into many short segments by the buffer rule as small as its rows.
__global__ void __launch_bounds__(256) table_sizes_kernel(const u64* __restrict__ seg_start, u32 nseg, u64* __restrict__ table_at) {
    for (u32 s = blockIdx.x * blockDim.x + threadIdx.x; s <= nseg; s += gridDim.x * blockDim.x) {
        u64 cap = 0;
        if (s < nseg) {
            const u64 rows = seg_start[s + 1] - seg_start[s];
            cap = 8;
            while (cap < 2 * rows) cap <<= 1;
        }
        table_at[s] = cap;
    }
}

// 1. insert: slot word = (fingerprint << 32) | row index inside the segment.
__global__ void __launch_bounds__(256) insert_kernel(const Input in, const u64* __restrict__ seg_start, const u32* __restrict__ seg_of_row,
                                                     u64* table, const u64* __restrict__ table_at, u32* __restrict__ slot_of_row,
                                                     u32* __restrict__ max_len) {
    const u64 lo = (u64)blockIdx.x * kRowsPerBlock, hi = min(in.n, lo + kRowsPerBlock);
    for (u64 g = lo + threadIdx.x; g < hi; g += blockDim.x) {
        u32 found = kNone;
        if (!is_null(in, g)) {
            const u32 s = seg_of_row[g];
            const u64 begin = seg_start[s];
            const u32 i = (u32)(g - begin);
            const u32 len = in.lengths[g];
            const u64 mx = string_hash(in.heap + in.starts[g], len);
            const u32 fp = (u32)(mx >> 32);
            const u64 want = slot_word(fp, i);
            u64* slots = table + table_at[s];
            const u32 mask = (u32)(table_at[s + 1] - table_at[s]) - 1;
            u32 h = (u32)mx & mask;
            for (;;) {
                u64 cur = *reinterpret_cast<volatile u64*>(slots + h);
                if (cur == kEmptySlot) {
                    cur = atomicCAS((unsigned long long*)&slots[h], (unsigned long long)kEmptySlot, (unsigned long long)want);
                    if (cur == kEmptySlot) break;
                }
                if ((u32)(cur >> 32) == fp && same_string(in, g, begin + (u32)cur)) {
                    if (i < (u32)cur) atomicMin((unsigned long long*)&slots[h], (unsigned long long)want);
                    break;
                }
                h = (h + 1) & mask;
            }
            found = h;
            if (len > __ldcg(&max_len[s])) atomicMax(&max_len[s], len);
        }
        slot_of_row[g] = found;
    }
}

// 2. flags.  counts: low 32 bits = first occurrence, high 32 = run start.
__global__ void __launch_bounds__(256) flags_kernel(const Input in, const u64* __restrict__ seg_start, const u32* __restrict__ seg_of_row,
                                                    const u64* __restrict__ table, const u64* __restrict__ table_at,
                                                    const u32* __restrict__ slot_of_row,
                                                    u32* __restrict__ first_of, u64* __restrict__ counts, u64* __restrict__ dict_bytes,
                                                    u64* __restrict__ run_bytes) {
    const u64 lo = (u64)blockIdx.x * kRowsPerBlock, hi = min(in.n + 1, lo + kRowsPerBlock);
    for (u64 g = lo + threadIdx.x; g < hi; g += blockDim.x) {
        if (g == in.n) {
            counts[g] = dict_bytes[g] = run_bytes[g] = 0;
            break;
        }
        const u32 s = seg_of_row[g];
        const u64 begin = seg_start[s];
        const u32 i = (u32)(g - begin);
        const bool nl = is_null(in, g);
        const u32 slot = slot_of_row[g];
        bool run_start = i == 0;
        if (!run_start) {
            const bool pnl = is_null(in, g - 1);
            run_start = pnl != nl || (!nl && slot_of_row[g - 1] != slot);
        }
        u32 f = kNone;
        if (!nl) f = (u32)table[table_at[s] + slot];  // the slot's row converged to the first row of the value
        first_of[g] = f;
        const u64 len = nl ? 0 : in.lengths[g];
        counts[g] = ((u64)run_start << 32) | (u64)(f == i);
        dict_bytes[g] = f == i ? len : 0;
        run_bytes[g] = run_start ? len : 0;
    }
}

// dictionary entries and run starts to their (column-wide) ranks
__global__ void __launch_bounds__(256) scatter_kernel(u64 n, const u64* __restrict__ counts, u32* __restrict__ dict_row, u32* __restrict__ run_row) {
    for (u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x; g < n; g += (u64)gridDim.x * blockDim.x) {
        const u64 here = counts[g], next = counts[g + 1];
        if ((u32)next != (u32)here) dict_row[(u32)here] = (u32)g;
        if ((next >> 32) != (here >> 32)) run_row[(u32)(here >> 32)] = (u32)g;
    }
}

struct SegWork {
    u64 begin, count;
    u64 dsize, runs;
    u64 direct_bytes, dict_bytes, rle_bytes;
    u32 type, expected, max_diff, max_len;
    u64 struct_words;      // 8-byte words of the parts before the string data
    u64 word_prefix;       // structured words of the earlier segments
    u64 data_offset;
};

struct Scans {
    const u64* P;       // non-null bytes
    const u64* counts;  // first occurrences | run starts << 32
    const u64* D;       // dictionary bytes
    const u64* Q;       // run bytes
};

// 3a. sizes, layout, expected length
__global__ void __launch_bounds__(256) decide_kernel(const u64* __restrict__ seg_start, u32 nseg, const Scans S, const u32* __restrict__ max_len,
                                                     SegWork* __restrict__ work) {
    for (u32 s = blockIdx.x * blockDim.x + threadIdx.x; s < nseg; s += gridDim.x * blockDim.x) {
        SegWork w{};
        w.begin = seg_start[s];
        const u64 end = seg_start[s + 1];
        w.count = end - w.begin;
        const u64 a = S.counts[w.begin], b = S.counts[end];
        w.dsize = (u32)b - (u32)a;
        w.runs = (u32)(b >> 32) - (u32)(a >> 32);
        w.direct_bytes = S.P[end] - S.P[w.begin];
        w.dict_bytes = S.D[end] - S.D[w.begin];
        w.rle_bytes = S.Q[end] - S.Q[w.begin];
        w.max_len = max_len[s];
        const i32 sizes[4] = {
            (i32)(w.dict_bytes + packed_bytes(w.max_len, w.dsize) + packed_bytes(w.dsize + 1, w.runs) + packed_bytes(w.count, w.runs)),
            (i32)(w.dict_bytes + packed_bytes(w.max_len, w.dsize) + packed_bytes(w.dsize + 1, w.count)),
            (i32)(w.rle_bytes + packed_bytes(w.max_len, w.runs) + packed_bytes(w.count, w.runs) + w.count / 8),
            (i32)(w.direct_bytes + packed_bytes(w.max_len, w.count) + w.count / 8),
        };
        u32 type = 0;
        for (u32 t = 1; t < 4; ++t)
            if (sizes[t] < sizes[type]) type = t;
        w.type = type;
        const u64 total = type == 3 ? w.direct_bytes : (type == 2 ? w.rle_bytes : w.dict_bytes);
        const u64 elems = type == 3 ? w.count : (type == 2 ? w.runs : w.dsize);
        w.expected = 0;
        if (elems) {  // DivRound<int>
            const int num = (int)(u32)total, den = (int)elems;
            w.expected = (u32)(num / den + ((num % den) >= (den + 1) / 2 ? 1 : 0));
        }
        w.max_diff = 0;
        work[s] = w;
    }
}

// element k of the offsets vector of a segment: end offset minus (k + 1) * expected, zig-zag encoded
__device__ __forceinline__ u32 offset_diff(u64 end_offset, u32 expected, u64 k) {
    return zigzag32((i32)((u32)end_offset - (u32)((u64)expected * (k + 1))));
}

// 3b. the largest difference of the chosen offsets vector
__global__ void __launch_bounds__(256) max_diff_kernel(u64 n, const u32* __restrict__ seg_of_row, const Scans S, SegWork* work) {
    for (u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x; g < n; g += (u64)gridDim.x * blockDim.x) {
        const u32 s = seg_of_row[g];
        const SegWork& w = work[s];
        const u64 here = S.counts[g], next = S.counts[g + 1], base = S.counts[w.begin];
        u32 z = 0;
        bool has = false;
        if (w.type == 3) {
            z = offset_diff(S.P[g + 1] - S.P[w.begin], w.expected, g - w.begin);
            has = true;
        } else if (w.type == 2) {
            if ((next >> 32) != (here >> 32)) {
                z = offset_diff(S.Q[g + 1] - S.Q[w.begin], w.expected, (u32)(here >> 32) - (u32)(base >> 32));
                has = true;
            }
        } else if ((u32)next != (u32)here) {
            z = offset_diff(S.D[g + 1] - S.D[w.begin], w.expected, (u32)here - (u32)base);
            has = true;
        }
        if (has && z > __ldcg(&work[s].max_diff)) atomicMax(&work[s].max_diff, z);
    }
}

// 3c. widths, part sizes, offsets
__global__ void __launch_bounds__(256) layout_kernel(u32 nseg, u64 chunk_row_offset, const u32* __restrict__ run_row, const Scans S,
                                                     SegWork* __restrict__ work, ytgpu_string_segment* __restrict__ segs, u64* __restrict__ totals) {
    for (u32 s = threadIdx.x; s < nseg; s += blockDim.x) {
        SegWork& w = work[s];
        ytgpu_string_segment d{};
        d.type = w.type;
        d.row_count = (u32)w.count;
        d.chunk_row_count = chunk_row_offset + w.begin + w.count;
        d.direct = w.type >= 2;
        d.expected_length = w.expected;
        d.offsets_width = (u8)width_of(w.max_diff);
        const u64 last_run = run_row[(u32)(S.counts[w.begin] >> 32) + (u32)w.runs - 1] - w.begin;
        int strings_part;
        if (w.type == 3) {
            d.offsets_size = (u32)w.count;
            d.part_bytes[0] = packed_bytes(w.max_diff, w.count);
            d.part_bytes[1] = 8 * ((w.count + 63) / 64);
            d.part_bytes[2] = w.direct_bytes;
            strings_part = 2;
        } else if (w.type == 1) {
            d.ids_size = (u32)w.count;
            d.ids_width = (u8)width_of(w.dsize + 1);
            d.offsets_size = (u32)w.dsize;
            d.part_bytes[0] = packed_bytes(w.dsize + 1, w.count);
            d.part_bytes[1] = packed_bytes(w.max_diff, w.dsize);
            d.part_bytes[2] = w.dict_bytes;
            strings_part = 2;
        } else if (w.type == 2) {
            d.row_indexes_size = (u32)w.runs;
            d.row_indexes_width = (u8)width_of(last_run);
            d.offsets_size = (u32)w.runs;
            d.part_bytes[0] = packed_bytes(last_run, w.runs);
            d.part_bytes[1] = packed_bytes(w.max_diff, w.runs);
            d.part_bytes[2] = 8 * ((w.runs + 63) / 64);
            d.part_bytes[3] = w.rle_bytes;
            strings_part = 3;
        } else {
            d.row_indexes_size = (u32)w.runs;
            d.row_indexes_width = (u8)width_of(last_run);
            d.ids_size = (u32)w.runs;
            d.ids_width = (u8)width_of(w.dsize);
            d.offsets_size = (u32)w.dsize;
            d.part_bytes[0] = packed_bytes(last_run, w.runs);
            d.part_bytes[1] = packed_bytes(w.dsize, w.runs);
            d.part_bytes[2] = packed_bytes(w.max_diff, w.dsize);
            d.part_bytes[3] = w.dict_bytes;
            strings_part = 3;
        }
        u64 structured = 0;
        for (int p = 0; p < strings_part; ++p) structured += d.part_bytes[p];
        w.struct_words = structured / 8;
        d.data_bytes = structured + d.part_bytes[strings_part];
        segs[s] = d;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        u64 at = 0, words = 0;
        for (u32 s = 0; s < nseg; ++s) {
            at = (at + 7) & ~7ull;
            segs[s].data_offset = at;
            work[s].data_offset = at;
            work[s].word_prefix = words;
            words += work[s].struct_words;
            at += segs[s].data_bytes;
        }
        totals[0] = at;
        totals[1] = words;
    }
}

struct PackArgs {
    Input in;
    Scans S;
    const u32* first_of;
    const u32* dict_row;
    const u32* run_row;
    const SegWork* work;
    const ytgpu_string_segment* segs;
    u32 nseg;
    u64 total_words;
};

enum PartKind { PK_DENSE_OFFSETS, PK_DENSE_NULLS, PK_DENSE_IDS, PK_DICT_OFFSETS, PK_ROW_INDEXES, PK_RLE_OFFSETS, PK_RLE_NULLS, PK_RLE_IDS };

__device__ __forceinline__ u64 dictionary_id(const PackArgs& a, const SegWork& w, u64 g) {  // 0 = NULL, else 1-based first-seen id
    const u32 f = a.first_of[g];
    if (f == kNone) return 0;
    return (u64)((u32)a.S.counts[w.begin + f] - (u32)a.S.counts[w.begin]) + 1;
}

__device__ __forceinline__ u64 part_elem(const PackArgs& a, const SegWork& w, int kind, u64 j) {
    switch (kind) {
        case PK_DENSE_OFFSETS: return offset_diff(a.S.P[w.begin + j + 1] - a.S.P[w.begin], w.expected, j);
        case PK_DENSE_NULLS: return is_null(a.in, w.begin + j) ? 1 : 0;
        case PK_DENSE_IDS: return dictionary_id(a, w, w.begin + j);
        case PK_DICT_OFFSETS: {
            const u64 g = a.dict_row[(u32)a.S.counts[w.begin] + (u32)j];
            return offset_diff(a.S.D[g + 1] - a.S.D[w.begin], w.expected, j);
        }
        default: {
            const u64 g = a.run_row[(u32)(a.S.counts[w.begin] >> 32) + (u32)j];
            if (kind == PK_ROW_INDEXES) return g - w.begin;
            if (kind == PK_RLE_OFFSETS) return offset_diff(a.S.Q[g + 1] - a.S.Q[w.begin], w.expected, j);
            if (kind == PK_RLE_NULLS) return is_null(a.in, g) ? 1 : 0;
            return dictionary_id(a, w, g);  // PK_RLE_IDS
        }
    }
}

// 4a. one thread per structured output word
__global__ void __launch_bounds__(256) pack_words_kernel(const PackArgs a, u8* __restrict__ out) {
    for (u64 gw = (u64)blockIdx.x * blockDim.x + threadIdx.x; gw < a.total_words; gw += (u64)gridDim.x * blockDim.x) {
        u32 lo = 0, hi = a.nseg;  // last segment with word_prefix <= gw that owns words
        while (hi - lo > 1) {
            const u32 mid = (lo + hi) >> 1;
            if (a.work[mid].word_prefix <= gw) lo = mid;
            else hi = mid;
        }
        const u32 s = lo;
        const SegWork& w = a.work[s];
        const ytgpu_string_segment& d = a.segs[s];
        u64 lw = gw - w.word_prefix;
        const u64 out_word = w.data_offset / 8 + lw;
        int p = 0;
        while (lw >= d.part_bytes[p] / 8) {
            lw -= d.part_bytes[p] / 8;
            ++p;
        }
        int kind;
        u64 count;
        u32 width;
        bool bitmap = false;
        if (d.type == 3) {
            kind = p == 0 ? PK_DENSE_OFFSETS : PK_DENSE_NULLS;
            count = d.row_count;
            width = d.offsets_width;
            bitmap = p == 1;
        } else if (d.type == 1) {
            kind = p == 0 ? PK_DENSE_IDS : PK_DICT_OFFSETS;
            count = p == 0 ? d.ids_size : d.offsets_size;
            width = p == 0 ? d.ids_width : d.offsets_width;
        } else if (d.type == 2) {
            kind = p == 0 ? PK_ROW_INDEXES : (p == 1 ? PK_RLE_OFFSETS : PK_RLE_NULLS);
            count = d.row_indexes_size;
            width = p == 0 ? d.row_indexes_width : d.offsets_width;
            bitmap = p == 2;
        } else {
            kind = p == 0 ? PK_ROW_INDEXES : (p == 1 ? PK_RLE_IDS : PK_DICT_OFFSETS);
            count = p == 2 ? d.offsets_size : d.row_indexes_size;
            width = p == 0 ? d.row_indexes_width : (p == 1 ? d.ids_width : d.offsets_width);
        }
        u64 word = 0;
        if (bitmap) {
            const u64 j0 = lw * 64, j1 = min(count, j0 + 64);
            for (u64 j = j0; j < j1; ++j) word |= part_elem(a, w, kind, j) << (j - j0);
        } else if (lw == 0) {
            word = count | ((u64)width << 56);
        } else {
            const u64 bit0 = (lw - 1) * 64;  // payload bits [bit0, bit0 + 64); width > 0 here (a zero-width vector is its header)
            for (u64 j = bit0 / width; j < count && j * width < bit0 + 64; ++j) {
                const u64 v = part_elem(a, w, kind, j);
                const i64 pos = (i64)(j * width) - (i64)bit0;
                word |= pos >= 0 ? (v << pos) : (v >> (-pos));
            }
        }
        reinterpret_cast<u64*>(out)[out_word] = word;
    }
}

// 4b. string bytes: every warp takes 32 rows; the rows that contribute a string (all non-null rows / first occurrences /
// non-null run starts, by layout) are copied one after the other by the whole warp.
__global__ void __launch_bounds__(256) copy_strings_kernel(const PackArgs a, const u32* __restrict__ seg_of_row, u8* __restrict__ out) {
    const u32 lane = threadIdx.x & 31;
    const u64 warps = ((u64)gridDim.x * blockDim.x) >> 5;
    for (u64 base = ((u64)blockIdx.x * blockDim.x + threadIdx.x - lane); base < a.in.n; base += warps * 32) {
        const u64 g = base + lane;
        u64 dst = 0;
        bool item = false;
        if (g < a.in.n && !is_null(a.in, g)) {
            const u32 s = seg_of_row[g];
            const SegWork& w = a.work[s];
            const u64 here = a.S.counts[g], next = a.S.counts[g + 1];
            const u64 strings_at = w.data_offset + w.struct_words * 8;
            if (w.type == 3) {
                item = true;
                dst = strings_at + (a.S.P[g] - a.S.P[w.begin]);
            } else if (w.type == 2) {
                item = (next >> 32) != (here >> 32);
                dst = strings_at + (a.S.Q[g] - a.S.Q[w.begin]);
            } else {
                item = (u32)next != (u32)here;
                dst = strings_at + (a.S.D[g] - a.S.D[w.begin]);
            }
        }
        u32 m = __ballot_sync(0xffffffffu, item);
        while (m) {
            const int src_lane = __ffs(m) - 1;
            m &= m - 1;
            const u64 row = base + src_lane;
            const u64 to = __shfl_sync(0xffffffffu, dst, src_lane);
            const u32 len = a.in.lengths[row];
            const u8* from = a.in.heap + a.in.starts[row];
            for (u32 k = lane; k < len; k += 32) out[to + k] = from[k];
        }
    }
}

inline u32 grid_for(u64 items, int threads, int per_sm) {
    return (u32)std::max<u64>(1, std::min<u64>((items + threads - 1) / threads, (u64)kNumSms * per_sm));
}

Status encode_string_impl(Context* ctx, const u8* heap, u64 heap_bytes, const u64* starts, const u32* lengths, const u8* null_bytemap, u64 n,
                          u32 max_values, u64 max_buffer, u64 chunk_row_offset, int mem, u8* out_data, u64 out_capacity, u64* out_bytes,
                          ytgpu_string_segment* out_segments, u32 seg_capacity, u32* out_seg_count) {
    if (!out_bytes || !out_seg_count) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    *out_bytes = 0;
    *out_seg_count = 0;
    if (max_values == 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "max_segment_value_count must be positive");
    if (max_buffer == 0) max_buffer = 32ull << 20;  // MaxBufferSize, string_column_writer.cpp:25
    if (max_buffer >= (1ull << 31)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "max_buffer_bytes must be below 2^31 (offsets are 32-bit)");
    if (n == 0) return Status{};
    if (!starts || !lengths || (heap_bytes && !heap)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null input");
    if (n >= (1ull << 32)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "one call encodes fewer than 2^32 rows");
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));

    StagedStrings staged;
    YTGPU_TRY(stage_strings(ctx, ytgpu_string_column{heap, heap_bytes, starts, lengths, null_bytemap, n, mem, 0}, &staged));
    const Input in = input_of(staged, n);

    // 0. prefix sums of the non-null lengths, segment cuts
    DevBuf<u64> P, sums, totals, seg_start;
    DevBuf<u32> nseg_dev;
    YTGPU_TRY(P.allocate(ctx, n + 1));
    YTGPU_TRY(sums.allocate(ctx, scan_block_count(n + 1)));
    YTGPU_TRY(totals.allocate(ctx, 4));
    YTGPU_TRY(nseg_dev.allocate(ctx, 1));
    u64 total_string_bytes = 0;
    {
        KernelTimer t(ctx, KC_DECODE, 4);
        lengths_kernel<<<grid_for(n + 1, 256, 8), 256, 0, ctx->stream>>>(in, P.p);
        exclusive_scan_u64(ctx->stream, P.p, n + 1, sums.p, totals.p);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_CUDA_TRY(cudaMemcpyAsync(&total_string_bytes, totals.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (mem == YTGPU_MEM_HOST && total_string_bytes > heap_bytes)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "string lengths add up to more than the heap holds");
    const u64 cut_capacity64 = (n + max_values - 1) / max_values + total_string_bytes / (max_buffer + 1) + 2;
    if (cut_capacity64 > (1u << 24)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "too many segments (%llu)", (unsigned long long)cut_capacity64);
    const u32 cut_capacity = (u32)cut_capacity64;
    YTGPU_TRY(seg_start.allocate(ctx, cut_capacity + 1));
    cut_kernel<<<1, 1, 0, ctx->stream>>>(P.p, n, max_values, max_buffer, seg_start.p, cut_capacity, nseg_dev.p);
    ctx->count_launch();
    u32 nseg = 0;
    YTGPU_CUDA_TRY(cudaMemcpyAsync(&nseg, nseg_dev.p, 4, cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (nseg == kNone || nseg == 0) return make_status(YTGPU_ERR_CUDA, "segment cut failed");
    *out_seg_count = nseg;

    // 1.-3.
    DevBuf<u64> table_at;
    YTGPU_TRY(table_at.allocate(ctx, (u64)nseg + 1));
    {
        KernelTimer t(ctx, KC_DECODE, 4);
        table_sizes_kernel<<<grid_for((u64)nseg + 1, 256, 4), 256, 0, ctx->stream>>>(seg_start.p, nseg, table_at.p);
        exclusive_scan_u64(ctx->stream, table_at.p, (u64)nseg + 1, sums.p, totals.p + 1);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    u64 table_slots = 0;
    YTGPU_CUDA_TRY(cudaMemcpyAsync(&table_slots, totals.p + 1, 8, cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    DevBuf<u32> seg_of_row, slot_of_row, first_of, dict_row, run_row, max_len;
    DevBuf<u64> table, counts, D, Q;
    DevBuf<SegWork> work;
    DevBuf<ytgpu_string_segment> segs;
    YTGPU_TRY(seg_of_row.allocate(ctx, n));
    YTGPU_TRY(slot_of_row.allocate(ctx, n));
    YTGPU_TRY(first_of.allocate(ctx, n));
    YTGPU_TRY(dict_row.allocate(ctx, n));
    YTGPU_TRY(run_row.allocate(ctx, n));
    YTGPU_TRY(max_len.allocate(ctx, nseg));
    YTGPU_TRY(table.allocate(ctx, table_slots));
    YTGPU_TRY(counts.allocate(ctx, n + 1));
    YTGPU_TRY(D.allocate(ctx, n + 1));
    YTGPU_TRY(Q.allocate(ctx, n + 1));
    YTGPU_TRY(work.allocate(ctx, nseg));
    YTGPU_TRY(segs.allocate(ctx, nseg));
    YTGPU_CUDA_TRY(cudaMemsetAsync(table.p, 0xff, table_slots * 8, ctx->stream));
    YTGPU_CUDA_TRY(cudaMemsetAsync(max_len.p, 0, (u64)nseg * 4, ctx->stream));
    const Scans S{P.p, counts.p, D.p, Q.p};
    {
        KernelTimer t(ctx, KC_DECODE, 17);
        const u32 row_blocks = (u32)((n + kRowsPerBlock - 1) / kRowsPerBlock);
        segment_of_row_kernel<<<grid_for(n, 256, 8), 256, 0, ctx->stream>>>(seg_start.p, nseg, n, seg_of_row.p);
        insert_kernel<<<row_blocks, 256, 0, ctx->stream>>>(in, seg_start.p, seg_of_row.p, table.p, table_at.p, slot_of_row.p, max_len.p);
        flags_kernel<<<(u32)((n + kRowsPerBlock) / kRowsPerBlock), 256, 0, ctx->stream>>>(in, seg_start.p, seg_of_row.p, table.p, table_at.p,
                                                                                         slot_of_row.p, first_of.p, counts.p, D.p, Q.p);
        exclusive_scan_u64(ctx->stream, counts.p, n + 1, sums.p, totals.p + 1);
        exclusive_scan_u64(ctx->stream, D.p, n + 1, sums.p, totals.p + 1);
        exclusive_scan_u64(ctx->stream, Q.p, n + 1, sums.p, totals.p + 1);
        scatter_kernel<<<grid_for(n, 256, 8), 256, 0, ctx->stream>>>(n, counts.p, dict_row.p, run_row.p);
        decide_kernel<<<grid_for(nseg, 256, 4), 256, 0, ctx->stream>>>(seg_start.p, nseg, S, max_len.p, work.p);
        max_diff_kernel<<<grid_for(n, 256, 8), 256, 0, ctx->stream>>>(n, seg_of_row.p, S, work.p);
        layout_kernel<<<1, 256, 0, ctx->stream>>>(nseg, chunk_row_offset, run_row.p, S, work.p, segs.p, totals.p + 2);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    u64 layout[2] = {0, 0};  // bytes, structured words
    YTGPU_CUDA_TRY(cudaMemcpyAsync(layout, totals.p + 2, 16, cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    const u64 bytes = layout[0];
    *out_bytes = bytes;
    if (!out_segments || nseg > seg_capacity)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "column needs %u segment descriptors, capacity is %u", nseg, seg_capacity);
    if (!out_data || bytes > out_capacity)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "column data needs %llu bytes, capacity is %llu", (unsigned long long)bytes,
                           (unsigned long long)out_capacity);
    YTGPU_CUDA_TRY(cudaMemcpyAsync(out_segments, segs.p, (size_t)nseg * sizeof(ytgpu_string_segment), cudaMemcpyDeviceToHost, ctx->stream));

    // 4.
    if (mem != YTGPU_MEM_HOST && (reinterpret_cast<uintptr_t>(out_data) & 7))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "out_data must be 8-byte aligned");
    OutBuf<u8> dst;
    YTGPU_TRY(dst.prepare(ctx, out_data, bytes + 8, mem));
    YTGPU_CUDA_TRY(cudaMemsetAsync(dst.p, 0, bytes, ctx->stream));  // the alignment gaps between segments
    PackArgs args{in, S, first_of.p, dict_row.p, run_row.p, work.p, segs.p, nseg, layout[1]};
    {
        KernelTimer t(ctx, KC_DECODE, 2);
        pack_words_kernel<<<grid_for(layout[1], 256, 8), 256, 0, ctx->stream>>>(args, dst.p);
        copy_strings_kernel<<<grid_for(n, 256, 8), 256, 0, ctx->stream>>>(args, seg_of_row.p, dst.p);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_TRY(dst.download(ctx, bytes));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    return Status{};
}

// ---- string values -> canonical ids (string GROUP BY keys) ----
// id[i] = index of the FIRST row holding the same string as row i (NULL rows: kNone).  The same slot scheme as the writer's
// dictionary, over the whole column as one segment.
__global__ void __launch_bounds__(256) value_ids_kernel(const Input in, const u64* __restrict__ table, u32 cap, const u32* __restrict__ slot_of_row,
                                                        u64* __restrict__ out_ids, u8* __restrict__ out_null) {
    for (u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x; g < in.n; g += (u64)gridDim.x * blockDim.x) {
        const u32 slot = slot_of_row[g];
        out_ids[g] = slot == kNone ? 0 : (u64)(u32)table[slot];
        if (out_null) out_null[g] = slot == kNone ? 1 : 0;
    }
}

u64 value_table_slots(u64 n) {
    u64 cap = 8;
    while (cap < 2 * n) cap <<= 1;
    return cap;
}

// The insert over the n rows of `in` as one segment, then the ids.  bounds (device, 4 words) = {0, n, 0, cap}: the
// segment's rows, then its table's slots.  table (cap words) is left as the insert leaves it.
Status insert_value_ids(Context* ctx, int timer_class, const Input& in, const u64* bounds, u64* table, u64 cap, u64* out_ids, u8* out_null) {
    const u64 n = in.n;
    DevBuf<u32> seg_of_row, slot_of_row, max_len;
    YTGPU_TRY(seg_of_row.allocate(ctx, n));
    YTGPU_TRY(slot_of_row.allocate(ctx, n));
    YTGPU_TRY(max_len.allocate(ctx, 1));
    YTGPU_CUDA_TRY(cudaMemsetAsync(table, 0xff, cap * 8, ctx->stream));
    YTGPU_CUDA_TRY(cudaMemsetAsync(seg_of_row.p, 0, n * 4, ctx->stream));  // one segment: every row belongs to segment 0
    YTGPU_CUDA_TRY(cudaMemsetAsync(max_len.p, 0, 4, ctx->stream));
    KernelTimer t(ctx, timer_class, 2);
    insert_kernel<<<(u32)((n + kRowsPerBlock - 1) / kRowsPerBlock), 256, 0, ctx->stream>>>(in, bounds, seg_of_row.p, table, bounds + 2,
                                                                                         slot_of_row.p, max_len.p);
    value_ids_kernel<<<grid_for(n, 256, 8), 256, 0, ctx->stream>>>(in, table, (u32)cap, slot_of_row.p, out_ids, out_null);
    YTGPU_CUDA_TRY(cudaGetLastError());
    return Status{};
}

Status string_value_ids_impl(Context* ctx, const u8* heap, u64 heap_bytes, const u64* starts, const u32* lengths, const u8* null_bytemap, u64 n,
                             u64* out_ids, u8* out_null, int mem) {
    if (n == 0) return Status{};
    if (!starts || !lengths || !out_ids || (heap_bytes && !heap)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    if (n > (1ull << 30)) return make_status(YTGPU_ERR_UNSUPPORTED, "at most 2^30 rows per call");
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    StagedStrings staged;
    YTGPU_TRY(stage_strings(ctx, ytgpu_string_column{heap, heap_bytes, starts, lengths, null_bytemap, n, mem, 0}, &staged));
    const u64 cap = value_table_slots(n);
    OutBuf<u64> ids;
    OutBuf<u8> nulls;
    DevBuf<u64> table, seg_start;
    YTGPU_TRY(table.allocate(ctx, cap));
    YTGPU_TRY(seg_start.allocate(ctx, 4));
    const u64 bounds[4] = {0, n, 0, cap};
    YTGPU_CUDA_TRY(cudaMemcpyAsync(seg_start.p, bounds, 32, cudaMemcpyHostToDevice, ctx->stream));
    YTGPU_TRY(ids.prepare(ctx, out_ids, n, mem));
    YTGPU_TRY(nulls.prepare(ctx, out_null, n, mem));
    YTGPU_TRY(insert_value_ids(ctx, KC_GROUPBY, input_of(staged, n), seg_start.p, table.p, cap, ids.p, nulls.p));
    YTGPU_TRY(ids.download(ctx, n));
    YTGPU_TRY(nulls.download(ctx, n));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));  // bounds[] lives on this frame
    return Status{};
}

// ---- the string dictionary (string_dict.cuh) ----
__device__ __forceinline__ bool in_heap(u64 start, u32 len, u64 heap_bytes) { return start <= heap_bytes && len <= heap_bytes - start; }

// Build, step 1: each row's length in the dictionary's heap, at n the 0 that makes the scan's last word the total.  A NULL
// row and a value outside its heap (which sets the error bit) take no bytes.
__global__ void __launch_bounds__(256) dict_lengths_kernel(const Input in, u64 heap_bytes, u64* __restrict__ out, u32* err_word) {
    u32 bad = 0;
    for (u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x; g <= in.n; g += (u64)gridDim.x * blockDim.x) {
        u64 len = 0;
        if (g < in.n && !is_null(in, g)) {
            const u32 l = in.lengths[g];
            if (in_heap(in.starts[g], l, heap_bytes)) len = l;
            else bad = 1;
        }
        out[g] = len;
    }
    if (bad) atomicOr(err_word, (u32)DE_STRING_OUT_OF_HEAP);
}

// Build, step 2, after the scan of step 1 (at[g] = value g's start in the dictionary's heap): each warp takes 32 rows,
// writes their lengths and null bits, and copies their bytes one value after the other with the whole warp.
__global__ void __launch_bounds__(256) dict_copy_kernel(const Input in, const u64* __restrict__ at, u8* __restrict__ heap,
                                                        u32* __restrict__ lengths, u32* __restrict__ null_bits) {
    const u32 lane = threadIdx.x & 31;
    const u64 warps = ((u64)gridDim.x * blockDim.x) >> 5;
    for (u64 base = (u64)blockIdx.x * blockDim.x + threadIdx.x - lane; base < in.n; base += warps * 32) {
        const u64 g = base + lane;
        u32 len = 0;
        if (g < in.n) {
            len = (u32)(at[g + 1] - at[g]);
            lengths[g] = len;
        }
        if (null_bits) {
            const u32 m = __ballot_sync(0xffffffffu, g < in.n && is_null(in, g));
            if (lane == 0) null_bits[base >> 5] = m;
        }
        u32 m = __ballot_sync(0xffffffffu, len != 0);
        while (m) {
            const int src = __ffs(m) - 1;
            m &= m - 1;
            const u64 row = base + src;
            const u32 l = __shfl_sync(0xffffffffu, len, src);
            const u8* from = in.heap + in.starts[row];
            u8* to = heap + at[row];
            for (u32 k = lane; k < l; k += 32) to[k] = from[k];
        }
    }
}

// The lookup: one thread per row hashes its value as the insert does and walks the kept table from the value's first slot,
// comparing the fingerprint, then the length and the bytes, until the value's slot or an empty one (the table is at most
// half full).
__global__ void __launch_bounds__(256) dict_lookup_kernel(const Input dict, const u64* __restrict__ slots, u32 mask, const Input in,
                                                          u64 heap_bytes, u64* __restrict__ ids, u32* __restrict__ null_bits, u32* err_word) {
    const u32 lane = threadIdx.x & 31;
    u32 bad = 0;
    for (u64 base = (u64)blockIdx.x * blockDim.x + threadIdx.x - lane; base < in.n; base += (u64)gridDim.x * blockDim.x) {
        const u64 g = base + lane;
        const bool nul = g < in.n && is_null(in, g);
        if (g < in.n) {
            u64 id = 0;
            if (!nul) {
                id = kStringDictMiss;
                const u64 start = in.starts[g];
                const u32 len = in.lengths[g];
                if (!in_heap(start, len, heap_bytes)) {
                    bad = 1;
                } else {
                    const u8* p = in.heap + start;
                    const u64 mx = string_hash(p, len);
                    const u32 fp = (u32)(mx >> 32);
                    u32 h = (u32)mx & mask;
                    for (;;) {
                        const u64 w = slots[h];
                        if (w == kEmptySlot) break;
                        const u32 row = (u32)w;
                        if ((u32)(w >> 32) == fp && dict.lengths[row] == len && same_bytes(dict.heap + dict.starts[row], p, len)) {
                            id = row;
                            break;
                        }
                        h = (h + 1) & mask;
                    }
                }
            }
            ids[g] = id;
        }
        if (null_bits) {
            const u32 m = __ballot_sync(0xffffffffu, nul);
            if (lane == 0) null_bits[base >> 5] = m;
        }
    }
    if (bad) atomicOr(err_word, (u32)DE_STRING_OUT_OF_HEAP);
}

// Append, step 1: flags[g] = 1 at the first row of each value the dictionary lacks (its lookup missed and the block's
// value-ids insert names the row itself), new_bytes[g] = that value's length; at n, the 0s that make the scans' last words
// the totals.
__global__ void __launch_bounds__(256) dict_new_values_kernel(const Input in, const u64* __restrict__ ids, const u64* __restrict__ first_row,
                                                              u64* __restrict__ flags, u64* __restrict__ new_bytes) {
    for (u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x; g <= in.n; g += (u64)gridDim.x * blockDim.x) {
        const bool fresh = g < in.n && !is_null(in, g) && ids[g] == kStringDictMiss && first_row[g] == g;
        flags[g] = fresh ? 1 : 0;
        new_bytes[g] = fresh ? in.lengths[g] : 0;
    }
}

// Inserts value id's slot word into a dictionary's slots (at most half full, so an empty slot is always found).  The
// values are distinct: no comparison, a CAS on an empty slot only.
__device__ __forceinline__ void dict_insert_slot(u64* slots, u32 mask, const u8* p, u32 len, u32 id) {
    const u64 mx = string_hash(p, len);
    u32 h = (u32)mx & mask;
    const unsigned long long want = slot_word((u32)(mx >> 32), id);
    while (atomicCAS((unsigned long long*)&slots[h], (unsigned long long)kEmptySlot, want) != (unsigned long long)kEmptySlot) h = (h + 1) & mask;
}

// Append, step 2 (rank, at: the scans of step 1): each new value gets id count + rank, its bytes at bytes + at, and its slot.
// Each warp takes 32 rows and copies their new values' bytes one after the other with the whole warp, as dict_copy_kernel.
__global__ void __launch_bounds__(256) dict_append_kernel(const Input in, const u64* __restrict__ rank, const u64* __restrict__ at, u64 count,
                                                          u64 bytes, u8* __restrict__ heap, u64* __restrict__ starts, u32* __restrict__ lengths,
                                                          u64* slots, u32 mask, u64* __restrict__ ids) {
    const u32 lane = threadIdx.x & 31;
    const u64 warps = ((u64)gridDim.x * blockDim.x) >> 5;
    for (u64 base = (u64)blockIdx.x * blockDim.x + threadIdx.x - lane; base < in.n; base += warps * 32) {
        const u64 g = base + lane;
        const bool fresh = g < in.n && rank[g + 1] != rank[g];
        u32 len = 0;
        if (fresh) {
            const u64 id = count + rank[g];
            len = in.lengths[g];
            starts[id] = bytes + at[g];
            lengths[id] = len;
            dict_insert_slot(slots, mask, in.heap + in.starts[g], len, (u32)id);
            ids[g] = id;
        }
        u32 m = __ballot_sync(0xffffffffu, len != 0);
        while (m) {
            const int src = __ffs(m) - 1;
            m &= m - 1;
            const u64 row = base + src;
            const u32 l = __shfl_sync(0xffffffffu, len, src);
            const u8* from = in.heap + in.starts[row];
            u8* to = heap + bytes + at[row];
            for (u32 k = lane; k < l; k += 32) to[k] = from[k];
        }
    }
}

// Append, step 3: the other rows of a new value take the id of its first row (set by step 2).
__global__ void __launch_bounds__(256) dict_map_new_kernel(const Input in, const u64* __restrict__ first_row, u64* ids) {
    for (u64 g = (u64)blockIdx.x * blockDim.x + threadIdx.x; g < in.n; g += (u64)gridDim.x * blockDim.x)
        if (!is_null(in, g) && ids[g] == kStringDictMiss) ids[g] = ids[first_row[g]];
}

// The slots of a grown dictionary, from its kept values.
__global__ void __launch_bounds__(256) dict_rehash_kernel(const u8* __restrict__ heap, const u64* __restrict__ starts, const u32* __restrict__ lengths,
                                                          u64 count, u64* slots, u32 mask) {
    for (u64 id = (u64)blockIdx.x * blockDim.x + threadIdx.x; id < count; id += (u64)gridDim.x * blockDim.x)
        dict_insert_slot(slots, mask, heap + starts[id], lengths[id], (u32)id);
}

}  // namespace

namespace ytgpu {

Status string_dicts_build(Context* ctx, const ytgpu_string_column* cols, u32 count, u64 n, StringDict* dicts, DevBuf<u64>* ids,
                          DevBuf<u32>* null_bits) {
    if (count == 0) return Status{};
    const u64 cap = value_table_slots(n);
    for (u32 c = 0; c < count; ++c) YTGPU_TRY(dicts[c].slots.allocate(ctx, cap));
    if (n == 0) {  // an empty table: every lookup misses
        for (u32 c = 0; c < count; ++c) YTGPU_CUDA_TRY(cudaMemsetAsync(dicts[c].slots.p, 0xff, cap * 8, ctx->stream));
        return Status{};
    }
    std::vector<StagedStrings> staged(count);
    DevBuf<u64> bounds_dev, sums, totals;
    YTGPU_TRY(bounds_dev.allocate(ctx, 4));
    YTGPU_TRY(sums.allocate(ctx, scan_block_count(n + 1)));
    YTGPU_TRY(totals.allocate(ctx, count));
    const u64 bounds[4] = {0, n, 0, cap};  // read before the synchronisation below
    YTGPU_CUDA_TRY(cudaMemcpyAsync(bounds_dev.p, bounds, 32, cudaMemcpyHostToDevice, ctx->stream));
    for (u32 c = 0; c < count; ++c) {
        const ytgpu_string_column& s = cols[c];
        YTGPU_TRY(stage_strings(ctx, s, &staged[c]));  // the key columns hold n rows each
        YTGPU_TRY(dicts[c].starts.allocate(ctx, n + 1));
        KernelTimer t(ctx, KC_JOIN, 4);
        dict_lengths_kernel<<<grid_for(n + 1, 256, 8), 256, 0, ctx->stream>>>(input_of(staged[c], n), s.heap_bytes, dicts[c].starts.p,
                                                                              ctx->dev_err);
        exclusive_scan_u64(ctx->stream, dicts[c].starts.p, n + 1, sums.p, totals.p + c);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    std::vector<u64> bytes(count);
    YTGPU_CUDA_TRY(cudaMemcpyAsync(bytes.data(), totals.p, (size_t)count * 8, cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_TRY(check_device_errors(ctx));  // synchronises: the heap sizes and the bounds checks of every column
    for (u32 c = 0; c < count; ++c) {
        StringDict& d = dicts[c];
        YTGPU_TRY(d.heap.allocate(ctx, bytes[c]));
        YTGPU_TRY(d.lengths.allocate(ctx, n));
        YTGPU_TRY(ids[c].allocate(ctx, n));
        u32* bits = nullptr;
        if (cols[c].null_bytemap) {
            YTGPU_TRY(null_bits[c].allocate(ctx, (n + 31) / 32));
            bits = null_bits[c].p;
        }
        {
            KernelTimer t(ctx, KC_JOIN);
            dict_copy_kernel<<<grid_for(n, 256, 8), 256, 0, ctx->stream>>>(input_of(staged[c], n), d.starts.p, d.heap.p, d.lengths.p, bits);
            YTGPU_CUDA_TRY(cudaGetLastError());
        }
        const Input copy{d.heap.p, d.starts.p, d.lengths.p, staged[c].dev.nulls, n};
        YTGPU_TRY(insert_value_ids(ctx, KC_JOIN, copy, bounds_dev.p, d.slots.p, cap, ids[c].p, nullptr));
    }
    return Status{};
}

Status string_dict_lookup(Context* ctx, const StringDict& dict, const ytgpu_string_column& col, u64 n, u64* ids, u32* null_bits) {
    StagedStrings staged;
    YTGPU_TRY(stage_strings(ctx, col, &staged));  // col holds n rows
    const Input d{dict.heap.p, dict.starts.p, dict.lengths.p, nullptr, 0};
    KernelTimer t(ctx, KC_JOIN);
    dict_lookup_kernel<<<grid_for(n, 256, 16), 256, 0, ctx->stream>>>(d, dict.slots.p, (u32)dict.slots.n - 1, input_of(staged, n), col.heap_bytes, ids,
                                                                      col.null_bytemap ? null_bits : nullptr, ctx->dev_err);
    YTGPU_CUDA_TRY(cudaGetLastError());
    return Status{};
}

Status string_dict_append(Context* ctx, StringDict* dict, u64* count, u64* bytes, const ytgpu_string_column& col, u64 n, u64* ids) {
    if (n == 0) return Status{};
    StagedStrings staged;
    YTGPU_TRY(stage_strings(ctx, col, &staged));
    const Input in = input_of(staged, n);
    // the block's own value ids: the first row of each value
    const u64 cap = value_table_slots(n);
    DevBuf<u64> table, bounds_dev, first_row, rank, at, sums, totals;
    YTGPU_TRY(table.allocate(ctx, cap));
    YTGPU_TRY(bounds_dev.allocate(ctx, 4));
    YTGPU_TRY(first_row.allocate(ctx, n));
    YTGPU_TRY(rank.allocate(ctx, n + 1));
    YTGPU_TRY(at.allocate(ctx, n + 1));
    YTGPU_TRY(sums.allocate(ctx, scan_block_count(n + 1)));
    YTGPU_TRY(totals.allocate(ctx, 2));
    const u64 bounds[4] = {0, n, 0, cap};  // read before the synchronisation below
    YTGPU_CUDA_TRY(cudaMemcpyAsync(bounds_dev.p, bounds, 32, cudaMemcpyHostToDevice, ctx->stream));
    YTGPU_TRY(insert_value_ids(ctx, KC_GROUPBY, in, bounds_dev.p, table.p, cap, first_row.p, nullptr));
    {
        KernelTimer t(ctx, KC_GROUPBY, 7);
        dict_new_values_kernel<<<grid_for(n + 1, 256, 8), 256, 0, ctx->stream>>>(in, ids, first_row.p, rank.p, at.p);
        exclusive_scan_u64(ctx->stream, rank.p, n + 1, sums.p, totals.p);
        exclusive_scan_u64(ctx->stream, at.p, n + 1, sums.p, totals.p + 1);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    u64 added[2] = {0, 0};
    YTGPU_CUDA_TRY(cudaMemcpyAsync(added, totals.p, 16, cudaMemcpyDeviceToHost, ctx->stream));
    YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));
    if (added[0] == 0) return Status{};  // every value was there already: the lookup's ids are final
    const u64 c = *count + added[0], b = *bytes + added[1];
    YTGPU_TRY(grow_buf(ctx, &dict->heap, *bytes, b));
    YTGPU_TRY(grow_buf(ctx, &dict->starts, *count, c));
    YTGPU_TRY(grow_buf(ctx, &dict->lengths, *count, c));
    if (dict->slots.n < 2 * c) {
        u64 slots = dict->slots.n;
        while (slots < 2 * c) slots <<= 1;
        YTGPU_TRY(dict->slots.allocate(ctx, slots));
        YTGPU_CUDA_TRY(cudaMemsetAsync(dict->slots.p, 0xff, slots * 8, ctx->stream));
        if (*count) {
            KernelTimer t(ctx, KC_GROUPBY);
            dict_rehash_kernel<<<grid_for(*count, 256, 8), 256, 0, ctx->stream>>>(dict->heap.p, dict->starts.p, dict->lengths.p, *count, dict->slots.p,
                                                                                (u32)slots - 1);
            YTGPU_CUDA_TRY(cudaGetLastError());
        }
    }
    {
        KernelTimer t(ctx, KC_GROUPBY, 2);
        dict_append_kernel<<<grid_for(n, 256, 8), 256, 0, ctx->stream>>>(in, rank.p, at.p, *count, *bytes, dict->heap.p, dict->starts.p,
                                                                         dict->lengths.p, dict->slots.p, (u32)dict->slots.n - 1, ids);
        dict_map_new_kernel<<<grid_for(n, 256, 8), 256, 0, ctx->stream>>>(in, first_row.p, ids);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    *count = c;
    *bytes = b;
    return Status{};
}

}  // namespace ytgpu

extern "C" {

int ytgpu_string_value_ids(ytgpu_context* h, const uint8_t* string_heap, uint64_t string_heap_bytes, const uint64_t* starts,
                           const uint32_t* lengths, const uint8_t* null_bytemap, uint64_t row_count, uint64_t* out_ids,
                           uint8_t* out_null_bytemap, int mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, string_value_ids_impl(as_context(h), string_heap, string_heap_bytes, starts, lengths, null_bytemap, row_count,
                                                 out_ids, out_null_bytemap, mem));
}

int ytgpu_encode_string_column(ytgpu_context* h, const uint8_t* string_heap, uint64_t string_heap_bytes, const uint64_t* starts,
                               const uint32_t* lengths, const uint8_t* null_bytemap, uint64_t row_count,
                               uint32_t max_segment_value_count, uint64_t max_buffer_bytes, uint64_t chunk_row_offset, int mem,
                               uint8_t* out_data, uint64_t out_capacity, uint64_t* out_data_bytes, ytgpu_string_segment* out_segments,
                               uint32_t segment_capacity, uint32_t* out_segment_count, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, encode_string_impl(as_context(h), string_heap, string_heap_bytes, starts, lengths, null_bytemap, row_count,
                                              max_segment_value_count, max_buffer_bytes, chunk_row_offset, mem, out_data, out_capacity,
                                              out_data_bytes, out_segments, segment_capacity, out_segment_count));
}

}  // extern "C"
