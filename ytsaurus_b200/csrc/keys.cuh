// keys.cuh — order-preserving key normalisation (host + device).
//
// A composite key (the first TComparator::GetLength() values of a row) becomes a fixed-width byte
// string whose unsigned lexicographic order equals TComparator::CompareKeys
// (yt/yt/client/table_client/comparator.cpp:174-200) built on CompareRowValues
// (unversioned_row.cpp:392-464):
//   per column:  [type byte]  payload
//     type byte  = EValueType code (row_base.h:11-28) — type order first, unversioned_row.cpp:440-442;
//                  omitted for `required` columns whose type is fixed by the schema
//     Int64      = value ^ 0x8000..., big-endian          Uint64 = big-endian
//     Double     = -0 -> +0, any NaN -> one quiet NaN pattern above +inf (compare-inl.h:49-66),
//                  then the usual sign transform, big-endian
//     Boolean    = 1 byte                                 Null / Min / Max / Bottom = zero payload
//     String     = bytes zero-padded to the column width W, followed by the length (big-endian),
//                  so that "ab" < "ab\0" (string_view::compare, compare-inl.h:32-41)
//   descending column: all of the column's bytes inverted (comparator.cpp:56-58)
// The byte string is cut into big-endian u64 chunks (chunk 0 most significant) for the radix sort.
#pragma once

#include "common.cuh"
#include "radix_sort.cuh"

namespace ytgpu {

constexpr int kMaxKeyColumns = 32;

struct KeyColLayout {
    u32 index;          // rowset: value position; fixed rows: byte offset
    u32 width;          // string width W
    u32 payload_bytes;  // bytes after the optional type byte
    u32 len_bytes;      // length-field bytes for strings (0 for fixed rows)
    u32 byte_offset;    // offset of this column inside the normalised key
    u8 type;            // declared type, 0 = any scalar
    u8 descending;
    u8 has_type_byte;
    u8 pad;
};

struct KeyLayout {
    KeyColLayout col[kMaxKeyColumns];
    u32 ncols;
    u32 total_bytes;
    u32 nchunks;
    u32 fixed_rows;  // 1: columns address bytes of a fixed-width row
};

inline u32 string_len_bytes(u32 w) { return w < 255 ? 1 : (w < 65535 ? 2 : 4); }

// Builds the layout; string widths must be final (non-zero unless the column cannot hold strings).
inline Status build_key_layout(const ytgpu_sort_spec* spec, bool fixed_rows, bool force_type_byte, KeyLayout* L) {
    if (!spec || spec->column_count == 0 || spec->column_count > (u32)kMaxKeyColumns)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key column count must be in [1, %d]", kMaxKeyColumns);
    L->ncols = spec->column_count;
    L->fixed_rows = fixed_rows;
    L->nchunks = 0;  // > kMaxKeyChunks on return: every column was laid out, only the total width does not fit
    u32 off = 0;
    for (u32 c = 0; c < L->ncols; ++c) {
        const ytgpu_key_column& k = spec->columns[c];
        KeyColLayout& o = L->col[c];
        o = KeyColLayout{};
        o.index = k.index;
        o.width = k.width;
        o.type = k.type;
        o.descending = k.descending ? 1 : 0;
        u8 t = k.type;
        if (t == YTGPU_TYPE_ANY || t == YTGPU_TYPE_COMPOSITE)
            return make_status(YTGPU_ERR_UNSUPPORTED,
                               "key column %u has type Any/Composite: YSON comparison is not available on the GPU path", c);
        if (fixed_rows) {
            if (t != YTGPU_TYPE_INT64 && t != YTGPU_TYPE_UINT64 && t != YTGPU_TYPE_DOUBLE &&
                t != YTGPU_TYPE_BOOLEAN && t != YTGPU_TYPE_STRING)
                return make_status(YTGPU_ERR_INVALID_ARGUMENT, "fixed-row key column %u needs a concrete scalar type", c);
            o.has_type_byte = force_type_byte ? 1 : 0;
            o.len_bytes = 0;
            o.payload_bytes = t == YTGPU_TYPE_STRING ? k.width : (t == YTGPU_TYPE_BOOLEAN ? 1 : 8);
            if (t == YTGPU_TYPE_STRING && k.width == 0)
                return make_status(YTGPU_ERR_INVALID_ARGUMENT, "fixed-row string key column %u needs a width", c);
        } else {
            bool known = t == YTGPU_TYPE_INT64 || t == YTGPU_TYPE_UINT64 || t == YTGPU_TYPE_DOUBLE ||
                         t == YTGPU_TYPE_BOOLEAN || t == YTGPU_TYPE_STRING || t == YTGPU_TYPE_NULL || t == 0;
            if (!known) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key column %u: bad declared type 0x%x", c, t);
            o.has_type_byte = (force_type_byte || !k.required || t == 0) ? 1 : 0;
            bool may_string = t == YTGPU_TYPE_STRING || t == 0;
            bool may_num8 = t == 0 || t == YTGPU_TYPE_INT64 || t == YTGPU_TYPE_UINT64 || t == YTGPU_TYPE_DOUBLE;
            u32 p = 0;
            if (may_string) {
                o.len_bytes = string_len_bytes(k.width);
                p = k.width + o.len_bytes;
            }
            if (may_num8 && p < 8) p = 8;
            if (t == YTGPU_TYPE_BOOLEAN && p < 1) p = 1;
            o.payload_bytes = p;
        }
        o.byte_offset = off;
        off += o.has_type_byte + o.payload_bytes;
    }
    L->total_bytes = off;
    L->nchunks = (off + 7) / 8;
    if (L->nchunks == 0) L->nchunks = 1;
    if (L->nchunks > (u32)kMaxKeyChunks)
        return make_status(YTGPU_ERR_UNSUPPORTED, "normalised key is %u bytes; the GPU path supports up to %d", off,
                           kMaxKeyChunks * 8);
    return Status{};
}

__host__ __device__ inline u64 normalize_double_bits(u64 bits) {
    const u64 exp_mask = 0x7ff0000000000000ull, frac_mask = 0x000fffffffffffffull;
    if ((bits & exp_mask) == exp_mask && (bits & frac_mask) != 0) bits = 0x7ff8000000000000ull;  // NaN
    if ((bits << 1) == 0) bits = 0;                                                              // -0 -> +0
    return (bits >> 63) ? ~bits : (bits | 0x8000000000000000ull);
}

// Appends bytes most-significant-first into u64 chunks.
struct ChunkWriter {
    u64* out;      // chunk words of one key (local array or staging)
    u32 nbytes = 0;
    u64 acc = 0;
    u32 word = 0;
    u8 inv = 0;
    __host__ __device__ explicit ChunkWriter(u64* o) : out(o) {}
    __host__ __device__ inline void byte(u8 b) {
        acc = (acc << 8) | (u8)(b ^ inv);
        if (++nbytes == 8) {
            out[word++] = acc;
            acc = 0;
            nbytes = 0;
        }
    }
    __host__ __device__ inline void be64(u64 v) {
#pragma unroll
        for (int s = 56; s >= 0; s -= 8) byte((u8)(v >> s));
    }
    __host__ __device__ inline void zeros(u32 n) {
        for (u32 i = 0; i < n; ++i) byte(0);
    }
    __host__ __device__ inline void finish() {
        if (nbytes) {
            // pad the tail with the SAME filler for every key: plain zeros (not inverted)
            acc <<= 8 * (8 - nbytes);
            out[word++] = acc;
            acc = 0;
            nbytes = 0;
        }
    }
};

// Normalises one rowset value into the writer.  Returns DevErr bits.
__host__ __device__ inline u32 normalize_value(const KeyColLayout& c, const ytgpu_value& v, const u8* heap,
                                               ChunkWriter& w) {
    u32 err = 0;
    const u8 t = v.type;
    w.inv = c.descending ? 0xff : 0;
    if (t == YTGPU_TYPE_ANY || t == YTGPU_TYPE_COMPOSITE) err |= DE_UNSUPPORTED_TYPE;
    if (c.type != 0 && t != c.type) {
        if (!(t == YTGPU_TYPE_NULL && c.has_type_byte)) err |= DE_SCHEMA_VIOLATION;
    }
    if (c.has_type_byte) w.byte(t);
    u32 used = 0;
    switch (t) {
        case YTGPU_TYPE_INT64:
            if (c.payload_bytes >= 8) { w.be64(v.data ^ 0x8000000000000000ull); used = 8; }
            break;
        case YTGPU_TYPE_UINT64:
            if (c.payload_bytes >= 8) { w.be64(v.data); used = 8; }
            break;
        case YTGPU_TYPE_DOUBLE:
            if (c.payload_bytes >= 8) { w.be64(normalize_double_bits(v.data)); used = 8; }
            break;
        case YTGPU_TYPE_BOOLEAN:
            if (c.payload_bytes >= 1) { w.byte((v.data & 0xff) != 0); used = 1; }
            break;
        case YTGPU_TYPE_STRING: {
            u32 len = v.length;
            if (len > c.width || c.len_bytes == 0) {
                err |= DE_STRING_TOO_LONG;
                len = len > c.width ? c.width : len;
            }
            const u8* s = heap + v.data;
            for (u32 i = 0; i < len; ++i) w.byte(s[i]);
            w.zeros(c.width - len);
            for (int b = (int)c.len_bytes - 1; b >= 0; --b) w.byte((u8)(v.length >> (8 * b)));
            used = c.width + c.len_bytes;
            break;
        }
        default:
            break;  // Null and sentinels: zero payload
    }
    w.zeros(c.payload_bytes - used);
    return err;
}

// ---- width-free key words (rowset keys whose fixed-width form exceeds kMaxKeyChunks chunks; long_keys.cu) ----
// Column c of a row is the byte string E_c = [type byte] payload, the type byte under the same rule as above:
//   Int64 / Uint64 / Double / Boolean payloads as above (8, 8, 8 and 1 bytes); Null and the sentinels: none;
//   String of length L: L/7 + 1 blocks of 8 bytes, each 7 raw bytes (the last one zero-padded) and a tag byte = the
//   number of raw bytes in the block, or 8 when the block is full and the string continues.  So "ab" < "ab\0" and
//   "abcdefg" < "abcdefg\0" without padding to a width.
// A descending column inverts every byte of E_c.  E_c is cut into big-endian u64 words from the column's own start;
// the tail of the last word is zero padding, never inverted.  Every E_c is order-preserving and prefix-free (rows
// whose words agree up to the end of one row's E_c end it at the same word), so comparing two rows word by word,
// column after column, gives TComparator order.
// A position in the word sequence of a row is a cursor (c << 32) | w; kKeyEnd = past the last column.
constexpr u64 kKeyEnd = ~0ull;

__host__ __device__ inline u64 key_cursor(u32 c, u32 w) { return ((u64)c << 32) | w; }

// Type/schema errors of one key value (the checks normalize_value makes, with the string limit from the layout).
__host__ __device__ inline u32 key_value_errors(const KeyColLayout& c, const ytgpu_value& v) {
    u32 err = 0;
    if (v.type == YTGPU_TYPE_ANY || v.type == YTGPU_TYPE_COMPOSITE) err |= DE_UNSUPPORTED_TYPE;
    if (c.type != 0 && v.type != c.type && !(v.type == YTGPU_TYPE_NULL && c.has_type_byte)) err |= DE_SCHEMA_VIOLATION;
    if (v.type == YTGPU_TYPE_STRING && v.length > c.width) err |= DE_STRING_TOO_LONG;
    return err;
}

__host__ __device__ inline u32 key_string_blocks(u32 len) { return len / 7 + 1; }

// Number of words of E_c.
__host__ __device__ inline u32 key_col_words(const KeyColLayout& c, const ytgpu_value& v) {
    u64 bytes = c.has_type_byte;
    switch (v.type) {
        case YTGPU_TYPE_INT64: case YTGPU_TYPE_UINT64: case YTGPU_TYPE_DOUBLE: bytes += 8; break;
        case YTGPU_TYPE_BOOLEAN: bytes += 1; break;
        case YTGPU_TYPE_STRING: bytes += 8ull * key_string_blocks(v.length); break;
        default: break;
    }
    return (u32)((bytes + 7) / 8);
}

// Bytes [7k, 7k + 7) of a string of length len, zero-padded, as a 56-bit big-endian number.
__host__ __device__ inline u64 key_string_raw7(const u8* s, u32 len, u32 k) {
    u64 r = 0;
    const u32 b0 = 7 * k;
#pragma unroll
    for (u32 i = 0; i < 7; ++i) r = (r << 8) | (b0 + i < len ? s[b0 + i] : 0);
    return r;
}

__host__ __device__ inline u64 key_string_tag(u32 len, u32 k) {
    return k + 1 < key_string_blocks(len) ? 8 : len - 7 * k;
}

// Word w (< key_col_words) of E_c.
__host__ __device__ inline u64 key_col_word(const KeyColLayout& c, const ytgpu_value& v, const u8* heap, u32 w) {
    const u32 tb = c.has_type_byte;
    u64 word;
    u32 bytes;  // meaningful bytes of this word (the rest is padding)
    if (v.type == YTGPU_TYPE_STRING) {
        const u8* s = heap + v.data;
        const u32 nb = key_string_blocks(v.length);
        if (!tb) {  // word w = block w
            word = (key_string_raw7(s, v.length, w) << 8) | key_string_tag(v.length, w);
            bytes = 8;
        } else {    // word w = tag of block w-1 (or the type byte), then the raw bytes of block w
            word = (w == 0 ? (u64)v.type : key_string_tag(v.length, w - 1)) << 56;
            if (w < nb) word |= key_string_raw7(s, v.length, w);
            bytes = w < nb ? 8 : 1;
        }
    } else {
        u64 p = 0;
        u32 pb = 0;
        switch (v.type) {
            case YTGPU_TYPE_INT64: p = v.data ^ 0x8000000000000000ull; pb = 8; break;
            case YTGPU_TYPE_UINT64: p = v.data; pb = 8; break;
            case YTGPU_TYPE_DOUBLE: p = normalize_double_bits(v.data); pb = 8; break;
            case YTGPU_TYPE_BOOLEAN: p = (u64)((v.data & 0xff) != 0) << 56; pb = 1; break;
            default: break;
        }
        // E_c = [type] p (pb bytes, left-aligned in p): at most 9 bytes, words 0 and 1
        const u32 total = tb + pb;
        if (tb) word = w == 0 ? ((u64)v.type << 56) | (p >> 8) : p << 56;
        else word = p;
        bytes = total - 8 * w < 8 ? total - 8 * w : 8;
    }
    const u64 mask = bytes >= 8 ? ~0ull : ~(~0ull >> (8 * bytes));
    if (c.descending) word ^= mask;
    return word & mask;
}

__host__ __device__ inline const ytgpu_value& key_value(const KeyColLayout& c, const ytgpu_value* row) {
    return row[c.index];
}

// First cursor at or after `cur` where rows a and b differ (kKeyEnd: equal from there on).  A cursor past the end of
// a column's words moves on to the next column.
__host__ __device__ inline u64 key_first_diff(const KeyLayout& L, const ytgpu_value* a, const ytgpu_value* b,
                                              const u8* heap, u64 cur) {
    u32 w0 = (u32)cur;
    for (u32 c = (u32)(cur >> 32); c < L.ncols; ++c, w0 = 0) {
        const KeyColLayout& k = L.col[c];
        const ytgpu_value va = key_value(k, a), vb = key_value(k, b);
        const u32 na = key_col_words(k, va), nb = key_col_words(k, vb);
        const u32 nw = na < nb ? na : nb;
        for (u32 w = w0; w < nw; ++w)
            if (key_col_word(k, va, heap, w) != key_col_word(k, vb, heap, w)) return key_cursor(c, w);
        if (na != nb) return key_cursor(c, w0 > nw ? w0 : nw);
    }
    return kKeyEnd;
}

// Word at a cursor returned by key_first_diff (0 past the row's last word).
__host__ __device__ inline u64 key_word_at(const KeyLayout& L, const ytgpu_value* row, const u8* heap, u64 cur) {
    if (cur == kKeyEnd) return 0;
    const KeyColLayout& k = L.col[(u32)(cur >> 32)];
    const ytgpu_value v = key_value(k, row);
    const u32 w = (u32)cur;
    return w < key_col_words(k, v) ? key_col_word(k, v, heap, w) : 0;
}

// Three-way comparison of rows a and b, which are known to be equal before `cur`.
__host__ __device__ inline int key_compare_from(const KeyLayout& L, const ytgpu_value* a, const ytgpu_value* b,
                                                const u8* heap, u64 cur) {
    const u64 d = key_first_diff(L, a, b, heap, cur);
    if (d == kKeyEnd) return 0;
    const KeyColLayout& k = L.col[(u32)(d >> 32)];
    const ytgpu_value va = key_value(k, a), vb = key_value(k, b);
    const u32 w = (u32)d;
    const u32 na = key_col_words(k, va), nb = key_col_words(k, vb);
    if (w >= na || w >= nb) return na < nb ? -1 : 1;  // a shorter E_c (cannot happen for prefix-free E_c)
    return key_col_word(k, va, heap, w) < key_col_word(k, vb, heap, w) ? -1 : 1;
}

// Fixed-row column: raw little-endian scalar / exact-width string at a byte offset.
__host__ __device__ inline void normalize_fixed(const KeyColLayout& c, const u8* row, ChunkWriter& w) {
    w.inv = c.descending ? 0xff : 0;
    if (c.has_type_byte) w.byte(c.type);
    const u8* p = row + c.index;
    if (c.type == YTGPU_TYPE_STRING) {
        for (u32 i = 0; i < c.width; ++i) w.byte(p[i]);
    } else if (c.type == YTGPU_TYPE_BOOLEAN) {
        w.byte(p[0] != 0);
    } else {
        u64 v = 0;
        for (int i = 7; i >= 0; --i) v = (v << 8) | p[i];
        if (c.type == YTGPU_TYPE_INT64) v ^= 0x8000000000000000ull;
        else if (c.type == YTGPU_TYPE_DOUBLE) v = normalize_double_bits(v);
        w.be64(v);
    }
}

}  // namespace ytgpu
