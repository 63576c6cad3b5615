// strings.cuh — a flat string column (ytgpu_string_column) on the device: bounds-checked value access, QL string order
// and the upload of HOST columns, for groupby_multi.cu's string aggregates and the program evaluators (filter.cu,
// expression.cu), and the formats those two share: compiled LIKE / substring patterns and sorted IN lists, with their
// host checks (add_pattern, add_in_list).  Everything is TU-local (anonymous namespace) so several .cu files may include it.
#pragma once

#include <algorithm>
#include <string>
#include <vector>

#include "columnar.cuh"
#include "common.cuh"
#include "context.cuh"
#include "keys.cuh"

namespace {

using namespace ytgpu;

struct StringDev {
    const u8* heap;
    u64 heap_bytes;
    const u64* starts;
    const u32* lengths;
    const u8* nulls;  // nullable bytemap
    u32 present;      // 0: the argument is a scalar ColumnDev
};

// Value i of a string argument: false for NULL; a value that leaves the heap sets the error bit and counts as absent, so
// no later read goes outside the heap.
__device__ __forceinline__ bool string_at(const StringDev& c, u64 i, ytgpu_value* v, u32* bad) {
    if (c.nulls && c.nulls[i]) return false;
    const u64 s = c.starts[i];
    const u32 l = c.lengths[i];
    if (s > c.heap_bytes || (u64)l > c.heap_bytes - s) {
        *bad = 1;
        return false;
    }
    v->type = YTGPU_TYPE_STRING;
    v->length = l;
    v->data = s;
    return true;
}

__device__ __forceinline__ ytgpu_value string_of(const StringDev& c, u64 row) {
    ytgpu_value v{};
    v.type = YTGPU_TYPE_STRING;
    v.length = c.lengths[row];
    v.data = c.starts[row];
    return v;
}

// QL string order through the width-free key words of keys.cuh (a one-column, required, ascending String key): the order
// the long-key sort and the ordered partitioner already use.  Words are prefix-free, so the first differing word decides.
// Two-heap form: a's bytes live in heap_a, b's in heap_b (a column value against a constant of the caller's buffer).
__device__ __forceinline__ int string_compare2(const u8* heap_a, const ytgpu_value& a, const u8* heap_b, const ytgpu_value& b) {
    KeyColLayout L{};
    L.type = YTGPU_TYPE_STRING;
    const u32 na = key_string_blocks(a.length), nb = key_string_blocks(b.length);
    const u32 nw = na < nb ? na : nb;
    for (u32 w = 0; w < nw; ++w) {
        const u64 x = key_col_word(L, a, heap_a, w), y = key_col_word(L, b, heap_b, w);
        if (x != y) return x < y ? -1 : 1;
    }
    return 0;
}

__device__ __forceinline__ int string_compare(const u8* heap, const ytgpu_value& a, const ytgpu_value& b) {
    return string_compare2(heap, a, heap, b);
}

// ---- LIKE patterns and substring needles (semantics and limits in ytgpu.h, YTGPU_FILTER_LIKE) ----
// A pattern is split at % into non-empty segments of positions (a literal byte or _).  All positions of a pattern are
// numbered in one bit space of W = ceil(positions / 64) words; a segment owns the bits [first, last].  Shift-And over a
// value byte b of byte class c:
//   D' = (((D << 1) | inject at first) & table[c]) | (D & any1 & (b is a continuation byte ? ~0 : 0)),  masked to the segment
// where table[c] has the bit of every literal position of a byte in c and of every _ position when c holds bytes outside
// 0x80..0xBF, and any1 has the bits of the _ positions (a _ loops on continuation bytes).  Compiled form, 8-byte aligned:
//   PatternHead | u8 class_of[256] | PatternSeg[segments] | u64 any1[W] | u64 table[classes][W]
// = 272 + 8 * segments + 8 * W * (classes + 1) bytes, the size ytgpu.h states.
struct PatternHead {
    u32 segments;
    u32 flags;  // kPatternAnchorStart: no leading %; kPatternAnchorEnd: no trailing %
    u32 words;
    u32 classes;
};
struct PatternSeg {
    u16 first, last;  // bit range of the segment's positions
    u32 pad;
};
constexpr u32 kPatternAnchorStart = 1, kPatternAnchorEnd = 2;
constexpr u32 kPatternMaxWords = (YTGPU_FILTER_MAX_PATTERN_POSITIONS + 63) / 64;
static_assert(sizeof(PatternHead) == 16 && sizeof(PatternSeg) == 8, "compiled pattern layout");

// The bytes of a contiguous value, for pattern_match.
struct ContiguousBytes {
    const u8* s;
    __device__ __forceinline__ u32 operator()(u32 j) { return __ldg(s + j); }
};

// Whether the value of len bytes matches the compiled pattern at pat (8-byte aligned).  Every middle segment takes its
// earliest end: the % that follows it absorbs any gap, so a later end never admits a match an earlier one does not.  The
// first segment is anchored at 0 when the pattern has no leading %, the last must end at len when it has no trailing %.
// Each value byte is read by at most one segment scan: at most len * W + segments steps.  kWords >= the pattern's W.
// src(j) is byte j of the value; the scan asks for j = 0, 1, 2, ... in order, each at most once, so a source may walk a
// list of pieces instead of indexing (ContiguousBytes for a flat value, expression.cu's piece walk).
template <u32 kWords, class Src>
__device__ __forceinline__ bool pattern_match_words(const u8* pat, Src& src, u32 len) {
    const PatternHead h = *reinterpret_cast<const PatternHead*>(pat);
    const u8* class_of = pat + sizeof(PatternHead);
    const PatternSeg* segs = reinterpret_cast<const PatternSeg*>(class_of + 256);
    const u64* any1 = reinterpret_cast<const u64*>(segs + h.segments);
    const u64* table = any1 + h.words;
    u32 pos = 0;
    for (u32 g = 0; g < h.segments; ++g) {
        const PatternSeg sg = segs[g];
        const bool anchored = g == 0 && (h.flags & kPatternAnchorStart);
        const bool to_end = g + 1 == h.segments && (h.flags & kPatternAnchorEnd);
        u64 D[kWords], M[kWords];
#pragma unroll
        for (u32 w = 0; w < kWords; ++w) {
            D[w] = 0;
            const u32 lo = w * 64;
            const u32 a = sg.first > lo ? sg.first - lo : 0, e = sg.last + 1 - lo;  // e > 64: the word is covered to its top
            M[w] = sg.first >= lo + 64 || sg.last < lo ? 0 : ((e >= 64 ? ~0ull : (1ull << e) - 1) & ~((1ull << a) - 1));
        }
        const u32 fw = sg.first >> 6, lw = sg.last >> 6;
        const u64 fbit = 1ull << (sg.first & 63), lbit = 1ull << (sg.last & 63);
        bool accept = false;
        u32 j = pos;
        while (j < len) {
            const u32 b = src(j);
            const u64* t = table + (u32)class_of[b] * h.words;
            const u64 loop = (b & 0xC0) == 0x80 ? ~0ull : 0;
            const bool inject = !anchored || j == pos;
            u64 carry = 0, alive = 0;
#pragma unroll
            for (u32 w = 0; w < kWords; ++w) {
                if (w < h.words) {
                    u64 sh = (D[w] << 1) | carry;
                    carry = D[w] >> 63;
                    if (inject && w == fw) sh |= fbit;
                    D[w] = ((sh & t[w]) | (D[w] & any1[w] & loop)) & M[w];
                    alive |= D[w];
                }
            }
            ++j;
            accept = false;
#pragma unroll
            for (u32 w = 0; w < kWords; ++w)
                if (w == lw) accept = (D[w] & lbit) != 0;
            if (accept && !to_end) break;  // the earliest end of this segment
            if (anchored && !alive) return false;
        }
        if (!accept) return false;
        if (to_end) return j == len;
        pos = j;
    }
    return true;
}

// A pattern of at most 64 positions (every CONTAINS needle of up to 64 bytes, most LIKE patterns) runs the one-word scan.
template <class Src>
__device__ __forceinline__ bool pattern_match(const u8* pat, Src& src, u32 len) {
    const PatternHead h = *reinterpret_cast<const PatternHead*>(pat);
    if (h.segments == 0) return h.flags == 0 || len == 0;  // all %: any value; the empty pattern: the empty value
    return h.words == 1 ? pattern_match_words<1>(pat, src, len) : pattern_match_words<kPatternMaxWords>(pat, src, len);
}

__device__ __forceinline__ bool pattern_match(const u8* pat, const u8* s, u32 len) {
    ContiguousBytes src{s};
    return pattern_match(pat, src, len);
}

// Compiles a LIKE pattern (like = true; escape -1 or 0..255) or a CONTAINS needle (like = false: the pattern %needle%
// without wildcards), appending its compiled form to *out.  Returns nullptr or the reason the pattern is refused.
inline const char* compile_pattern(const u8* p, u32 len, bool like, int escape, std::vector<u8>* out) {
    constexpr int kStar = -1, kAny = -2;
    std::vector<int> tok;  // literal byte, kStar or kAny
    if (!like) tok.push_back(kStar);
    for (u32 k = 0; k < len; ++k) {
        const int b = p[k];
        if (like && b == escape) {
            if (++k == len) return "the pattern ends in a lone escape byte";
            tok.push_back(p[k]);
        } else {
            tok.push_back(like && b == '%' ? kStar : (like && b == '_' ? kAny : b));
        }
    }
    if (!like) tok.push_back(kStar);
    std::vector<PatternSeg> segs;
    std::vector<int> pos_tok;  // the token of every position
    bool open = false;
    for (int t : tok) {
        if (t == kStar) {
            open = false;
            continue;
        }
        if (!open) segs.push_back(PatternSeg{(u16)pos_tok.size(), 0, 0});
        open = true;
        pos_tok.push_back(t);
        segs.back().last = (u16)(pos_tok.size() - 1);
        if (pos_tok.size() > (size_t)YTGPU_FILTER_MAX_PATTERN_POSITIONS) return "more than YTGPU_FILTER_MAX_PATTERN_POSITIONS positions";
    }
    const u32 words = std::max<u32>(1, (u32)(pos_tok.size() + 63) / 64);
    bool literal[256] = {};
    for (int t : pos_tok)
        if (t >= 0) literal[t] = true;
    u8 class_of[256];
    u32 classes = 0;
    for (int b = 0; b < 256; ++b)
        if (literal[b]) class_of[b] = (u8)classes++;
    int other[2] = {-1, -1};  // the class of the other bytes outside / inside 0x80..0xBF
    for (int b = 0; b < 256; ++b) {
        if (literal[b]) continue;
        int& o = other[(b & 0xC0) == 0x80];
        if (o < 0) o = (int)classes++;
        class_of[b] = (u8)o;
    }
    bool class_cont[256] = {};
    for (int b = 0; b < 256; ++b) class_cont[class_of[b]] = (b & 0xC0) == 0x80;  // every class is all one kind
    std::vector<u64> any1(words, 0), table((size_t)classes * words, 0);
    for (size_t i = 0; i < pos_tok.size(); ++i) {
        const u64 bit = 1ull << (i & 63);
        if (pos_tok[i] >= 0) {
            table[(size_t)class_of[pos_tok[i]] * words + i / 64] |= bit;
        } else {
            any1[i / 64] |= bit;
            for (u32 c = 0; c < classes; ++c)
                if (!class_cont[c]) table[(size_t)c * words + i / 64] |= bit;
        }
    }
    PatternHead h{(u32)segs.size(), 0, words, classes};
    if (tok.empty() || tok.front() != kStar) h.flags |= kPatternAnchorStart;
    if (tok.empty() || tok.back() != kStar) h.flags |= kPatternAnchorEnd;
    auto put = [&](const void* src, size_t bytes) {
        const u8* q = static_cast<const u8*>(src);
        out->insert(out->end(), q, q + bytes);
    };
    put(&h, sizeof h);
    put(class_of, 256);
    put(segs.data(), segs.size() * sizeof(PatternSeg));
    put(any1.data(), any1.size() * 8);
    put(table.data(), table.size() * 8);
    return nullptr;
}

// The patterns of one node, compiled and appended to *patterns (LIKE: escape -1 or 0..255; CONTAINS: escape -1), within the
// per-call limit on compiled bytes.
inline Status add_pattern(u32 k, const u8* p, u32 len, bool like, int escape, std::vector<u8>* patterns) {
    if (like && (escape < -1 || escape > 255))
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: LIKE escape %d outside -1 .. 255", k, escape);
    if (const char* why = compile_pattern(p, len, like, escape, patterns)) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: %s", k, why);
    if (patterns->size() > (size_t)YTGPU_FILTER_MAX_PATTERN_BYTES)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "the patterns of a call compile to more than %d bytes", YTGPU_FILTER_MAX_PATTERN_BYTES);
    return Status{};
}

// ---- IN lists (semantics in ytgpu.h, YTGPU_FILTER_IN and YTGPU_EXPR_IN) ----
constexpr u32 kStagedListEntries = 1024;  // sorted IN entries kept in shared memory per CTA (8 KB)

// A value canonicalised for the IN search: -0.0 becomes +0.0 (the EQ rule says they are equal).
__host__ __device__ __forceinline__ u64 in_key(u8 vtype, u64 bits) {
    if (vtype == YTGPU_TYPE_DOUBLE && bits == 0x8000000000000000ull) bits = 0;
    return minmax_encode(vtype, bits);
}

// Appends the count entries e[] of an IN list over vtype to *out, sorted for the device's binary search: a number's
// in_key words ascending, NaN entries dropped (they never match); a STRING's (offset << 32) | length entries in unsigned
// byte order of consts[offset, offset + length).  Returns -1, or the index of a STRING entry outside the const_bytes
// bytes of consts.
inline i64 prepare_in_list(u8 vtype, const u64* e, u32 count, const u8* consts, u64 const_bytes, std::vector<u64>* out) {
    std::vector<u64> sorted;
    sorted.reserve(count);
    if (vtype == YTGPU_TYPE_STRING) {
        for (u32 j = 0; j < count; ++j) {
            const u64 off = e[j] >> 32, len = e[j] & 0xffffffffu;
            if (off > const_bytes || len > const_bytes - off) return j;
            sorted.push_back(e[j]);
        }
        auto bytes = [&](u64 x) { return std::string(reinterpret_cast<const char*>(consts) + (x >> 32), (size_t)(x & 0xffffffffu)); };
        std::sort(sorted.begin(), sorted.end(), [&](u64 a, u64 b) { return bytes(a) < bytes(b); });  // unsigned bytes
    } else {
        for (u32 j = 0; j < count; ++j) {
            const u64 x = e[j];
            if (vtype == YTGPU_TYPE_DOUBLE && (x & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) continue;  // NaN never matches
            sorted.push_back(in_key(vtype, x));
        }
        std::sort(sorted.begin(), sorted.end());
    }
    out->insert(out->end(), sorted.begin(), sorted.end());
    return -1;
}

// The IN list of node k (count entries e[] over vtype), sorted and appended to *lists; *in_entries counts the entries of
// the call against its limit.
inline Status add_in_list(u32 k, u8 vtype, const u64* e, u32 count, const u8* consts, u64 const_bytes, u64* in_entries,
                          std::vector<u64>* lists) {
    *in_entries += count;
    if (*in_entries > (u64)YTGPU_FILTER_MAX_IN_ENTRIES)
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "at most %d IN entries per call", YTGPU_FILTER_MAX_IN_ENTRIES);
    const i64 bad = prepare_in_list(vtype, e, count, consts, const_bytes, lists);
    if (bad >= 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "node %u: IN entry %u outside string_constants", k, (u32)bad);
    return Status{};
}


// A string column on the device (HOST inputs are uploaded).
struct StagedStrings {
    StringDev dev{};
    InBuf<u8> heap, nulls;
    InBuf<u64> starts;
    InBuf<u32> lengths;
};

Status stage_strings(Context* ctx, const ytgpu_string_column& c, StagedStrings* s) {
    const u64 n = c.row_count;
    YTGPU_TRY(s->heap.stage(ctx, c.heap, c.heap_bytes, c.mem));
    YTGPU_TRY(s->starts.stage(ctx, c.starts, n, c.mem));
    YTGPU_TRY(s->lengths.stage(ctx, c.lengths, n, c.mem));
    YTGPU_TRY(s->nulls.stage(ctx, c.null_bytemap, n, c.mem));
    StringDev& d = s->dev;
    d.heap = s->heap.p;
    d.heap_bytes = c.heap_bytes;
    d.starts = s->starts.p;
    d.lengths = s->lengths.p;
    d.nulls = s->nulls.p;
    d.present = 1;
    return Status{};
}

}  // namespace
