// yt_oracle.cpp — CPU ORACLE (test infrastructure, NOT product code).
//
// A plain C++ restatement of the reference algorithms on the hot path
// (sort / partition / merge / columnar decode / group-by), written from the
// semantics in the reference sources cited next to each function.  Only
// tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
// leg may load this library.  The product (ytsaurus_b200/csrc) never links it.
//
// Parity pinning: the fingerprint / partitioner / compare / columnar functions
// are checked against the golden vectors transcribed from the reference's own
// unit tests (tests/golden/*.json), the FarmHash functions also against known
// answers of the reference's vendored FarmHash (tests/golden/farmhash_fingerprints.json).
//
// All paths relative to the reference tree's root.

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <functional>
#include <numeric>
#include <string_view>
#include <thread>
#include <unordered_map>
#include <map>
#include <vector>

namespace {

using u8 = uint8_t;
using u16 = uint16_t;
using u32 = uint32_t;
using u64 = uint64_t;
using i32 = int32_t;
using i64 = int64_t;

// ---------------------------------------------------------------------------
// Row model.  yt/yt/client/table_client/unversioned_value.h:37-62 (16-byte POD),
// row_base.h:11-28 (type codes).  In the flat interchange form used by the
// tests, a string value's Data field holds an OFFSET into a byte heap instead
// of a pointer.
// ---------------------------------------------------------------------------
enum : u8 {
    T_MIN = 0x00, T_BOTTOM = 0x01, T_NULL = 0x02, T_INT64 = 0x03, T_UINT64 = 0x04,
    T_DOUBLE = 0x05, T_BOOLEAN = 0x06, T_STRING = 0x10, T_ANY = 0x11, T_COMPOSITE = 0x12,
    T_MAX = 0xef,
};

struct Value {
    u16 id;
    u8 type;
    u8 flags;
    u32 length;
    u64 data;  // i64 / u64 / double bits / bool in low byte / heap offset for strings
};
static_assert(sizeof(Value) == 16, "value must be 16 bytes");

inline double as_double(u64 bits) { double d; std::memcpy(&d, &bits, 8); return d; }
inline std::string_view as_string(const Value& v, const char* heap) {
    return std::string_view(heap + v.data, v.length);
}

enum { ERR_OK = 0, ERR_UNSUPPORTED_TYPE = 1, ERR_BAD_ARGUMENT = 2, ERR_PARTITION = 3 };

// ---------------------------------------------------------------------------
// FarmHash fingerprints.  contrib/libs/farmhash (version 2017-06-26, ya.make:7):
// farmhash.h:158-181 (Fingerprint(u64), Fingerprint(u128)), farmhash.cc:408-578
// (farmhashna::Hash64 == util::Fingerprint64, farmhash.cc:1957-1959).
// Restated from the published algorithm; validated bit-for-bit against the
// vendored source (known answers in tests/golden/farmhash_fingerprints.json).
// ---------------------------------------------------------------------------
constexpr u64 K0 = 0xc3a5c85c97cb3127ULL;
constexpr u64 K1 = 0xb492b66fbe98f273ULL;
constexpr u64 K2 = 0x9ae16a3b2f90404fULL;
constexpr u64 KMUL = 0x9ddfea08eb382d69ULL;

inline u64 rd64(const char* p) { u64 x; std::memcpy(&x, p, 8); return x; }
inline u64 rd32(const char* p) { u32 x; std::memcpy(&x, p, 4); return x; }
inline u64 ror(u64 v, int s) { return s == 0 ? v : ((v >> s) | (v << (64 - s))); }
inline u64 smix(u64 v) { return v ^ (v >> 47); }

inline u64 fp_u64(u64 x) {  // farmhash.h:172-181
    u64 b = x * KMUL;
    b ^= b >> 44;
    b *= KMUL;
    b ^= b >> 41;
    b *= KMUL;
    return b;
}
inline u64 fp_u128(u64 lo, u64 hi) {  // farmhash.h:158-169
    u64 a = (lo ^ hi) * KMUL;
    a ^= a >> 47;
    u64 b = (hi ^ a) * KMUL;
    b ^= b >> 44;
    b *= KMUL;
    b ^= b >> 41;
    b *= KMUL;
    return b;
}
inline u64 h128to64(u64 lo, u64 hi) {  // farmhash.h:131-141
    u64 a = (lo ^ hi) * KMUL;
    a ^= a >> 47;
    u64 b = (hi ^ a) * KMUL;
    b ^= b >> 47;
    b *= KMUL;
    return b;
}
inline u64 hl16(u64 u, u64 v, u64 mul) {
    u64 a = (u ^ v) * mul;
    a ^= a >> 47;
    u64 b = (v ^ a) * mul;
    b ^= b >> 47;
    return b * mul;
}
struct P2 { u64 a, b; };
inline P2 weak32(u64 w, u64 x, u64 y, u64 z, u64 a, u64 b) {
    a += w;
    b = ror(b + a + z, 21);
    u64 c = a;
    a += x;
    a += y;
    b += ror(a, 44);
    return {a + z, b + c};
}
inline P2 weak32(const char* s, u64 a, u64 b) {
    return weak32(rd64(s), rd64(s + 8), rd64(s + 16), rd64(s + 24), a, b);
}

u64 fp_bytes(const char* s, size_t len) {
    if (len <= 16) {
        if (len >= 8) {
            u64 mul = K2 + len * 2;
            u64 a = rd64(s) + K2;
            u64 b = rd64(s + len - 8);
            u64 c = ror(b, 37) * mul + a;
            u64 d = (ror(a, 25) + b) * mul;
            return hl16(c, d, mul);
        }
        if (len >= 4) {
            u64 mul = K2 + len * 2;
            u64 a = rd32(s);
            return hl16(len + (a << 3), rd32(s + len - 4), mul);
        }
        if (len > 0) {
            u8 a = (u8)s[0], b = (u8)s[len >> 1], c = (u8)s[len - 1];
            u32 y = (u32)a + ((u32)b << 8);
            u32 z = (u32)len + ((u32)c << 2);
            return smix(y * K2 ^ z * K0) * K2;
        }
        return K2;
    }
    if (len <= 32) {
        u64 mul = K2 + len * 2;
        u64 a = rd64(s) * K1;
        u64 b = rd64(s + 8);
        u64 c = rd64(s + len - 8) * mul;
        u64 d = rd64(s + len - 16) * K2;
        return hl16(ror(a + b, 43) + ror(c, 30) + d, a + ror(b + K2, 18) + c, mul);
    }
    if (len <= 64) {
        u64 mul = K2 + len * 2;
        u64 a = rd64(s) * K2;
        u64 b = rd64(s + 8);
        u64 c = rd64(s + len - 8) * mul;
        u64 d = rd64(s + len - 16) * K2;
        u64 y = ror(a + b, 43) + ror(c, 30) + d;
        u64 z = hl16(y, a + ror(b + K2, 18) + c, mul);
        u64 e = rd64(s + 16) * mul;
        u64 f = rd64(s + 24);
        u64 g = (y + rd64(s + len - 32)) * mul;
        u64 h = (z + rd64(s + len - 24)) * mul;
        return hl16(ror(e + f, 43) + ror(g, 30) + h, e + ror(f + a, 18) + g, mul);
    }
    const u64 seed = 81;
    u64 x = seed;
    u64 y = seed * K1 + 113;
    u64 z = smix(y * K2 + 113) * K2;
    P2 v{0, 0}, w{0, 0};
    x = x * K2 + rd64(s);
    const char* end = s + ((len - 1) / 64) * 64;
    const char* last64 = end + ((len - 1) & 63) - 63;
    do {
        x = ror(x + y + v.a + rd64(s + 8), 37) * K1;
        y = ror(y + v.b + rd64(s + 48), 42) * K1;
        x ^= w.b;
        y += v.a + rd64(s + 40);
        z = ror(z + w.a, 33) * K1;
        v = weak32(s, v.b * K1, x + w.a);
        w = weak32(s + 32, z + w.b, y + rd64(s + 16));
        std::swap(z, x);
        s += 64;
    } while (s != end);
    u64 mul = K1 + ((z & 0xff) << 1);
    s = last64;
    w.a += ((len - 1) & 63);
    v.a += w.a;
    w.a += v.a;
    x = ror(x + y + v.a + rd64(s + 8), 37) * mul;
    y = ror(y + v.b + rd64(s + 48), 42) * mul;
    x ^= w.b * 9;
    y += v.a * 9 + rd64(s + 40);
    z = ror(z + w.a, 33) * mul;
    v = weak32(s, v.b * mul, x + w.a);
    w = weak32(s + 32, z + w.b, y + rd64(s + 16));
    std::swap(z, x);
    return hl16(hl16(v.a, w.a, mul) + smix(y) * K0 + z, hl16(v.b, w.b, mul) + x, mul);
}

// yt/yt/client/table_client/unversioned_value.cpp:33-72.
int value_fingerprint(const Value& v, const char* heap, u64* out) {
    switch (v.type) {
        case T_STRING: *out = fp_bytes(heap + v.data, v.length); return ERR_OK;
        case T_INT64:
        case T_UINT64:
        case T_DOUBLE: *out = fp_u64(v.data); return ERR_OK;
        case T_BOOLEAN: *out = fp_u64((u64)((v.data & 0xff) != 0)); return ERR_OK;
        case T_NULL: *out = fp_u64(0); return ERR_OK;
        default: return ERR_UNSUPPORTED_TYPE;  // Any/Composite need YSON hashing; sentinels throw.
    }
}

// library/cpp/yt/farmhash/farm_hash.h:51-59.
int range_fingerprint(const Value* begin, u32 count, const char* heap, u64* out) {
    u64 h = 0xdeadc0de;
    for (u32 i = 0; i < count; ++i) {
        u64 f;
        if (int e = value_fingerprint(begin[i], heap, &f)) return e;
        h = fp_u128(h, f);  // FarmFingerprint(first, second) = Fingerprint(Uint128(first, second)): low=first
    }
    *out = h ^ (u64)count;
    return ERR_OK;
}

// ---------------------------------------------------------------------------
// Comparison.  yt/yt/client/table_client/unversioned_row.cpp:392-464
// (CompareRowValues), library/cpp/yt/misc/compare-inl.h:18-66, and
// comparator.cpp:52-61,174-200 (sort orders), :77-103 (TestKey).
// Any/Composite need the YSON comparer: rejected, like the GPU path.
// ---------------------------------------------------------------------------
inline int tern(u64 a, u64 b) { return a == b ? 0 : (a < b ? -1 : 1); }
inline int terni(i64 a, i64 b) { return a == b ? 0 : (a < b ? -1 : 1); }
inline int nan_safe(double a, double b) {
    if (a < b) return -1;
    if (a > b) return 1;
    if (std::isnan(a)) return std::isnan(b) ? 0 : 1;
    if (std::isnan(b)) return -1;
    return 0;
}
inline int sgn(int x) { return (x > 0) - (x < 0); }

inline bool is_complex(u8 t) { return t == T_ANY || t == T_COMPOSITE; }

int compare_values(const Value& l, const char* lheap, const Value& r, const char* rheap) {
    if (l.type != r.type) return tern(l.type, r.type);
    switch (l.type) {
        case T_INT64: return terni((i64)l.data, (i64)r.data);
        case T_UINT64: return tern(l.data, r.data);
        case T_DOUBLE: return nan_safe(as_double(l.data), as_double(r.data));
        case T_BOOLEAN: return tern((l.data & 0xff) != 0, (r.data & 0xff) != 0);
        case T_STRING: return sgn(as_string(l, lheap).compare(as_string(r, rheap)));
        default: return 0;  // sentinels / null equal to themselves
    }
}

struct Comparator {
    u32 length;
    const u8* descending;  // per key column, may be null (all ascending)
    int compare_value(u32 idx, const Value& l, const char* lh, const Value& r, const char* rh) const {
        int c = compare_values(l, lh, r, rh);
        return (descending && descending[idx]) ? -c : c;
    }
    int compare_keys(const Value* l, const char* lh, const Value* r, const char* rh) const {
        for (u32 i = 0; i < length; ++i) {
            int c = compare_value(i, l[i], lh, r[i], rh);
            if (c) return c;
        }
        return 0;
    }
    // comparator.cpp:77-103; lower bounds only need IsUpper=false, kept general.
    bool test_key(const Value* key, const char* kh, const Value* prefix, u32 prefix_len,
                  const char* bh, bool inclusive, bool upper) const {
        int c = 0;
        for (u32 i = 0; i < prefix_len; ++i) {
            c = compare_value(i, key[i], kh, prefix[i], bh);
            if (c) break;
        }
        if (upper) c = -c;
        return c > 0 || (c == 0 && inclusive);
    }
};

bool keys_supported(const Value* v, size_t nrows, u32 ncols, u32 nkey) {
    for (size_t r = 0; r < nrows; ++r)
        for (u32 c = 0; c < nkey; ++c)
            if (is_complex(v[r * ncols + c].type)) return false;
    return true;
}

double now_s() {
    return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// ---------------------------------------------------------------------------
// TPartitionSortReader restated: key-only buffer, 10 000-row buckets sorted with
// std::sort over i32 indices, k-way heap merge.
// yt/yt/ytlib/table_client/partition_sort_reader.cpp:362-363 (bucket size),
// :461-472 (DoSortBucket), :484-529 (DoMerge).  The reference's heap helpers
// (MakeHeap/AdjustHeapFront/ExtractHeap) are a binary min-heap; std::*_heap
// with the inverted predicate yields the same pop order up to ties, and ties
// are unspecified in the reference (docs sort.md:5-9).
// ---------------------------------------------------------------------------
constexpr int kSortBucketSize = 10000;

template <class Less>
void bucket_sort_merge(u32 n, Less less, u32* out) {
    std::vector<u32> idx(n);
    std::iota(idx.begin(), idx.end(), 0u);
    std::vector<u32> starts;
    for (u32 s = 0; s < n; s += kSortBucketSize) starts.push_back(s);
    size_t nb = starts.size();
    for (size_t b = 0; b < nb; ++b) {
        u32 e = std::min<u32>(n, starts[b] + kSortBucketSize);
        std::sort(idx.begin() + starts[b], idx.begin() + e, less);
    }
    struct Cur { u32 pos, end; };
    std::vector<Cur> heap;
    for (size_t b = 0; b < nb; ++b) heap.push_back({starts[b], std::min<u32>(n, starts[b] + kSortBucketSize)});
    auto heap_greater = [&](const Cur& a, const Cur& b) { return less(idx[b.pos], idx[a.pos]); };
    std::make_heap(heap.begin(), heap.end(), heap_greater);
    u32 o = 0;
    while (!heap.empty()) {
        std::pop_heap(heap.begin(), heap.end(), heap_greater);
        Cur& c = heap.back();
        out[o++] = idx[c.pos++];
        if (c.pos == c.end) heap.pop_back();
        else std::push_heap(heap.begin(), heap.end(), heap_greater);
    }
}

// ---------------------------------------------------------------------------
// Columnar helpers (yt/yt/client/table_client/columnar-inl.h, columnar.cpp).
// ---------------------------------------------------------------------------
inline bool get_bit(const u8* bitmap, i64 i) { return (bitmap[i >> 3] >> (i & 7)) & 1; }
inline i64 zigzag_decode64(u64 v) { return (i64)(v >> 1) ^ -(i64)(v & 1); }
inline i32 zigzag_decode32(u32 v) { return (i32)(v >> 1) ^ -(i32)(v & 1); }

// columnar.cpp:737-770 TranslateRleIndex: largest k with rle[k] <= index.
inline i64 translate_rle_index(const u64* rle, i64 n_rle, i64 index) {
    const u64* it = std::upper_bound(rle, rle + n_rle, (u64)index);
    return (it - rle) - 1;
}

}  // namespace

// ===========================================================================
// C ABI for ctypes (tests) and bench.py's CPU baseline.
// ===========================================================================
extern "C" {

u64 yto_farm_fingerprint_u64(u64 x) { return fp_u64(x); }
u64 yto_farm_fingerprint_u128(u64 lo, u64 hi) { return fp_u128(lo, hi); }
u64 yto_farm_fingerprint_bytes(const char* s, size_t n) { return fp_bytes(s, n); }
u64 yto_hash128to64(u64 lo, u64 hi) { return h128to64(lo, hi); }

int yto_value_fingerprints(const Value* v, const char* heap, size_t n, u64* out) {
    for (size_t i = 0; i < n; ++i)
        if (int e = value_fingerprint(v[i], heap, &out[i])) return e;
    return ERR_OK;
}

// GetFarmFingerprint(row.FirstNElements(min(k, ncols))) per row.
int yto_row_fingerprints(const Value* v, const char* heap, size_t nrows, u32 ncols, u32 k, u64* out) {
    u32 cnt = std::min(k, ncols);
    for (size_t r = 0; r < nrows; ++r)
        if (int e = range_fingerprint(v + r * ncols, cnt, heap, &out[r])) return e;
    return ERR_OK;
}

int yto_compare_values(const Value* a, const Value* b, const char* heap, int* out) {
    if (is_complex(a->type) || is_complex(b->type)) return ERR_UNSUPPORTED_TYPE;
    *out = compare_values(*a, heap, *b, heap);
    return ERR_OK;
}

int yto_compare_keys(const Value* a, const Value* b, const char* heap, u32 nkey, const u8* desc, int* out) {
    Comparator c{nkey, desc};
    *out = c.compare_keys(a, heap, b, heap);
    return ERR_OK;
}

// algo: 0 = TSortingReader (std::sort, sorting_reader.cpp:179-187)
//       1 = std::stable_sort with the same comparator (strict oracle for the stable GPU sort)
//       2 = TPartitionSortReader (buckets of 10 000 + heap merge)
int yto_sort_rows(const Value* v, const char* heap, size_t nrows, u32 ncols, u32 nkey, const u8* desc,
                  int algo, u32* perm, double* seconds) {
    if (nkey > ncols) return ERR_BAD_ARGUMENT;
    if (!keys_supported(v, nrows, ncols, nkey)) return ERR_UNSUPPORTED_TYPE;
    Comparator cmp{nkey, desc};
    auto less = [&](u32 a, u32 b) {
        return cmp.compare_keys(v + (size_t)a * ncols, heap, v + (size_t)b * ncols, heap) < 0;
    };
    double t0 = now_s();
    if (algo == 2) {
        bucket_sort_merge((u32)nrows, less, perm);
    } else {
        std::iota(perm, perm + nrows, 0u);
        if (algo == 0) std::sort(perm, perm + nrows, less);
        else std::stable_sort(perm, perm + nrows, less);
    }
    if (seconds) *seconds = now_s() - t0;
    return ERR_OK;
}

// TOrderedPartitioner::GetPartitionIndex, yt/yt/ytlib/table_client/partitioner.cpp:41-57.
// bounds: nbounds rows of `bcols` values each; bound b uses its first bound_len[b] values as the prefix
// (bound 0 is normally universal: len 0, inclusive).  All are LOWER bounds (IsUpper=false).
int yto_partition_ordered(const Value* v, const char* heap, size_t nrows, u32 ncols, u32 nkey, const u8* desc,
                          const Value* bounds, const char* bheap, u32 nbounds, u32 bcols,
                          const u32* bound_len, const u8* bound_inclusive, i32* out, double* seconds) {
    if (!keys_supported(v, nrows, ncols, nkey)) return ERR_UNSUPPORTED_TYPE;
    Comparator cmp{nkey, desc};
    double t0 = now_s();
    for (size_t r = 0; r < nrows; ++r) {
        const Value* key = v + r * ncols;
        // upper_bound with comp(key, bound) = !TestKey(key, bound)
        u32 lo = 0, cnt = nbounds;
        while (cnt > 0) {
            u32 step = cnt / 2, mid = lo + step;
            bool comp = !cmp.test_key(key, heap, bounds + (size_t)mid * bcols, bound_len[mid], bheap,
                                      bound_inclusive[mid] != 0, false);
            if (!comp) { lo = mid + 1; cnt -= step + 1; } else cnt = step;
        }
        if (lo == 0) return ERR_PARTITION;  // YT_VERIFY(partitionsIt != begin)
        out[r] = (i32)lo - 1;
    }
    if (seconds) *seconds = now_s() - t0;
    return ERR_OK;
}

// THashPartitioner, partitioner.cpp:84-113: Salt_ = FarmHash(salt) (ctor), index = hash % P.
int yto_partition_hash(const Value* v, const char* heap, size_t nrows, u32 ncols, i32 partition_count,
                       i32 key_column_count, u64 salt, i32* out, double* seconds) {
    u64 salt_h = fp_u64(salt);
    double t0 = now_s();
    for (size_t r = 0; r < nrows; ++r) {
        u32 cnt = (u32)std::min<i64>(key_column_count, ncols);
        u64 h;
        if (int e = range_fingerprint(v + r * ncols, cnt, heap, &h)) return e;
        if (salt_h != 0) h = fp_u64(h ^ salt_h);
        out[r] = (i32)(h % (u64)partition_count);
    }
    if (seconds) *seconds = now_s() - t0;
    return ERR_OK;
}

// TColumnBasedPartitioner, partitioner.cpp:122-173.  Returns per-row index or an error code:
// 10 = bad type, 11 = negative, 12 = out of bounds, 13 = column missing.
int yto_partition_column(const Value* v, size_t nrows, u32 ncols, i32 partition_count, u16 column_id, i32* out) {
    for (size_t r = 0; r < nrows; ++r) {
        bool found = false;
        for (u32 c = 0; c < ncols && !found; ++c) {
            const Value& x = v[r * ncols + c];
            if (x.id != column_id) continue;
            if (x.type != T_UINT64 && x.type != T_INT64) return 10;
            if (x.type == T_INT64 && (i64)x.data < 0) return 11;
            if (x.data >= (u64)partition_count) return 12;
            out[r] = (i32)x.data;
            found = true;
        }
        if (!found) return 13;
    }
    return ERR_OK;
}

// TSortedMergingReader, sorted_merging_reader.cpp:395-409,438-545: heap of streams ordered by
// (key, table index).  Runs are consecutive slices [run_off[i], run_off[i+1]) of the row array.
int yto_merge_sorted(const Value* v, const char* heap, u32 ncols, u32 nkey, const u8* desc,
                     const u64* run_off, u32 nruns, u32* perm) {
    Comparator cmp{nkey, desc};
    struct S { u64 pos, end; u32 idx; };
    std::vector<S> h;
    for (u32 i = 0; i < nruns; ++i)
        if (run_off[i] < run_off[i + 1]) h.push_back({run_off[i], run_off[i + 1], i});
    auto greater = [&](const S& a, const S& b) {
        int c = cmp.compare_keys(v + a.pos * ncols, heap, v + b.pos * ncols, heap);
        if (c) return c > 0;
        return a.idx > b.idx;
    };
    std::make_heap(h.begin(), h.end(), greater);
    u64 o = 0;
    while (!h.empty()) {
        std::pop_heap(h.begin(), h.end(), greater);
        S& s = h.back();
        perm[o++] = (u32)s.pos++;
        if (s.pos == s.end) h.pop_back();
        else std::push_heap(h.begin(), h.end(), greater);
    }
    return ERR_OK;
}

// TSortedJoiningReader::Read without interrupts, sorted_merging_reader.cpp:566-760.  Stream 0 is the primary stream
// (the merged primary readers), streams 1.. are the foreign readers; every stream is sorted by the join key (the first
// nkey values) and carries ONE table index — TSortedStream evaluates it once, from the first row it reads
// (sorted_merging_reader.cpp:101-104).  The heap orders the streams by (join key of the head row, table index)
// (CompareStreams :395-409).  A primary row is always emitted; a foreign row is emitted iff its join key equals the
// last primary key consumed or the key of the primary stream's head row (:722-738).
// perm receives the emitted rows in order, *out_count their number.
int yto_join_sorted(const Value* v, const char* heap, u32 ncols, u32 nkey, const u8* desc, const u64* run_off,
                    u32 nruns, const i32* table_index /* per stream */, u32* perm, u64* out_count) {
    Comparator cmp{nkey, desc};
    struct S { u64 pos, end; u32 idx; i32 table; };
    std::vector<S> h;
    for (u32 i = 0; i < nruns; ++i)
        if (run_off[i] < run_off[i + 1]) h.push_back({run_off[i], run_off[i + 1], i, table_index[i]});
    auto greater = [&](const S& a, const S& b) {
        int c = cmp.compare_keys(v + a.pos * ncols, heap, v + b.pos * ncols, heap);
        if (c) return c > 0;
        return a.table > b.table;
    };
    std::make_heap(h.begin(), h.end(), greater);
    u64 primary_pos = run_off[0];            // head of the primary stream
    const u64 primary_end = nruns ? run_off[1] : 0;
    bool have_last = false;
    u64 last_primary = 0;
    u64 o = 0;
    while (!h.empty()) {
        std::pop_heap(h.begin(), h.end(), greater);
        S& s = h.back();
        const u64 row = s.pos;
        bool output = false;
        if (s.idx == 0) {
            output = true;
            have_last = true;
            last_primary = row;
            primary_pos = row + 1;
        } else {
            if (have_last && cmp.compare_keys(v + last_primary * ncols, heap, v + row * ncols, heap) == 0) output = true;
            if (!output && primary_pos < primary_end &&
                cmp.compare_keys(v + primary_pos * ncols, heap, v + row * ncols, heap) == 0)
                output = true;
        }
        if (output) perm[o++] = (u32)row;
        ++s.pos;
        if (s.pos == s.end) h.pop_back();
        else std::push_heap(h.begin(), h.end(), greater);
    }
    *out_count = o;
    return ERR_OK;
}

// ---------------------------------------------------------------------------
// Fixed-width row tables (the benchmark's "64-byte row"): rows are row_bytes-wide
// records, key columns at fixed offsets.  To time what the reference actually does
// we first build the reference's in-memory model — 8 B header + 16 B values, string
// bytes out of line (unversioned_row.h:153-156,272-352) — OUTSIDE the timed region,
// then run the reference sort over row pointers INSIDE it.
// column kinds: type code (INT64/UINT64/DOUBLE/BOOLEAN/STRING) + width (strings).
// ---------------------------------------------------------------------------
struct FixedCol { u32 offset; u32 width; u8 type; u8 descending; u8 pad[2]; };

struct RefRow { u32 count, capacity; Value values[1]; };  // header + values (flexible)

static void build_ref_rows(const u8* rows, size_t n, u32 row_bytes, const FixedCol* cols, u32 ncols_key,
                           std::vector<u8>& pool, std::vector<const Value*>& ptrs) {
    // Each row: header + (ncols_key + 1) values: key columns then one payload string = whole record.
    size_t stride = 8 + 16 * (size_t)(ncols_key + 1);
    pool.resize(n * stride);
    ptrs.resize(n);
    for (size_t r = 0; r < n; ++r) {
        u8* p = pool.data() + r * stride;
        u32 hdr[2] = {ncols_key + 1, ncols_key + 1};
        std::memcpy(p, hdr, 8);
        Value* vals = reinterpret_cast<Value*>(p + 8);
        const u8* rec = rows + r * row_bytes;
        for (u32 c = 0; c < ncols_key; ++c) {
            Value v{(u16)c, cols[c].type, 0, 0, 0};
            if (cols[c].type == T_STRING) {
                v.length = cols[c].width;
                v.data = (u64)(uintptr_t)(rec + cols[c].offset);  // absolute pointer; heap base = nullptr
            } else if (cols[c].type == T_BOOLEAN) {
                v.data = rec[cols[c].offset] != 0;
            } else {
                std::memcpy(&v.data, rec + cols[c].offset, 8);
            }
            vals[c] = v;
        }
        vals[ncols_key] = Value{(u16)ncols_key, T_STRING, 0, row_bytes, (u64)(uintptr_t)rec};
        ptrs[r] = vals;
    }
}

// algo as in yto_sort_rows; threads>1: `threads` independent range partitions (sampled pivots,
// ordered partitioner), each sorted as its own "job" with algo 2, outputs concatenated — models YT
// running one sort job per CPU slot (SURVEY §8d ref-sort-NT).  Returns seconds of the timed region.
int yto_sort_fixed_rows(const u8* rows, size_t n, u32 row_bytes, const FixedCol* cols, u32 nkey,
                        int algo, int threads, u32* perm, double* seconds) {
    std::vector<u8> pool;
    std::vector<const Value*> ptrs;
    build_ref_rows(rows, n, row_bytes, cols, nkey, pool, ptrs);
    std::vector<u8> desc(nkey);
    for (u32 c = 0; c < nkey; ++c) desc[c] = cols[c].descending;
    Comparator cmp{nkey, desc.data()};
    const char* heap0 = nullptr;  // string data fields hold absolute addresses
    auto less = [&](u32 a, u32 b) { return cmp.compare_keys(ptrs[a], heap0, ptrs[b], heap0) < 0; };
    double t0 = now_s();
    if (threads <= 1) {
        if (algo == 2) bucket_sort_merge((u32)n, less, perm);
        else {
            std::iota(perm, perm + n, 0u);
            if (algo == 0) std::sort(perm, perm + n, less);
            else std::stable_sort(perm, perm + n, less);
        }
    } else {
        // sample -> pivots -> partition (partition job) -> per-partition sort job.
        u32 P = (u32)threads;
        std::vector<u32> samples;
        size_t ns = std::min<size_t>(n, 1000 * (size_t)P);
        for (size_t i = 0; i < ns; ++i) samples.push_back((u32)((i * 2654435761ull) % n));
        std::sort(samples.begin(), samples.end(), less);
        std::vector<u32> pivots;
        for (u32 p = 1; p < P; ++p) pivots.push_back(samples[(size_t)p * ns / P]);
        // Partition phase: `threads` partition jobs over contiguous input slices (each emits P buckets),
        // then sort job p reads bucket p of every partition job in job order (stable concatenation).
        std::vector<std::vector<std::vector<u32>>> sub(P, std::vector<std::vector<u32>>(P));
        {
            std::vector<std::thread> pt;
            for (u32 t = 0; t < P; ++t) {
                pt.emplace_back([&, t] {
                    size_t lo_r = n * t / P, hi_r = n * (t + 1) / P;
                    for (auto& v : sub[t]) v.reserve((hi_r - lo_r) / P + 64);
                    for (size_t r = lo_r; r < hi_r; ++r) {
                        // partition index = number of pivots <= key (inclusive lower bounds)
                        u32 lo = 0, cnt = (u32)pivots.size();
                        while (cnt > 0) {
                            u32 step = cnt / 2, mid = lo + step;
                            if (!less((u32)r, pivots[mid])) { lo = mid + 1; cnt -= step + 1; } else cnt = step;
                        }
                        sub[t][lo].push_back((u32)r);
                    }
                });
            }
            for (auto& t : pt) t.join();
        }
        std::vector<std::vector<u32>> parts(P);
        for (u32 p = 0; p < P; ++p) {
            size_t tot = 0;
            for (u32 t = 0; t < P; ++t) tot += sub[t][p].size();
            parts[p].reserve(tot);
        }
        {
            std::vector<std::thread> ct;
            for (u32 p = 0; p < P; ++p)
                ct.emplace_back([&, p] {
                    for (u32 t = 0; t < P; ++t) parts[p].insert(parts[p].end(), sub[t][p].begin(), sub[t][p].end());
                });
            for (auto& t : ct) t.join();
        }
        std::vector<size_t> offs(P + 1, 0);
        for (u32 p = 0; p < P; ++p) offs[p + 1] = offs[p] + parts[p].size();
        std::vector<std::thread> th;
        for (u32 p = 0; p < P; ++p) {
            th.emplace_back([&, p] {
                auto& ids = parts[p];
                auto less_l = [&](u32 a, u32 b) { return less(ids[a], ids[b]); };
                std::vector<u32> local(ids.size());
                bucket_sort_merge((u32)ids.size(), less_l, local.data());
                for (size_t i = 0; i < ids.size(); ++i) perm[offs[p] + i] = ids[local[i]];
            });
        }
        for (auto& t : th) t.join();
    }
    if (seconds) *seconds = now_s() - t0;
    return ERR_OK;
}

// ---------------------------------------------------------------------------
// Bit-packed unsigned vectors, yt/yt/core/misc/bit_packed_unsigned_vector-inl.h:31-173.
// ---------------------------------------------------------------------------
static inline u32 bit_width_of(u64 max_value) { return max_value == 0 ? 0 : 64 - __builtin_clzll(max_value); }

size_t yto_bit_pack(const u64* values, size_t n, u64 max_value, u64* dst /* zeroed, 1 + ceil(w*n/64) words */) {
    u64 width = bit_width_of(max_value);
    dst[0] = (u64)n | (width << 56);
    if (width == 0) return 1;
    size_t words = (width * n + 63) >> 6;
    for (size_t i = 0; i < n; ++i) {
        u64 bit = i * width;
        size_t w = bit >> 6;
        u32 off = bit & 63;
        dst[1 + w] |= values[i] << off;
        if (off + width > 64) dst[2 + w] |= values[i] >> (64 - off);
    }
    return 1 + words;
}

void yto_bit_unpack(const u64* packed, u64* out) {
    u64 size = packed[0] & ((1ull << 56) - 1);
    u32 width = (u32)(packed[0] >> 56);
    const u64* data = packed + 1;
    for (u64 i = 0; i < size; ++i) {
        if (width == 0) { out[i] = 0; continue; }
        u64 bit = i * width;
        const u64* word = data + (bit >> 6);
        u32 off = bit & 63;
        u64 w1 = word[0] >> off;
        if (off + width > 64) {
            u64 w2 = (word[1] & ((1ull << ((off + width) & 63)) - 1)) << (64 - off);
            out[i] = w1 | w2;
        } else {
            out[i] = width == 64 ? w1 : (w1 & ((1ull << width) - 1));
        }
    }
}

// DecodeIntegerVector, columnar-inl.h:355-376 (+ :66-182, :236-247).  `values` is the (already
// bit-unpacked) ui64 vector of the value column; dict_idx / rle_idx / bitmap may be null.
// Semantics per element: resolve RLE run, resolve dictionary (0 => default value 0), null => 0,
// else (raw + base) then zigzag.
void yto_decode_integer_vector(i64 start, i64 end, u64 base, int zigzag, const u32* dict_idx,
                               const u64* rle_idx, i64 n_rle, const u8* bitmap, const u64* values, u64* out) {
    for (i64 i = start; i < end; ++i) {
        i64 pos = i;
        if (rle_idx) pos = translate_rle_index(rle_idx, n_rle, i);
        bool is_null = false;
        bool is_default = false;
        u64 raw = 0;
        if (dict_idx) {
            u32 d = dict_idx[pos];
            if (d == 0) is_default = true;
            else if (bitmap && get_bit(bitmap, (i64)d - 1)) is_null = true;
            else raw = values[d - 1];
        } else {
            if (bitmap && get_bit(bitmap, pos)) is_null = true;
            else raw = values[pos];
        }
        u64 dec = 0;
        if (!is_null) {
            // NB: a dictionary index of 0 yields a value-initialised raw (0) that is STILL run
            // through the decoder (columnar-inl.h:162-178), i.e. base/zigzag apply to raw 0.
            (void)is_default;
            u64 x = raw + base;
            dec = zigzag ? (u64)zigzag_decode64(x) : x;
        }
        out[i - start] = dec;
    }
}

// Null bytemaps, chyt/server/columnar_conversion.cpp:948-999 and columnar.cpp:350-383,603,638.
// mode 0: from bitmap (DecodeBytemapFromBitmap)      1: from dictionary indexes, zero = null
//      2: from RLE + null bitmap over RLE values     3: from RLE + dictionary indexes, zero = null
//      4: all non-null (Values present, no bitmap)   5: all null
void yto_build_null_bytemap(int mode, i64 start, i64 end, const u8* bitmap, const u32* dict_idx,
                            const u64* rle_idx, i64 n_rle, u8* out) {
    for (i64 i = start; i < end; ++i) {
        u8 r = 0;
        switch (mode) {
            case 0: r = get_bit(bitmap, i); break;
            case 1: r = dict_idx[i] == 0; break;
            case 2: r = get_bit(bitmap, translate_rle_index(rle_idx, n_rle, i)); break;
            case 3: r = dict_idx[translate_rle_index(rle_idx, n_rle, i)] == 0; break;
            case 4: r = 0; break;
            default: r = 1; break;
        }
        out[i - start] = r;
    }
}

// DecodeStringOffsets, columnar.cpp:654-684 / columnar-inl.h:20-30: offset_k = avg*k + zigzag32(values[k-1]).
// Emits end-start+1 offsets, rebased so that the first one is 0 (as the reference's consumers get them).
void yto_decode_string_offsets(const u32* enc, u32 avg_length, i64 start, i64 end, u32* out) {
    auto off = [&](i64 k) -> u32 { return k == 0 ? 0u : (u32)(avg_length * (u32)k + (u32)zigzag_decode32(enc[k - 1])); };
    u32 base = off(start);
    for (i64 k = start; k <= end; ++k) out[k - start] = off(k) - base;
}

// DecodeStringPointersAndLengths, columnar.cpp:686-707: sequential restatement (start offsets instead of pointers).
void yto_decode_string_pointers_and_lengths(const u32* enc, u32 avg_length, i64 n, u32* out_start, i32* out_length) {
    i64 start = 0, avg_times_index = 0;
    for (i64 i = 0; i < n; ++i) {
        out_start[i] = (u32)start;
        avg_times_index += avg_length;
        i64 end = avg_times_index + zigzag_decode64((u64)enc[i]);
        out_length[i] = (i32)(end - start);
        start = end;
    }
}

u64 yto_decode_integer_value(u64 value, u64 base, int zigzag) {  // columnar-inl.h:400-409
    value += base;
    return zigzag ? (u64)zigzag_decode64(value) : value;
}

i64 yto_translate_rle_index(const u64* rle, i64 n_rle, i64 index) { return translate_rle_index(rle, n_rle, index); }

i64 yto_count_ones(const u8* bitmap, i64 start, i64 end) {  // columnar.cpp:495 CountOnesInBitmap
    i64 c = 0;
    for (i64 i = start; i < end; ++i) c += get_bit(bitmap, i);
    return c;
}

// ---------------------------------------------------------------------------
// The remaining helpers of yt/yt/client/table_client/columnar.cpp, restated as the sequential run walks the reference
// performs (BuildBitmapFromRleImpl :137-194, BuildBytemapFromRleImpl :196-241): a cursor that moves to the next run
// when the row index reaches the run's threshold.  kind 0: flag = (dictionary index == 0) ("ZeroMeansNull");
// kind 1: flag = bit of a TBitmap.  `rle` == nullptr: value k(i) = i.
// ---------------------------------------------------------------------------
namespace {
struct FlagWalker {
    int kind;
    const void* data;
    const u64* rle;
    i64 n_rle;
    i64 index, run, threshold;
    bool cur;
    bool value_flag(i64 k) const { return kind == 0 ? static_cast<const u32*>(data)[k] == 0 : get_bit(static_cast<const u8*>(data), k); }
    FlagWalker(int kind_, const void* data_, const u64* rle_, i64 n_rle_, i64 start)
        : kind(kind_), data(data_), rle(rle_), n_rle(n_rle_), index(start), run(0), threshold(-1), cur(false) {
        if (rle) run = translate_rle_index(rle, n_rle, start) - 1;  // TranslateRleStartIndex; ++run happens on first use
    }
    bool next() {
        if (!rle) return value_flag(index++);
        if (index >= threshold) {  // columnar.cpp:180-183 / :217-226
            ++run;
            threshold = run + 1 < n_rle ? (i64)rle[run + 1] : INT64_MAX;
            cur = value_flag(run);
        }
        ++index;
        return cur;
    }
};
}  // namespace

// BuildValidityBitmapFrom{,Rle}DictionaryIndexesWithZeroNull :286-348, BuildValidityBitmapFromRleNullBitmap :623-636,
// CopyBitmapRangeToBitmap{,Negated} :60-135,:577-601.  Writes GetBitmapByteSize(end - start) bytes; the unused bits of
// the last byte are zero (:129-133, :318-330).
void yto_build_bitmap_from_flags(int kind, const void* data, const u64* rle, i64 n_rle, i64 start, i64 end, int negate, u8* dst) {
    const i64 bits = end - start;
    for (i64 b = 0; b < (bits + 7) / 8; ++b) dst[b] = 0;
    FlagWalker w(kind, data, rle, n_rle, start);
    for (i64 i = 0; i < bits; ++i)
        if (w.next() != (negate != 0)) dst[i >> 3] |= (u8)(1u << (i & 7));
}

// BuildNullBytemapFrom{,Rle}DictionaryIndexesWithZeroNull :350-382, BuildNullBytemapFromRleNullBitmap :638-652,
// DecodeBytemapFromBitmap :603-621.
void yto_build_bytemap_from_flags(int kind, const void* data, const u64* rle, i64 n_rle, i64 start, i64 end, int negate, u8* dst) {
    FlagWalker w(kind, data, rle, n_rle, start);
    for (i64 i = 0; i < end - start; ++i) dst[i] = (u8)(w.next() != (negate != 0));
}

// CountNullsIn{,Rle}DictionaryIndexesWithZeroNull :454-493, CountOnesInBitmap :495-548 (qword walk: head, middle, tail),
// CountOnesInRleBitmap :550-575: per run, (min(end, threshold) - current) rows when the run's flag is set.
i64 yto_count_flags(int kind, const void* data, const u64* rle, i64 n_rle, i64 start, i64 end) {
    i64 result = 0;
    if (!rle) {
        if (kind == 0) {
            const u32* d = static_cast<const u32*>(data);
            for (i64 i = start; i < end; ++i) result += d[i] == 0;
            return result;
        }
        // CountOnesInBitmap: whole qwords in the middle, masked head and tail.
        if (start == end) return 0;
        const u8* bm = static_cast<const u8*>(data);
        const i64 n_bytes = (end + 7) / 8;
        auto qword = [&](i64 q) { u64 v = 0; for (i64 b = 0; b < 8 && q * 8 + b < n_bytes; ++b) v |= (u64)bm[q * 8 + b] << (8 * b); return v; };
        i64 sq = start >> 6, eq = end >> 6;
        const int sr = (int)(start & 63), er = (int)(end & 63);
        if (sq == eq) return __builtin_popcountll((qword(sq) & ((1ull << er) - 1)) >> sr);
        if (sr) { result += __builtin_popcountll(qword(sq) >> sr); ++sq; }
        for (i64 q = sq; q < eq; ++q) result += __builtin_popcountll(qword(q));
        if (er) result += __builtin_popcountll(qword(eq) & ((1ull << er) - 1));
        return result;
    }
    i64 run = translate_rle_index(rle, n_rle, start), current = start;
    FlagWalker w(kind, data, nullptr, 0, 0);
    while (current < end) {
        const i64 threshold = run + 1 < n_rle ? (i64)rle[run + 1] : INT64_MAX;
        const i64 next = std::min(end, threshold);
        if (w.value_flag(run)) result += next - current;
        current = next;
        ++run;
    }
    return result;
}

// BuildDictionaryIndexesFrom{,Rle}DictionaryIndexesWithZeroNull :384-420 (null becomes 0xFFFFFFFF),
// BuildIotaDictionaryIndexesFromRleIndexes :422-452 (dict == nullptr: the run number counted from the first run touched).
void yto_build_dictionary_indexes(const u32* dict, const u64* rle, i64 n_rle, i64 start, i64 end, u32* dst) {
    if (!rle) {
        for (i64 i = start; i < end; ++i) dst[i - start] = dict[i] - 1;
        return;
    }
    i64 run = translate_rle_index(rle, n_rle, start) - 1, threshold = -1;
    u32 iota = (u32)-1, value = 0;
    for (i64 i = start; i < end; ++i) {
        if (i >= threshold) {
            ++run;
            threshold = run + 1 < n_rle ? std::min((i64)rle[run + 1], end) : end;
            ++iota;
            if (dict) value = dict[run] - 1;
        }
        dst[i - start] = dict ? value : iota;
    }
}

// CountTotalStringLengthInRleDictionaryIndexesWithZeroNull :709-735.
i64 yto_count_total_string_length(const u32* dict, const u64* rle, i64 n_rle, const i32* lengths, i64 start, i64 end) {
    i64 run = translate_rle_index(rle, n_rle, start), current = start, result = 0;
    while (current < end) {
        const i64 threshold = run + 1 < n_rle ? (i64)rle[run + 1] : INT64_MAX;
        const i64 next = std::min(end, threshold);
        const u32 d = dict[run];
        if (d != 0) result += (next - current) * (i64)lengths[d - 1];
        current = next;
        ++run;
    }
    return result;
}

// TranslateRleEndIndex :759-768.
i64 yto_translate_rle_end_index(const u64* rle, i64 n_rle, i64 index) {
    return index == 0 ? 0 : translate_rle_index(rle, n_rle, index - 1) + 1;
}

// ---------------------------------------------------------------------------
// TCHToYTConverter::ConvertColumnToUnversionedValues for simple types, yt/chyt/server/ch_to_yt_converter.cpp:
// TSimpleValueConverter::FillValueRange :131-215 (XX / TZ_XX type table :157-170, String :171-177 over ColumnString's
// offsets-with-terminating-zero layout, Bool :178-186, DateTime64 :187-206), then TNullableConverter :374-386.
// Type codes follow include/ytgpu.h (ytgpu_ch_type).  Returns 0, or 1 = "Cannot convert value to YT boolean",
// 2 = "Cannot convert value to YT timestamp", 3 = unsupported type.
// ---------------------------------------------------------------------------
int yto_ch_column_to_values(int type, const void* data, const u64* offsets, const u8* null_map, i64 adjust, i64 n, Value* out) {
    for (i64 i = 0; i < n; ++i) {
        Value v{};
        v.id = 0;
        switch (type) {
            case 1: v.type = T_INT64; v.data = (u64)(i64) static_cast<const int8_t*>(data)[i]; break;
            case 2: v.type = T_INT64; v.data = (u64)(i64) static_cast<const int16_t*>(data)[i]; break;
            case 3: v.type = T_INT64; v.data = (u64)(i64) static_cast<const i32*>(data)[i]; break;
            case 4: v.type = T_INT64; v.data = (u64) static_cast<const i64*>(data)[i]; break;
            case 5: v.type = T_UINT64; v.data = static_cast<const u8*>(data)[i]; break;
            case 6: v.type = T_UINT64; v.data = static_cast<const u16*>(data)[i]; break;
            case 7: v.type = T_UINT64; v.data = static_cast<const u32*>(data)[i]; break;
            case 8: v.type = T_UINT64; v.data = static_cast<const u64*>(data)[i]; break;
            case 9: { double d = static_cast<const float*>(data)[i]; v.type = T_DOUBLE; std::memcpy(&v.data, &d, 8); break; }
            case 10: v.type = T_DOUBLE; v.data = static_cast<const u64*>(data)[i]; break;
            case 11: {
                const u8 b = static_cast<const u8*>(data)[i];
                if (b > 1) return 1;
                v.type = T_BOOLEAN; v.data = b; break;
            }
            case 12: {  // getDataAt(i) = (chars + offsets[i - 1], sizeAt(i) - 1)
                const u64 begin = i ? offsets[i - 1] : 0;
                v.type = T_STRING; v.data = begin; v.length = (u32)(offsets[i] - begin - 1); break;
            }
            case 13: v.type = T_UINT64; v.data = static_cast<u16>(static_cast<const u16*>(data)[i] + adjust); break;
            case 14: v.type = T_INT64; v.data = (u64)(i64) static_cast<i32>(static_cast<const i32*>(data)[i] + adjust); break;
            case 15: v.type = T_UINT64; v.data = static_cast<u32>(static_cast<const u32*>(data)[i] + adjust); break;
            case 16: v.type = T_INT64; v.data = (u64)(static_cast<const i64*>(data)[i] + adjust); break;
            case 17: {
                const i64 t = static_cast<const i64*>(data)[i] + adjust;
                if (t < 0) return 2;
                v.type = T_UINT64; v.data = (u64)t; break;
            }
            default: return 3;
        }
        out[i] = v;
    }
    if (null_map)
        for (i64 i = 0; i < n; ++i)
            if (null_map[i]) { Value v{}; v.type = T_NULL; out[i] = v; }
    return 0;
}

// ---------------------------------------------------------------------------
// ConvertStringLikeYTColumnToCHColumn, yt/chyt/server/columnar_conversion.cpp:429-648: the rows of a string column
// (direct / dictionary / RLE / both; DecodeRawVector -> DecodeVectorRleImpl / DecodeVectorDirectImpl,
// client/table_client/columnar-inl.h:66-130,147-181) appended to ColumnString's chars, each followed by '\0'
// (uncheckedConsumer :485-492), offsets[i] = end of value i.  A zero dictionary index yields the empty pair
// (:90-92,:163-165); with a filter hint rejected rows are appended as empty strings (:532-540).
// out_chars == nullptr: only the size is computed.  Returns the chars size.
// ---------------------------------------------------------------------------
i64 yto_string_column_to_ch(const u32* offsets, u32 avg, const u8* chars, const u32* dict, const u64* rle, i64 n_rle,
                            i64 start, i64 count, const u8* filter, u8* out_chars, u64* out_offsets) {
    auto range = [&](i64 index, i64* b, i64* e) {  // DecodeStringRange, columnar-inl.h:31-50
        if (index == 0) { *b = 0; *e = (i64)avg + zigzag_decode64(offsets[0]); return; }
        const u32 base = avg * (u32)index;
        *b = (i64)base + zigzag_decode64(offsets[index - 1]);
        *e = (i64)base + (i64)avg + zigzag_decode64(offsets[index]);
    };
    i64 position = 0;
    i64 run = rle ? translate_rle_index(rle, n_rle, start) : 0, threshold = -1;
    i64 cur_b = 0, cur_e = 0;
    auto fetch = [&](i64 v) {  // the value behind entry v of the index vector
        cur_b = cur_e = 0;
        if (dict) {
            if (dict[v] != 0) range(dict[v] - 1, &cur_b, &cur_e);
        } else {
            range(v, &cur_b, &cur_e);
        }
    };
    for (i64 i = 0; i < count; ++i) {
        const i64 row = start + i;
        if (rle) {
            if (row >= threshold) {
                fetch(run);
                ++run;
                threshold = run < n_rle ? (i64)rle[run] : INT64_MAX;
            }
        } else {
            fetch(row);
        }
        const i64 length = (filter && !filter[i]) ? 0 : cur_e - cur_b;
        if (out_chars) {
            std::memcpy(out_chars + position, chars + cur_b, (size_t)length);
            out_chars[position + length] = 0;
        }
        position += length + 1;
        if (out_offsets) out_offsets[i] = (u64)position;
    }
    return position;
}

// ---------------------------------------------------------------------------
// GROUP BY key -> SUM(val), COUNT(*)  on decoded columns.
// style 0 = YT QL (registry.cpp:1783-1834 InsertGroupRow, udf/sum.c:12-36): row at a time into a hash
//           set, Null-skipping sum that starts Null, groups emitted in FIRST-SEEN order.
// style 1 = ClickHouse key64 (Aggregator.cpp:1006, AggregateFunctionSum.h:51-103): same results as a
//           set; emitted sorted by (key_null, key) because CH's order is hash-table order (unspecified).
// val_type: 0 = int64 (wrapping), 1 = uint64 (wrapping), 2 = double (plain adds in arrival order).
// A NULL key is its own group.  filter (bytemap, may be null): rows with 0 are dropped before grouping.
// Outputs sized for n groups by the caller; *ngroups receives the count.
// threads > 1 (style 1 only): per-thread tables over row slices merged at the end (CH two-level shape).
// ---------------------------------------------------------------------------
struct Agg { u64 sum_bits; u64 count; u8 has; };

static inline void agg_add(Agg& a, int val_type, u64 vbits, bool vnull) {
    a.count++;
    if (vnull) return;
    if (val_type == 2) {
        double s = a.has ? as_double(a.sum_bits) : 0.0;
        s += as_double(vbits);
        std::memcpy(&a.sum_bits, &s, 8);
    } else {
        a.sum_bits = (a.has ? a.sum_bits : 0) + vbits;
    }
    a.has = 1;
}
static inline void agg_merge(Agg& a, const Agg& b, int val_type) {
    a.count += b.count;
    if (!b.has) return;
    if (val_type == 2) {
        double s = (a.has ? as_double(a.sum_bits) : 0.0) + as_double(b.sum_bits);
        std::memcpy(&a.sum_bits, &s, 8);
    } else {
        a.sum_bits = (a.has ? a.sum_bits : 0) + b.sum_bits;
    }
    a.has = 1;
}

int yto_groupby_sum_count(const u64* keys, const u8* key_null, const u64* vals, const u8* val_null,
                          const u8* filter, size_t n, int val_type, int style, int threads,
                          u64* out_keys, u8* out_key_null, u64* out_sum, u8* out_sum_null, u64* out_count,
                          size_t* ngroups, double* seconds) {
    double t0 = now_s();
    struct Table {
        std::unordered_map<u64, u32> map;
        std::vector<u64> k;
        std::vector<Agg> a;
        i64 null_slot = -1;
    };
    // bucket < 0: take every row of [lo, hi); else only rows whose key hashes to `bucket` of `nbuckets`
    // (NULL keys belong to bucket 0).
    auto run = [&](Table& t, size_t lo, size_t hi, int bucket, int nbuckets) {
        t.map.reserve(1024);
        for (size_t i = lo; i < hi; ++i) {
            if (filter && !filter[i]) continue;
            bool kn = key_null && key_null[i];
            if (bucket >= 0) {
                int b = kn ? 0 : (int)((keys[i] * 0x9E3779B97F4A7C15ull >> 40) % (u64)nbuckets);
                if (b != bucket) continue;
            }
            u32 slot;
            if (kn) {
                if (t.null_slot < 0) { t.null_slot = (i64)t.k.size(); t.k.push_back(0); t.a.push_back({0, 0, 0}); }
                slot = (u32)t.null_slot;
            } else {
                auto it = t.map.find(keys[i]);
                if (it == t.map.end()) {
                    slot = (u32)t.k.size();
                    t.map.emplace(keys[i], slot);
                    t.k.push_back(keys[i]);
                    t.a.push_back({0, 0, 0});
                } else slot = it->second;
            }
            agg_add(t.a[slot], val_type, vals[i], val_null && val_null[i]);
        }
    };
    Table total;
    if (style == 2 && threads > 1) {
        // ClickHouse two-level aggregation (contrib/clickhouse/src/Interpreters/Aggregator.cpp:1486 convertToTwoLevel,
        // AggregatedDataVariants.h:64 key64_two_level; TwoLevelHashTable.h: 256 buckets selected by the top hash byte):
        // every thread aggregates ITS slice of the rows into 256 open-addressing tables, then bucket b of all threads is
        // merged by one thread (mergeBlocks per bucket, in parallel).  Each row is read once.
        struct Flat {
            std::vector<u64> k;
            std::vector<Agg> a;
            std::vector<u8> used;
            size_t size = 0, mask = 0;
            void grow() {
                size_t cap = mask ? (mask + 1) * 2 : 256;
                std::vector<u64> ok;
                std::vector<Agg> oa;
                std::vector<u8> ou;
                ok.swap(k); oa.swap(a); ou.swap(used);
                k.assign(cap, 0); a.assign(cap, Agg{0, 0, 0}); used.assign(cap, 0);
                mask = cap - 1;
                for (size_t i = 0; i < ou.size(); ++i)
                    if (ou[i]) { size_t h = slot_of(ok[i]); k[h] = ok[i]; a[h] = oa[i]; used[h] = 1; }
            }
            size_t slot_of(u64 key) const {
                size_t h = (size_t)((key * 0x9E3779B97F4A7C15ull) >> 8) & mask;
                while (used[h] && k[h] != key) h = (h + 1) & mask;
                return h;
            }
            Agg& at(u64 key) {
                if ((size + 1) * 2 > mask + 1) grow();
                size_t h = slot_of(key);
                if (!used[h]) { used[h] = 1; k[h] = key; ++size; }
                return a[h];
            }
        };
        constexpr int B = 256;
        struct Local { Flat b[B]; Agg null_agg{0, 0, 0}; bool has_null = false; };
        std::vector<Local> locals(threads);
        std::vector<std::thread> th;
        for (int q = 0; q < threads; ++q)
            th.emplace_back([&, q] {
                Local& L = locals[q];
                size_t lo = n * (size_t)q / threads, hi = n * (size_t)(q + 1) / threads;
                for (size_t i = lo; i < hi; ++i) {
                    if (filter && !filter[i]) continue;
                    if (key_null && key_null[i]) { L.has_null = true; agg_add(L.null_agg, val_type, vals[i], val_null && val_null[i]); continue; }
                    u64 key = keys[i];
                    agg_add(L.b[(key * 0x9E3779B97F4A7C15ull) >> 56].at(key), val_type, vals[i], val_null && val_null[i]);
                }
            });
        for (auto& x : th) x.join();
        th.clear();
        std::vector<Flat> merged(B);
        for (int q = 0; q < threads; ++q)
            th.emplace_back([&, q] {
                for (int b = q; b < B; b += threads)
                    for (int t = 0; t < threads; ++t) {
                        Flat& f = locals[t].b[b];
                        for (size_t i = 0; i < f.used.size(); ++i)
                            if (f.used[i]) agg_merge(merged[b].at(f.k[i]), f.a[i], val_type);
                    }
            });
        for (auto& x : th) x.join();
        Agg null_total{0, 0, 0};
        bool any_null = false;
        for (auto& L : locals)
            if (L.has_null) { any_null = true; agg_merge(null_total, L.null_agg, val_type); }
        if (seconds) *seconds = now_s() - t0;
        for (auto& f : merged)
            for (size_t i = 0; i < f.used.size(); ++i)
                if (f.used[i]) { total.k.push_back(f.k[i]); total.a.push_back(f.a[i]); }
        if (any_null) { total.null_slot = (i64)total.k.size(); total.k.push_back(0); total.a.push_back(null_total); }
        style = 1;  // emit ordered by (key_null, key) like the other CH flavour
        seconds = nullptr;
    } else if (threads <= 1 || style == 0) {
        run(total, 0, n, -1, 1);
    } else {
        // Hash-partitioned aggregation: thread q owns hash bucket q (ClickHouse's two-level tables bucket by
        // hash as well), scans the key column and aggregates only its keys, so no merge step is needed and
        // every thread's table holds ~groups/threads entries.  Rows of one key keep their arrival order.
        std::vector<Table> parts(threads);
        std::vector<std::thread> th;
        for (int q = 0; q < threads; ++q) th.emplace_back([&, q] { run(parts[q], 0, n, q, threads); });
        for (auto& x : th) x.join();
        for (auto& m : parts) {
            if (m.null_slot >= 0) total.null_slot = (i64)total.k.size() + m.null_slot;
            total.k.insert(total.k.end(), m.k.begin(), m.k.end());
            total.a.insert(total.a.end(), m.a.begin(), m.a.end());
        }
    }
    if (seconds) *seconds = now_s() - t0;  // the emission order below is the oracle's convenience, not timed
    size_t g = total.k.size();
    std::vector<u32> order(g);
    std::iota(order.begin(), order.end(), 0u);
    if (style == 1) {
        std::sort(order.begin(), order.end(), [&](u32 a, u32 b) {
            bool an = (i64)a == total.null_slot, bn = (i64)b == total.null_slot;
            if (an != bn) return bn;  // non-null first
            return total.k[a] < total.k[b];
        });
    }
    for (size_t i = 0; i < g; ++i) {
        u32 s = order[i];
        out_keys[i] = total.k[s];
        out_key_null[i] = (i64)s == total.null_slot;
        out_sum[i] = total.a[s].has ? total.a[s].sum_bits : 0;
        out_sum_null[i] = !total.a[s].has;
        out_count[i] = total.a[s].count;
    }
    *ngroups = g;
    return ERR_OK;
}

// ---------------------------------------------------------------------------
// Horizontal (schemaless) block codec.
//   writer: THorizontalBlockWriter::WriteRow/FlushBlock  yt/yt/ytlib/table_client/schemaless_block_writer.cpp:40-86
//           WriteRowValue                                 yt/yt/client/table_client/unversioned_row.cpp:159-206
//   reader: THorizontalBlockReader::JumpToRowIndex/GetRow yt/yt/ytlib/table_client/schemaless_block_reader.cpp:187-246,323-349
//           ReadRowValue                                  unversioned_row.cpp:208-280
//   varints: library/cpp/yt/coding/varint-inl.h (LEB128), zig_zag-inl.h (Int64 payloads are zig-zag varints)
// block = ui32 offsets[row_count] ++ rows; row = varuint32 value_count, then per value:
//   varuint32 id, varuint32 type, payload (Int64: zigzag varint, Uint64: varint, Double: 8 raw bytes,
//   Boolean: 1 byte, String/Any: varuint32 length + bytes; Composite is written as Any).
// ---------------------------------------------------------------------------
static inline size_t put_varuint(u8* out, u64 v) {
    size_t n = 0;
    while (v >= 0x80) { out[n++] = (u8)(v | 0x80); v >>= 7; }
    out[n++] = (u8)v;
    return n;
}
static inline size_t get_varuint(const u8* in, const u8* end, u64* v) {
    u64 r = 0;
    int shift = 0;
    size_t n = 0;
    while (in + n < end) {
        u8 b = in[n++];
        r |= (u64)(b & 0x7f) << shift;
        if (!(b & 0x80)) { *v = r; return n; }
        shift += 7;
        if (shift > 63) return 0;
    }
    return 0;
}
static inline u64 zigzag_encode64(i64 n) { return ((u64)n << 1) ^ (u64)(n >> 63); }

u64 yto_varuint_encode(u64 v, u8* out) { return put_varuint(out, v); }
u64 yto_zigzag_encode64(i64 v) { return zigzag_encode64(v); }

// row_value_counts (nullable): values of row r actually written, clamped to ncols as the device encoder does.
// Returns bytes written or 0 when `cap` is too small.
u64 yto_block_encode(const Value* v, const char* heap, size_t nrows, u32 ncols, const u32* row_value_counts,
                     u8* out, u64 cap) {
    std::vector<u8> data;
    std::vector<u32> offsets(nrows);
    u8 tmp[16];
    auto put = [&](u64 x) { size_t n = put_varuint(tmp, x); data.insert(data.end(), tmp, tmp + n); };
    for (size_t r = 0; r < nrows; ++r) {
        offsets[r] = (u32)data.size();
        u32 cnt = row_value_counts ? std::min(row_value_counts[r], ncols) : ncols;
        put(cnt);
        for (u32 c = 0; c < cnt; ++c) {
            const Value& x = v[r * ncols + c];
            u8 type = x.type == T_COMPOSITE ? (u8)T_ANY : x.type;
            put(x.id);
            put(type);
            switch (type) {
                case T_INT64: put(zigzag_encode64((i64)x.data)); break;
                case T_UINT64: put(x.data); break;
                case T_DOUBLE: { u8 b[8]; std::memcpy(b, &x.data, 8); data.insert(data.end(), b, b + 8); break; }
                case T_BOOLEAN: data.push_back((x.data & 0xff) ? 1 : 0); break;
                case T_STRING:
                case T_ANY:
                    put(x.length);
                    data.insert(data.end(), (const u8*)heap + x.data, (const u8*)heap + x.data + x.length);
                    break;
                default: break;  // Null / Min / Max / TheBottom: no payload
            }
        }
    }
    u64 total = nrows * 4 + data.size();
    if (total > cap) return 0;
    std::memcpy(out, offsets.data(), nrows * 4);
    if (!data.empty()) std::memcpy(out + nrows * 4, data.data(), data.size());
    return total;
}

// Decodes the first `value_count` values of every row (short rows padded with Null, id 0xffff); string
// `data` fields are byte offsets INTO THE BLOCK.  Returns 0 or an error code (20 = malformed block).
int yto_block_decode(const u8* block, u64 block_bytes, u32 nrows, u32 value_count, Value* out, u32* out_counts) {
    if ((u64)nrows * 4 > block_bytes) return 20;
    const u8* data = block + (u64)nrows * 4;
    const u8* end = block + block_bytes;
    for (u32 r = 0; r < nrows; ++r) {
        u32 off;
        std::memcpy(&off, block + (u64)r * 4, 4);
        const u8* p = data + off;
        if (p >= end) return 20;
        u64 cnt;
        size_t n = get_varuint(p, end, &cnt);
        if (!n) return 20;
        p += n;
        if (out_counts) out_counts[r] = (u32)cnt;
        for (u32 c = 0; c < value_count; ++c) {
            Value& o = out[(size_t)r * value_count + c];
            if (c >= cnt) { o = Value{0xffff, T_NULL, 0, 0, 0}; continue; }
            u64 id, type;
            if (!(n = get_varuint(p, end, &id))) return 20;
            p += n;
            if (!(n = get_varuint(p, end, &type)) || type > 0xff) return 20;
            p += n;
            o = Value{(u16)id, (u8)type, 0, 0, 0};
            switch ((u8)type) {
                case T_INT64: { u64 z; if (!(n = get_varuint(p, end, &z))) return 20; p += n; o.data = (u64)zigzag_decode64(z); break; }
                case T_UINT64: { u64 z; if (!(n = get_varuint(p, end, &z))) return 20; p += n; o.data = z; break; }
                case T_DOUBLE: if (p + 8 > end) return 20; std::memcpy(&o.data, p, 8); p += 8; break;
                case T_BOOLEAN: if (p + 1 > end) return 20; o.data = (*p == 1); p += 1; break;
                case T_STRING:
                case T_ANY:
                case T_COMPOSITE: {
                    u64 len;
                    if (!(n = get_varuint(p, end, &len))) return 20;
                    p += n;
                    if (len >= (1ull << 32) || len > (u64)(end - p)) return 20;  // p + len wraps for a length near 2^64
                    o.length = (u32)len;
                    o.data = (u64)(p - block);
                    p += len;
                    break;
                }
                case T_NULL: case T_MIN: case T_MAX: case T_BOTTOM: break;
                default: return 20;  // ThrowUnexpectedValueType
            }
        }
    }
    return 0;
}

// ---------------------------------------------------------------------------
// BuildPartitionKeysFromSamples, yt/yt/server/controller_agent/helpers.cpp:263-425 (ascending/descending key
// columns, no computed columns).  samples: nsamples rows of ncols key values.  Outputs (capacity
// partition_count - 1): the ORIGINAL index of the sample whose key is the lower bound, its inclusiveness and
// the maniac flag.  Returns the number of partition keys.
// ---------------------------------------------------------------------------
int yto_build_partition_keys(const Value* v, const char* heap, u32 nsamples, u32 ncols, const u8* desc,
                             const i64* weights, const u8* incomplete, int partition_count,
                             u32* out_sample, u8* out_inclusive, u8* out_maniac) {
    if (partition_count <= 1 || nsamples == 0) return 0;
    Comparator cmp{ncols, desc};
    std::vector<u32> order(nsamples);
    std::iota(order.begin(), order.end(), 0u);
    auto key_cmp = [&](u32 a, u32 b) { return cmp.compare_keys(v + (size_t)a * ncols, heap, v + (size_t)b * ncols, heap); };
    // The reference uses std::sort (tie order among equal (key, incomplete) samples unspecified; it only matters
    // through the weights); stable here so that the result is reproducible.
    std::stable_sort(order.begin(), order.end(), [&](u32 a, u32 b) {
        int c = key_cmp(a, b);
        if (c == 0) return incomplete[a] < incomplete[b];
        return c < 0;
    });
    i64 total = 0;
    for (u32 i = 0; i < nsamples; ++i) total += weights[i];
    const double per_partition = (double)total / partition_count;
    std::vector<u32> selected;
    i64 processed = 0;
    for (u32 s : order) {
        processed += weights[s];
        if (processed / per_partition > (double)(selected.size() + 1)) selected.push_back(s);
        if ((int)selected.size() == partition_count - 1) break;
    }
    int nkeys = 0;
    auto equals_last = [&](u32 s) {
        // CompareKeyBounds(inclusive lower bound of s, last lower bound) == 0
        return nkeys > 0 && out_inclusive[nkeys - 1] && key_cmp(s, out_sample[nkeys - 1]) == 0;
    };
    size_t idx = 0;
    while (idx < selected.size()) {
        u32 s = selected[idx];
        if (!equals_last(s)) {
            out_sample[nkeys] = s; out_inclusive[nkeys] = 1; out_maniac[nkeys] = 0; ++nkeys;
            ++idx;
            continue;
        }
        while (idx < selected.size() && equals_last(selected[idx])) ++idx;
        u32 last_maniac = selected[idx - 1];
        if (incomplete[last_maniac]) {
            if (idx >= selected.size()) break;
            out_sample[nkeys] = selected[idx]; out_inclusive[nkeys] = 1; out_maniac[nkeys] = 0; ++nkeys;
            ++idx;
        } else {
            out_maniac[nkeys - 1] = 1;
            out_sample[nkeys] = s; out_inclusive[nkeys] = 0; out_maniac[nkeys] = 0; ++nkeys;
        }
    }
    return nkeys;
}

// ---------------------------------------------------------------------------
// Columnar write side.
// TIntegerColumnConverter<T>::Convert, yt/yt/library/column_converters/integer_column_converter.cpp:69-161: MinValue_
// is initialised to 2^64-1 and never lowered, so every non-null word is (encoded - (2^64-1)) and the base is 2^64-1.
// ---------------------------------------------------------------------------
int yto_convert_integer_column(const Value* v, size_t nrows, u32 ncols, u32 column, u8 value_type, u64* out_values,
                               u8* out_bitmap /* zeroed, 8*ceil(n/64) bytes */, u64* out_base) {
    const u64 base = ~0ull;
    for (size_t r = 0; r < nrows; ++r) {
        const Value& x = v[r * ncols + column];
        if (x.type == T_NULL) {
            out_values[r] = 0;
            out_bitmap[r >> 3] |= (u8)(1u << (r & 7));
            continue;
        }
        if (x.type != value_type) return ERR_UNSUPPORTED_TYPE;
        u64 enc = value_type == T_INT64 ? zigzag_encode64((i64)x.data) : x.data;
        out_values[r] = enc - base;
    }
    *out_base = base;
    return ERR_OK;
}

// TUnversionedIntegerColumnWriter<T>, yt/yt/ytlib/table_chunk_format/integer_column_writer.cpp:318-590 (+ :36-112 the
// shared base): per segment min/max/distinct/run statistics, the four size estimates (:353-381), the first smallest
// in enum order {DictionaryRle, DictionaryDense, DirectRle, DirectDense} wins (:493-496), then the matching Dump*.
struct IntSegment {  // == ytgpu_integer_segment
    u32 type, row_count;
    u64 chunk_row_count, min_value, data_offset, data_bytes, part_bytes[3];
    u32 values_size, ids_size, row_indexes_size;
    u8 values_width, ids_width, row_indexes_width, direct;
};
static_assert(sizeof(IntSegment) == 80, "segment descriptor layout");

static inline u64 packed_bytes(u64 max_value, u64 count) { return 8 * (1 + ((bit_width_of(max_value) * count + 63) >> 6)); }

static u64 emit_packed(const std::vector<u64>& vals, u64 max_value, u8* out, u32* size, u8* width) {
    const u64 bytes = packed_bytes(max_value, vals.size());
    std::vector<u64> words(bytes / 8 + 1, 0);
    yto_bit_pack(vals.data(), vals.size(), max_value, words.data());
    memcpy(out, words.data(), bytes);
    *size = (u32)vals.size();
    *width = (u8)bit_width_of(max_value);
    return bytes;
}

static u64 emit_bitmap(const std::vector<u8>& bits, u8* out) {
    const u64 bytes = 8 * ((bits.size() + 63) / 64);
    memset(out, 0, bytes);
    for (size_t i = 0; i < bits.size(); ++i)
        if (bits[i]) out[i >> 3] |= (u8)(1u << (i & 7));
    return bytes;
}

int yto_encode_integer_column(const u64* raw, const u8* nulls, u64 n, int is_signed, u32 max_values, u64 chunk_row_offset,
                              u8* out, u64 out_capacity, u64* out_bytes, IntSegment* segs, u32 seg_capacity, u32* seg_count) {
    if (max_values == 0) return ERR_BAD_ARGUMENT;
    u64 at = 0;
    u32 ns = 0;
    u64 chunk_rows = chunk_row_offset;
    for (u64 begin = 0; begin < n; begin += max_values) {
        const u64 count = std::min<u64>(max_values, n - begin);
        std::vector<u64> values(count);
        std::vector<u8> isnull(count);
        u64 vmin = ~0ull, vmax = 0, runs = 0;
        std::unordered_map<u64, u64> distinct;  // value -> 1-based first-seen id
        for (u64 i = 0; i < count; ++i) {
            const bool nl = nulls && nulls[begin + i];
            u64 data = 0;
            if (!nl) {
                data = is_signed ? zigzag_encode64((i64)raw[begin + i]) : raw[begin + i];
                vmax = std::max(vmax, data);
                vmin = std::min(vmin, data);
                distinct.emplace(data, distinct.size() + 1);
            }
            if (i == 0 || isnull[i - 1] != (u8)nl || values[i - 1] != data) ++runs;
            values[i] = data;
            isnull[i] = nl;
        }
        chunk_rows += count;
        const u64 range = vmax - vmin;  // wraps to 1 for an all-null segment, as in the reference
        const u64 nd = distinct.size();
        const i32 sizes[4] = {
            (i32)(packed_bytes(range, nd) + packed_bytes(nd + 1, runs) + packed_bytes(chunk_rows, runs)),  // DictionaryRle
            (i32)(packed_bytes(range, nd) + packed_bytes(nd + 1, count)),                                  // DictionaryDense
            (i32)(packed_bytes(range, runs) + packed_bytes(chunk_rows, runs) + runs / 8),                  // DirectRle
            (i32)(packed_bytes(range, count) + count / 8),                                                 // DirectDense
        };
        u32 type = 0;
        for (u32 t = 1; t < 4; ++t)
            if (sizes[t] < sizes[type]) type = t;

        // run starts (both RLE layouts)
        std::vector<u64> run_start;
        if (type == 0 || type == 2) {
            for (u64 i = 0; i < count; ++i)
                if (i == 0 || isnull[i - 1] != isnull[i] || values[i - 1] != values[i]) run_start.push_back(i);
        }
        std::vector<u64> part[3];
        std::vector<u8> bitmap;
        u64 part_max[3] = {0, 0, 0};
        int bitmap_part = -1;
        if (type == 3) {  // DumpDirectValues :66-82
            part[0].resize(count);
            for (u64 i = 0; i < count; ++i) part[0][i] = isnull[i] ? 0 : values[i] - vmin;
            part_max[0] = range;
            bitmap = isnull;
            bitmap_part = 1;
        } else if (type == 1) {  // DumpDictionaryValues :84-112
            std::vector<u64> ids(count);
            for (u64 i = 0; i < count; ++i) {
                if (isnull[i]) continue;
                u64 id = distinct[values[i]];
                if (id > part[0].size()) part[0].push_back(values[i] - vmin);
                ids[i] = id;
            }
            part_max[0] = range;
            part_max[1] = part[0].size() + 1;
            part[1] = ids;
        } else if (type == 2) {  // DumpDirectRleValues :394-435
            for (u64 s : run_start) {
                part[0].push_back(isnull[s] ? 0 : values[s] - vmin);
                bitmap.push_back(isnull[s]);
            }
            part_max[0] = range;
            bitmap_part = 1;
            part[2] = run_start;
            part_max[2] = run_start.back();
        } else {  // DumpDictionaryRleValues :437-489
            for (u64 s : run_start) {
                u64 id = 0;
                if (!isnull[s]) {
                    id = distinct[values[s]];
                    if (id > part[0].size()) part[0].push_back(values[s] - vmin);
                }
                part[1].push_back(id);
            }
            part_max[0] = range;
            part_max[1] = part[0].size() + 1;
            part[2] = run_start;
            part_max[2] = run_start.back();
        }
        IntSegment seg{};
        seg.type = type;
        seg.row_count = (u32)count;
        seg.chunk_row_count = chunk_rows;
        seg.min_value = vmin;
        seg.data_offset = at;
        seg.direct = type >= 2;
        const int nparts = type == 1 || type == 3 ? 2 : 3;
        u64 need = 0;
        for (int p = 0; p < nparts; ++p)
            need += p == bitmap_part ? 8 * ((bitmap.size() + 63) / 64) : packed_bytes(part_max[p], part[p].size());
        if (ns < seg_capacity && at + need <= out_capacity) {
            for (int p = 0; p < nparts; ++p) {
                u64 b;
                if (p == bitmap_part) b = emit_bitmap(bitmap, out + at);
                else if (p == 0) b = emit_packed(part[0], part_max[0], out + at, &seg.values_size, &seg.values_width);
                else if (p == 1) b = emit_packed(part[1], part_max[1], out + at, &seg.ids_size, &seg.ids_width);
                else b = emit_packed(part[2], part_max[2], out + at, &seg.row_indexes_size, &seg.row_indexes_width);
                seg.part_bytes[p] = b;
                at += b;
            }
            seg.data_bytes = need;
            segs[ns] = seg;
        } else {
            at += need;
        }
        ++ns;
    }
    *out_bytes = at;
    *seg_count = ns;
    return (ns <= seg_capacity && at <= out_capacity) ? ERR_OK : ERR_BAD_ARGUMENT;
}

// ---------------------------------------------------------------------------
// YQL block aggregators, combine-all form: one AddMany of TSumBlockAggregator / TAvgBlockAggregator
// (mkql_block_agg_sum.cpp:160-232, 421-485), TMinMaxBlockFixedAggregator (mkql_block_agg_minmax.cpp:697-770, AggLess
// :20-31, InitialStateValue :76-101), count / count_all (mkql_block_agg_count.cpp), each run as its own sequential
// loop exactly as the reference does, over the same Arrow array.
// ---------------------------------------------------------------------------
struct BlockAggState {  // == ytgpu_block_agg_state
    u64 sum, min_value, max_value, count, count_all;
    u8 sum_valid, min_valid, max_valid, value_type;
    u32 reserved;
};

static bool agg_less_bits(u8 type, u64 a, u64 b) {
    if (type == T_UINT64) return a < b;
    if (type == T_INT64) return (i64)a < (i64)b;
    double x = as_double(a), y = as_double(b);
    if (std::isunordered(x, y)) return std::isnan(x) < std::isnan(y);
    return x < y;
}

void yto_block_agg_state_init(BlockAggState* s, u8 type, u8 nullable) {
    std::memset(s, 0, sizeof(*s));
    s->value_type = type;
    if (type == T_DOUBLE) {
        s->min_value = 0x7ff8000000000000ull;
        s->max_value = 0xfff0000000000000ull;
    } else if (type == T_INT64) {
        s->min_value = 0x7fffffffffffffffull;
        s->max_value = 0x8000000000000000ull;
    } else {
        s->min_value = ~0ull;
        s->max_value = 0;
    }
    s->sum_valid = s->min_valid = s->max_valid = nullable ? 0 : 1;
}

int yto_block_combine_all(const u64* values, const u8* validity, i64 offset, i64 length, u8 type, u8 nullable, const u8* filter,
                          BlockAggState* s) {
    const u64* ptr = values + offset;  // GetValues<TIn>(1)
    auto not_null = [&](i64 i) -> u8 {
        if (!validity) return 1;
        u64 full = (u64)(i + offset);
        return (validity[full >> 3] >> (full & 7)) & 1;
    };
    i64 null_count = 0;  // IsNullable ? array->GetNullCount() : 0
    if (nullable) for (i64 i = 0; i < length; ++i) null_count += !not_null(i);
    // count_all: += filtered ? *filtered : batchLength
    u64 passed = 0;
    if (filter) for (i64 i = 0; i < length; ++i) passed += filter[i] ? 1 : 0;
    s->count_all += filter ? passed : (u64)length;
    if (length - null_count == 0) return ERR_OK;
    const bool has_nulls = nullable && null_count != 0;
    // ---- sum ----
    {
        u64 valid_count = 0;
        if (type == T_DOUBLE) {
            double sum = as_double(s->sum);
            for (i64 i = 0; i < length; ++i) {
                u8 sel = (has_nulls ? not_null(i) : 1) & (filter ? (filter[i] ? 1 : 0) : 1);
                sum += sel ? as_double(ptr[i]) : 0.0;
                valid_count += sel;
            }
            std::memcpy(&s->sum, &sum, 8);
        } else {
            u64 sum = s->sum;
            for (i64 i = 0; i < length; ++i) {
                u8 sel = (has_nulls ? not_null(i) : 1) & (filter ? (filter[i] ? 1 : 0) : 1);
                sum += sel ? ptr[i] : 0;
                valid_count += sel;
            }
            s->sum = sum;
        }
        if (nullable) {
            if (!filter) s->sum_valid = 1;
            else if (has_nulls) s->sum_valid |= valid_count ? 1 : 0;
            else s->sum_valid = 1;
        }
        s->count += valid_count;  // TAvgState::Count / the Count aggregator
    }
    // ---- min / max ----
    {
        u64 mn = s->min_value, mx = s->max_value, valid_count = 0;
        for (i64 i = 0; i < length; ++i) {
            u8 sel = (has_nulls ? not_null(i) : 1) & (filter ? (filter[i] ? 1 : 0) : 1);
            if (sel) {
                mn = agg_less_bits(type, mn, ptr[i]) ? mn : ptr[i];
                mx = agg_less_bits(type, ptr[i], mx) ? mx : ptr[i];
            }
            valid_count += sel;
        }
        s->min_value = mn;
        s->max_value = mx;
        if (nullable) {
            u8 raised = !filter ? 1 : (valid_count ? 1 : 0);
            s->min_valid |= raised;
            s->max_valid |= raised;
        }
    }
    return ERR_OK;
}

// ---------------------------------------------------------------------------
// GROUP BY key -> MIN(value), MAX(value), row by row like the reference's per-group states:
//   style 0 (YQL): UpdateMinMax(TMaybe<T>& state, ...) — `!state || AggLess(value, *state)` replaces
//                  (mkql_block_agg_minmax.cpp:20-60; NaN is the biggest value, of equal values the first stays)
//   style 1 (QL):  min_iteration / max_iteration — min replaces when `state >= new`, max when `state < new`
//                  (yt/yt/library/query/engine/udf/min.c:28-62, max.c:28-62; NULL values are skipped, a group without
//                  values stays NULL)
// Output ordered by (key_null, key) like yto_groupby_sum_count; *_null = the aggregate is NULL.
// ---------------------------------------------------------------------------
int yto_groupby_min_max(const u64* keys, const u8* key_null, const u64* vals, const u8* val_null, const u8* filter, size_t n,
                        int val_kind, int style, u64* out_keys, u8* out_key_null, u64* out_min, u64* out_max, u8* out_null,
                        size_t* ngroups) {
    const int val_type = val_kind == 0 ? T_INT64 : val_kind == 1 ? T_UINT64 : T_DOUBLE;  // the VAL_* codes of yto_groupby_sum_count
    struct St { bool has = false; u64 mn = 0, mx = 0; };
    std::map<std::pair<u8, u64>, St> groups;
    auto less_raw = [&](u64 a, u64 b) {
        if (val_type == T_UINT64) return a < b;
        if (val_type == T_INT64) return (i64)a < (i64)b;
        return as_double(a) < as_double(b);
    };
    for (size_t i = 0; i < n; ++i) {
        if (filter && !filter[i]) continue;
        const u8 kn = key_null && key_null[i] ? 1 : 0;
        St& st = groups[{kn, kn ? 0 : keys[i]}];
        if (val_null && val_null[i]) continue;
        const u64 v = vals[i];
        if (!st.has) {
            st.has = true;
            st.mn = st.mx = v;
        } else if (style == 0) {
            if (agg_less_bits((u8)val_type, v, st.mn)) st.mn = v;
            if (agg_less_bits((u8)val_type, st.mx, v)) st.mx = v;
        } else {
            if (!less_raw(st.mn, v)) st.mn = v;   // state >= new (for doubles: !(state < new) differs only with NaN)
            if (less_raw(st.mx, v)) st.mx = v;
        }
    }
    size_t g = 0;
    for (auto& kv : groups) {
        out_keys[g] = kv.first.second;
        out_key_null[g] = kv.first.first;
        out_min[g] = kv.second.has ? kv.second.mn : 0;
        out_max[g] = kv.second.has ? kv.second.mx : 0;
        out_null[g] = kv.second.has ? 0 : 1;
        ++g;
    }
    *ngroups = g;
    return ERR_OK;
}

// ---------------------------------------------------------------------------
// GROUP BY (k1..kK) -> a list of aggregates, YT QL semantics, row at a time in arrival order:
//   groups appear in FIRST-SEEN order (InsertGroupRow appends, registry.cpp:1571-1655);
//   every aggregate state starts Null and an update is skipped when an argument is Null
//   (builtin_function_profiler.cpp:1304-1333 for avg / argmin / argmax; sum.c / min.c / max.c check Null themselves);
//   op 0 sum   (udf/sum.c:12-36: wrapping integer adds, plain double adds)
//   op 1 min, 2 max (udf/min.c:28-62, max.c: min replaces when state >= new, max when state < new)
//   op 3 count of non-null values
//   op 4 avg   = double(sum) / double(count), state (count, sum) (builtin_function_profiler.cpp:1425-1427,1483-1507,1583-1620)
//   op 5 argmin, 6 argmax (arg, by): the state is replaced only when new.by < state.by (resp. >): the first row wins ties
//                 (builtin_function_profiler.cpp:1442-1482)
//   op 7 first = the first non-null value (registry.cpp:3642-3663)
// val_type per value column: EValueType code (int64 / uint64 / double / boolean).
// style: the order of min / max / argmin / argmax, as in yto_groupby_min_max —
//   1 (QL):  the comparisons above on the raw values; next to a NaN both `state >= new` and `state < new` are false, so
//            the result depends on the row order;
//   0 (YQL): AggLess, NaN the biggest value, of equal values the first stays — the order-free total order the GPU kernels
//            implement.
// ---------------------------------------------------------------------------
int yto_groupby_multi(const u64* const* keys, const u8* const* key_null, u32 nk, const u64* const* vals,
                      const u8* const* val_null, const u8* val_type, u32 nv, const i32* agg_op, const i32* agg_col,
                      const i32* agg_by, u32 na, const u8* filter, size_t n, int style, u64* const* out_keys,
                      u8* const* out_key_null, u64* const* out_vals, u8* const* out_val_null, u64* out_counts, u64* out_first,
                      size_t* ngroups) {
    (void)nv;
    struct AggSt { bool has = false; u64 bits = 0; u64 by = 0; u64 count = 0; };
    struct Group { size_t first; u64 count = 0; std::vector<AggSt> st; };
    using Key = std::vector<u64>;  // (null mask, words...)
    std::map<Key, size_t> index;
    std::vector<Group> groups;
    auto less_typed = [style](u8 t, u64 a, u64 b) {
        if (t == T_INT64) return (i64)a < (i64)b;
        if (t == T_DOUBLE) return style == 0 ? agg_less_bits(T_DOUBLE, a, b) : as_double(a) < as_double(b);
        return a < b;  // uint64, boolean
    };
    // min replaces when state >= new (QL), when new < state (YQL: the first of equal values stays)
    auto min_replaces = [&](u8 t, u64 state, u64 v) {
        if (style == 0) return less_typed(t, v, state);
        if (t == T_DOUBLE) return as_double(state) >= as_double(v);
        return !less_typed(t, state, v);
    };
    for (size_t i = 0; i < n; ++i) {
        if (filter && !filter[i]) continue;
        Key key(nk + 1, 0);
        for (u32 k = 0; k < nk; ++k) {
            const bool kn = key_null && key_null[k] && key_null[k][i];
            if (kn) key[0] |= 1ull << k;
            else key[k + 1] = keys[k][i];
        }
        auto it = index.find(key);
        size_t gi;
        if (it == index.end()) {
            gi = groups.size();
            index.emplace(key, gi);
            groups.push_back(Group{i, 0, std::vector<AggSt>(na)});
        } else gi = it->second;
        Group& G = groups[gi];
        G.count++;
        for (u32 a = 0; a < na; ++a) {
            const int c = agg_col[a];
            const bool vn = val_null && val_null[c] && val_null[c][i];
            if (vn) continue;
            const u64 v = vals[c][i];
            const u8 t = val_type[c];
            AggSt& S = G.st[a];
            switch (agg_op[a]) {
                case 0:
                case 4:
                    if (t == T_DOUBLE) {
                        double s = (S.has ? as_double(S.bits) : 0.0) + as_double(v);
                        std::memcpy(&S.bits, &s, 8);
                    } else S.bits = (S.has ? S.bits : 0) + v;
                    S.has = true;
                    S.count++;
                    break;
                case 1:
                    if (!S.has || min_replaces(t, S.bits, v)) S.bits = v;
                    S.has = true;
                    break;
                case 2:
                    if (!S.has || less_typed(t, S.bits, v)) S.bits = v;
                    S.has = true;
                    break;
                case 3:
                    S.count++;
                    S.has = true;
                    break;
                case 5:
                case 6: {
                    const int b = agg_by[a];
                    if (val_null && val_null[b] && val_null[b][i]) break;
                    const u64 bv = vals[b][i];
                    const u8 bt = val_type[b];
                    const bool better = !S.has || (agg_op[a] == 5 ? less_typed(bt, bv, S.by) : less_typed(bt, S.by, bv));
                    if (better) { S.bits = v; S.by = bv; }
                    S.has = true;
                    break;
                }
                case 7:
                    if (!S.has) { S.bits = v; S.has = true; }
                    break;
                default:
                    return ERR_BAD_ARGUMENT;
            }
        }
    }
    for (size_t g = 0; g < groups.size(); ++g) {
        const Group& G = groups[g];
        for (u32 k = 0; k < nk; ++k) {
            const bool kn = key_null && key_null[k] && key_null[k][G.first];
            out_keys[k][g] = kn ? 0 : keys[k][G.first];
            out_key_null[k][g] = kn;
        }
        out_counts[g] = G.count;
        out_first[g] = G.first;
        for (u32 a = 0; a < na; ++a) {
            const AggSt& S = G.st[a];
            u64 bits = S.bits;
            bool nul = !S.has;
            if (agg_op[a] == 3) { bits = S.count; nul = false; }
            if (agg_op[a] == 4 && S.has) {
                const u8 t = val_type[agg_col[a]];
                const double s = t == T_DOUBLE ? as_double(S.bits) : (t == T_INT64 ? (double)(i64)S.bits : (double)S.bits);
                const double r = s / (double)(i64)S.count;
                std::memcpy(&bits, &r, 8);
            }
            out_vals[a][g] = nul ? 0 : bits;
            out_val_null[a][g] = nul;
        }
    }
    *ngroups = groups.size();
    return ERR_OK;
}

// ---------------------------------------------------------------------------
// Unversioned floating-point and boolean column writers, sequential restatement.
//   double:  TUnversionedFloatingPointColumnWriter<double>::AddValues / DumpSegment
//            (yt/yt/ytlib/table_chunk_format/floating_point_column_writer.cpp:213-256): NullBitmap_.Append(is null),
//            Values_.push_back(value.Data.Double) [a Null value carries a zero payload]; data = ui64 count | doubles (:21-31)
//            then the null bitmap.
//   boolean: TUnversionedBooleanColumnWriter::AddValues / DumpSegment (boolean_column_writer.cpp:196-238) with
//            DumpBooleanValues (:18-28): ui64 count, value bitmap (false for NULL), null bitmap.
// A segment is cut every max_values rows.
// ---------------------------------------------------------------------------
struct PlainSegment { u32 row_count, reserved; u64 chunk_row_count, data_offset, data_bytes, part_bytes[3]; };

int yto_encode_plain_column(int is_boolean, const void* values, const u8* nulls, u64 n, u32 max_values, u64 chunk_row_offset,
                            u8* out, u64 out_capacity, u64* out_bytes, PlainSegment* segs, u32 seg_capacity, u32* seg_count) {
    if (max_values == 0) return ERR_BAD_ARGUMENT;
    u64 at = 0;
    u32 ns = 0;
    for (u64 begin = 0; begin < n; begin += max_values) {
        const u64 count = std::min<u64>(max_values, n - begin);
        std::vector<u8> isnull(count), bools(count);
        std::vector<u64> payload(count);
        for (u64 i = 0; i < count; ++i) {
            isnull[i] = nulls && nulls[begin + i];
            if (is_boolean) bools[i] = !isnull[i] && static_cast<const u8*>(values)[begin + i] != 0;
            else payload[i] = isnull[i] ? 0 : static_cast<const u64*>(values)[begin + i];
        }
        const u64 bm = 8 * ((count + 63) / 64);
        const u64 need = is_boolean ? 8 + 2 * bm : 8 + 8 * count + bm;
        if (ns >= seg_capacity || at + need > out_capacity) return ERR_BAD_ARGUMENT;
        PlainSegment& S = segs[ns++];
        S = PlainSegment{};
        S.row_count = (u32)count;
        S.chunk_row_count = chunk_row_offset + begin + count;
        S.data_offset = at;
        std::memcpy(out + at, &count, 8);
        if (is_boolean) {
            S.part_bytes[0] = 8;
            S.part_bytes[1] = emit_bitmap(bools, out + at + 8);
            S.part_bytes[2] = emit_bitmap(isnull, out + at + 8 + bm);
        } else {
            std::memcpy(out + at + 8, payload.data(), 8 * count);
            S.part_bytes[0] = 8 + 8 * count;
            S.part_bytes[1] = emit_bitmap(isnull, out + at + 8 + 8 * count);
        }
        S.data_bytes = need;
        at += need;
    }
    *out_bytes = at;
    *seg_count = ns;
    return ERR_OK;
}

// ---------------------------------------------------------------------------
// TUnversionedStringColumnWriter<String>, sequential restatement (yt/yt/ytlib/table_chunk_format/string_column_writer.cpp):
//   CaptureValue :96-150   a non-null value enters the dictionary on first sight (ids are first-seen, 1-based);
//                          DictionaryByteSize_ / MaxValueLength_ grow with every NEW dictionary entry
//   AddValues :689-705     a run starts where the value differs from the previous one (null == null, :236-250); a segment
//                          ends once it holds max_values values or more than 32 MB of string bytes (:25,:701-703)
//   GetSegmentSize :646-676 the four estimates; the first smallest in enum order {DictionaryRle, DictionaryDense, DirectRle,
//                          DirectDense} wins (:589-593, private.h:32-37)
//   Dump* :152-229,:496-586 data parts; offsets are stored as zig-zag differences from i * expected_length
//                          (PrepareDiffFromExpected, core/misc/bit_packed_unsigned_vector.cpp:11-33)
// Input: value i = heap[starts[i], starts[i] + lengths[i]), nulls (bytemap, may be null).
// Segments are laid out 8-byte aligned in `out` (the reference hands every segment to the block writer on its own).
// ---------------------------------------------------------------------------
struct StrSegment {  // == ytgpu_string_segment
    u32 type, row_count;
    u64 chunk_row_count, data_offset, data_bytes, part_bytes[4];
    u32 expected_length, offsets_size, ids_size, row_indexes_size;
    u8 offsets_width, ids_width, row_indexes_width, direct;
    u32 reserved;
};
static_assert(sizeof(StrSegment) == 88, "string segment descriptor layout");

static inline u32 zigzag_encode32(i32 v) { return ((u32)v << 1) ^ (u32)(v >> 31); }

// PrepareDiffFromExpected: -> (expected, maxDiff), values rewritten in place.
static std::pair<u32, u32> diff_from_expected(std::vector<u64>* values) {
    u32 expected = 0, max_diff = 0;
    if (values->empty()) return {expected, max_diff};
    const int num = (int)(u32)values->back(), den = (int)values->size();
    expected = (u32)(num / den + ((num % den) >= (den + 1) / 2 ? 1 : 0));  // DivRound<int>, numeric_helpers-inl.h:29-33
    i64 expected_value = 0;
    for (size_t i = 0; i < values->size(); ++i) {
        expected_value += expected;
        const i32 diff = (i32)((u32)(*values)[i] - (u32)expected_value);  // ui32 - i64 -> i32 as in the reference
        (*values)[i] = zigzag_encode32(diff);
        max_diff = std::max<u32>(max_diff, (u32)(*values)[i]);
    }
    return {expected, max_diff};
}

int yto_encode_string_column(const u8* heap, const u64* starts, const u32* lengths, const u8* nulls, u64 n, u32 max_values,
                             u64 max_buffer_bytes, u64 chunk_row_offset, u8* out, u64 out_capacity, u64* out_bytes,
                             StrSegment* segs, u32 seg_capacity, u32* seg_count) {
    if (max_values == 0) return ERR_BAD_ARGUMENT;
    u64 at = 0;
    u32 ns = 0;
    u64 begin = 0;
    while (begin < n) {
        // ---- AddValues until the segment is full ----
        std::vector<std::string_view> values;
        std::vector<u8> isnull;
        std::map<std::string_view, u32> dictionary;  // value -> 1-based first-seen id
        std::vector<u64> run_rows;
        u64 direct_bytes = 0, dict_bytes = 0, rle_bytes = 0;
        u32 max_len = 0;
        u64 i = begin;
        for (; i < n; ++i) {
            const bool nl = nulls && nulls[i];
            std::string_view v = nl ? std::string_view() : std::string_view(reinterpret_cast<const char*>(heap + starts[i]), lengths[i]);
            if (!nl) {
                direct_bytes += v.size();
                if (dictionary.emplace(v, (u32)dictionary.size() + 1).second) {
                    dict_bytes += v.size();
                    max_len = std::max<u32>(max_len, (u32)v.size());
                }
            }
            const bool same = !values.empty() && isnull.back() == (u8)nl && (nl || values.back() == v);
            if (!same) {
                rle_bytes += v.size();
                run_rows.push_back(values.size());
            }
            values.push_back(v);
            isnull.push_back(nl);
            if (values.size() >= max_values || direct_bytes > max_buffer_bytes) { ++i; break; }
        }
        const u64 count = values.size(), runs = run_rows.size(), dsize = dictionary.size();
        // ---- GetSegmentSize ----
        const i64 sizes[4] = {
            (i64)(dict_bytes + packed_bytes(max_len, dsize) + packed_bytes(dsize + 1, runs) + packed_bytes(count, runs)),
            (i64)(dict_bytes + packed_bytes(max_len, dsize) + packed_bytes(dsize + 1, count)),
            (i64)(rle_bytes + packed_bytes(max_len, runs) + packed_bytes(count, runs) + count / 8),
            (i64)(direct_bytes + packed_bytes(max_len, count) + count / 8)};
        int type = 0;
        for (int t = 1; t < 4; ++t)
            if ((i32)sizes[t] < (i32)sizes[type]) type = t;  // i32 sizes, std::min_element: the first minimum
        // ---- Dump* into a scratch vector ----
        std::vector<u8> blob(16 * count + direct_bytes + 64 * 4 + 64, 0);
        StrSegment S{};
        S.type = (u32)type;
        S.row_count = (u32)count;
        S.chunk_row_count = chunk_row_offset + begin + count;
        S.direct = (type >= 2);
        u64 o = 0;
        auto put_offsets = [&](std::vector<u64>& offs, int part) {
            auto [expected, max_diff] = diff_from_expected(&offs);
            S.expected_length = expected;
            S.part_bytes[part] = emit_packed(offs, max_diff, blob.data() + o, &S.offsets_size, &S.offsets_width);
            o += S.part_bytes[part];
        };
        // dictionary in first-seen order, ids per value
        std::vector<u64> ids(count, 0);
        std::vector<std::string_view> dict_values;
        if (type == 0 || type == 1) {
            u32 seen = 0;
            for (u64 k = 0; k < count; ++k) {
                if (isnull[k]) continue;
                const u32 id = dictionary.at(values[k]);
                ids[k] = id;
                if (id > seen) { dict_values.push_back(values[k]); ++seen; }
            }
        }
        if (type == 3) {  // DirectDense: offsets | null bitmap | data
            std::vector<u64> offs;
            u64 acc = 0;
            for (u64 k = 0; k < count; ++k) { acc += values[k].size(); offs.push_back(acc); }
            put_offsets(offs, 0);
            S.part_bytes[1] = emit_bitmap(isnull, blob.data() + o);
            o += S.part_bytes[1];
            for (u64 k = 0; k < count; ++k) { memcpy(blob.data() + o, values[k].data(), values[k].size()); o += values[k].size(); }
            S.part_bytes[2] = direct_bytes;
        } else if (type == 1) {  // DictionaryDense: ids (max = dictionary size + 1) | dictionary offsets | dictionary data
            S.part_bytes[0] = emit_packed(ids, dsize + 1, blob.data() + o, &S.ids_size, &S.ids_width);
            o += S.part_bytes[0];
            std::vector<u64> offs;
            u64 acc = 0;
            for (auto v : dict_values) { acc += v.size(); offs.push_back(acc); }
            put_offsets(offs, 1);
            for (auto v : dict_values) { memcpy(blob.data() + o, v.data(), v.size()); o += v.size(); }
            S.part_bytes[2] = dict_bytes;
        } else if (type == 2) {  // DirectRle: row indexes | offsets | null bitmap over runs | data of the runs
            S.part_bytes[0] = emit_packed(run_rows, run_rows.back(), blob.data() + o, &S.row_indexes_size, &S.row_indexes_width);
            o += S.part_bytes[0];
            std::vector<u64> offs;
            std::vector<u8> run_null;
            u64 acc = 0;
            for (u64 r : run_rows) { acc += values[r].size(); offs.push_back(acc); run_null.push_back(isnull[r]); }
            put_offsets(offs, 1);
            S.part_bytes[2] = emit_bitmap(run_null, blob.data() + o);
            o += S.part_bytes[2];
            for (u64 r : run_rows) { memcpy(blob.data() + o, values[r].data(), values[r].size()); o += values[r].size(); }
            S.part_bytes[3] = rle_bytes;
        } else {  // DictionaryRle: row indexes | ids of the runs (max = dictionary size) | dictionary offsets | dictionary data
            S.part_bytes[0] = emit_packed(run_rows, run_rows.back(), blob.data() + o, &S.row_indexes_size, &S.row_indexes_width);
            o += S.part_bytes[0];
            std::vector<u64> run_ids;
            for (u64 r : run_rows) run_ids.push_back(ids[r]);
            S.part_bytes[1] = emit_packed(run_ids, dsize, blob.data() + o, &S.ids_size, &S.ids_width);
            o += S.part_bytes[1];
            std::vector<u64> offs;
            u64 acc = 0;
            for (auto v : dict_values) { acc += v.size(); offs.push_back(acc); }
            put_offsets(offs, 2);
            for (auto v : dict_values) { memcpy(blob.data() + o, v.data(), v.size()); o += v.size(); }
            S.part_bytes[3] = dict_bytes;
        }
        at = (at + 7) & ~7ull;
        if (ns >= seg_capacity || at + o > out_capacity) return ERR_BAD_ARGUMENT;
        S.data_offset = at;
        S.data_bytes = o;
        memcpy(out + at, blob.data(), o);
        at += o;
        segs[ns++] = S;
        begin = i;
    }
    *out_bytes = at;
    *seg_count = ns;
    return ERR_OK;
}

int yto_hardware_threads() { return (int)std::thread::hardware_concurrency(); }

}  // extern "C"
