// partition.cu — batched partitioners and the slab scatter of the shuffle's map side.
//
// Replaces the per-row loop TPartitionMultiChunkWriter::WriteRow -> IPartitioner::GetPartitionIndex
// (yt/yt/ytlib/table_client/schemaless_chunk_writer.cpp:1604-1623; partitioner.cpp:41-57 ordered,
// :84-113 hash, :122-173 column) with one kernel over the whole batch, and the P per-partition block
// writers with a stable scatter into partition-contiguous slabs (one radix pass over the partition
// index + one row gather).  Partition indices are bit-identical to the reference's
// (partitioner.cpp:13-16: the logic must never change between implementations).
#include <vector>

#include "context.cuh"
#include "farmhash.cuh"
#include "keys.cuh"
#include "radix_sort.cuh"
#include "rows.cuh"

using namespace ytgpu;

namespace {

constexpr int kMaxSmemPartitions = 4096;

struct DeviceBounds {
    const u64* words;      // [P][nchunks]
    const u32* nbytes;     // [P] prefix length in normalised bytes (0 = universal)
    const u8* inclusive;   // [P]
    u32 count;
    u32 nchunks;
};

// TComparator::TestKey for a LOWER bound (comparator.cpp:77-103) in normalised-byte space.
__device__ __forceinline__ bool test_key(const u64* key, const DeviceBounds& B, u32 b) {
    const u32 nb = __ldg(B.nbytes + b);
    const u64* w = B.words + (size_t)b * B.nchunks;
    const u32 full = nb >> 3, rem = nb & 7;
    int cmp = 0;
    for (u32 i = 0; i < full; ++i) {
        u64 bw = __ldg(w + i);
        if (key[i] != bw) {
            cmp = key[i] > bw ? 1 : -1;
            break;
        }
    }
    if (cmp == 0 && rem) {
        u64 mask = ~0ull << (8 * (8 - rem));
        u64 kw = key[full] & mask, bw = __ldg(w + full) & mask;
        if (kw != bw) cmp = kw > bw ? 1 : -1;
    }
    return cmp > 0 || (cmp == 0 && __ldg(B.inclusive + b));
}

// std::upper_bound(bounds, key, !TestKey) - 1   (partitioner.cpp:46-56)
__device__ __forceinline__ i32 ordered_index(const u64* key, const DeviceBounds& B) {
    u32 lo = 0, cnt = B.count;
    while (cnt > 0) {
        u32 step = cnt >> 1, mid = lo + step;
        if (test_key(key, B, mid)) {
            lo = mid + 1;
            cnt -= step + 1;
        } else {
            cnt = step;
        }
    }
    return (i32)lo - 1;
}

struct PartParams {
    int kind;
    u32 partition_count;
    KeyLayout layout;        // ordered / fixed-row hash
    DeviceBounds bounds;
    u32 key_column_count;    // hash
    u64 salt_hash;           // FarmHash(salt)
    u16 column_id;           // column
    // inputs
    const ytgpu_value* values;
    u32 value_count;
    const u8* heap;
    const u8* rows;          // fixed rows
    u32 row_bytes;
    u64 n;
    // outputs
    i32* out_index;          // nullable
    u64* out_chunk;          // nullable: partition index as a sort key chunk
    unsigned long long* histogram;  // nullable, [P]
    u32* err_word;
};

__device__ __forceinline__ ytgpu_value load_value(const ytgpu_value* p) {
    uint4 raw = *reinterpret_cast<const uint4*>(p);
    ytgpu_value v;
    v.id = (u16)(raw.x & 0xffff);
    v.type = (u8)((raw.x >> 16) & 0xff);
    v.flags = (u8)(raw.x >> 24);
    v.length = raw.y;
    v.data = ((u64)raw.w << 32) | raw.z;
    return v;
}

template <bool FIXED>
__global__ void __launch_bounds__(256) partition_index_kernel(const PartParams P) {
    extern __shared__ u32 s_hist[];
    const bool smem_hist = P.histogram && P.partition_count <= (u32)kMaxSmemPartitions;
    if (smem_hist) {
        for (u32 i = threadIdx.x; i < P.partition_count; i += blockDim.x) s_hist[i] = 0;
        __syncthreads();
    }
    u32 err = 0;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < P.n; i += (u64)gridDim.x * blockDim.x) {
        i32 idx = 0;
        if (P.kind == YTGPU_PARTITION_ORDERED) {
            u64 words[kMaxKeyChunks];
            ChunkWriter w(words);
            if (FIXED) {
                const u8* row = P.rows + i * P.row_bytes;
                for (u32 c = 0; c < P.layout.ncols; ++c) normalize_fixed(P.layout.col[c], row, w);
            } else {
                const ytgpu_value* row = P.values + i * P.value_count;
                for (u32 c = 0; c < P.layout.ncols; ++c)
                    err |= normalize_value(P.layout.col[c], load_value(row + P.layout.col[c].index), P.heap, w);
            }
            w.finish();
            idx = ordered_index(words, P.bounds);
            if (idx < 0) { err |= DE_PART_OUT_OF_BOUNDS; idx = 0; }
        } else if (P.kind == YTGPU_PARTITION_HASH) {
            u64 h = 0xdeadc0deULL;
            u32 cnt;
            if (FIXED) {
                cnt = min(P.key_column_count, P.layout.ncols);
                const u8* row = P.rows + i * P.row_bytes;
                for (u32 c = 0; c < cnt; ++c) {
                    const KeyColLayout& kc = P.layout.col[c];
                    u64 f;
                    if (kc.type == YTGPU_TYPE_STRING) f = fh::fingerprint_bytes(row + kc.index, kc.width);
                    else if (kc.type == YTGPU_TYPE_BOOLEAN) f = fh::fingerprint_u64(row[kc.index] != 0);
                    else f = fh::fingerprint_u64(fh::load64(row + kc.index));
                    h = fh::fingerprint_u128(h, f);
                }
            } else {
                cnt = min(P.key_column_count, P.value_count);
                const ytgpu_value* row = P.values + i * P.value_count;
                for (u32 c = 0; c < cnt; ++c) {
                    u64 f;
                    err |= fh::value_fingerprint(load_value(row + c), P.heap, &f);
                    h = fh::fingerprint_u128(h, f);
                }
            }
            h ^= (u64)cnt;
            if (P.salt_hash != 0) h = fh::fingerprint_u64(h ^ P.salt_hash);
            idx = (i32)(h % (u64)P.partition_count);
        } else {  // column based (rowset only)
            const ytgpu_value* row = P.values + i * P.value_count;
            bool found = false;
            for (u32 c = 0; c < P.value_count && !found; ++c) {
                ytgpu_value v = load_value(row + c);
                if (v.id != P.column_id) continue;
                found = true;
                if (v.type != YTGPU_TYPE_UINT64 && v.type != YTGPU_TYPE_INT64) err |= DE_PART_BAD_TYPE;
                else if (v.type == YTGPU_TYPE_INT64 && (i64)v.data < 0) err |= DE_PART_NEGATIVE;
                else if (v.data >= (u64)P.partition_count) err |= DE_PART_OUT_OF_BOUNDS;
                else idx = (i32)v.data;
            }
            if (!found) err |= DE_PART_NO_COLUMN;
        }
        if (P.out_index) P.out_index[i] = idx;
        if (P.out_chunk) P.out_chunk[i] = (u64)(u32)idx;
        if (P.histogram) {
            if (smem_hist) atomicAdd(&s_hist[idx], 1u);
            else atomicAdd(&P.histogram[idx], 1ull);
        }
    }
    if (err) atomicOr(P.err_word, err);
    if (smem_hist) {
        __syncthreads();
        for (u32 i = threadIdx.x; i < P.partition_count; i += blockDim.x) {
            u32 c = s_hist[i];
            if (c) atomicAdd(&P.histogram[i], (unsigned long long)c);
        }
    }
}

// ---- ordered partitioner over the width-free key words of keys.cuh (rowset keys whose fixed-width normalised form
// does not fit in kMaxKeyChunks chunks) ----
// Bound b compares its first plen[b] key columns; column c of it is the E_c words of the bound's value, at
// words[col_off[b * (ncols + 1) + c] .. col_off[b * (ncols + 1) + c + 1]).  The key's words are computed from its values
// and the heap as the probes need them: no per-row key is stored.
struct WordBounds {
    const u64* words;
    const u64* col_off;   // [P][ncols + 1]
    const u32* plen;      // [P] effective prefix length in columns
    const u8* inclusive;  // [P] effective inclusiveness
    u32 count;
};

constexpr u32 kHeadWords = 4;

// Key column 0 and its first kHeadWords words, kept in registers: every probe of the binary search starts there.
struct KeyHead {
    ytgpu_value v0;
    u32 n0;  // words of E_0
    u64 w[kHeadWords];
};

__host__ __device__ __forceinline__ ytgpu_value key_load(const ytgpu_value* p) {
#ifdef __CUDA_ARCH__
    return load_value(p);
#else
    return *p;
#endif
}

__host__ __device__ __forceinline__ KeyHead key_head(const KeyLayout& L, const ytgpu_value* row, const u8* heap) {
    KeyHead h;
    const KeyColLayout& k = L.col[0];
    h.v0 = key_load(row + k.index);
    h.n0 = key_col_words(k, h.v0);
#pragma unroll
    for (u32 w = 0; w < kHeadWords; ++w) h.w[w] = w < h.n0 ? key_col_word(k, h.v0, heap, w) : 0;
    return h;
}

// Sign of (key - bound b) over the bound's effective prefix, column by column and word by word: TComparator::TestKey
// (comparator.cpp:77-103) before the bound's inclusiveness is applied.
__host__ __device__ __forceinline__ int compare_key_bound(const KeyLayout& L, const ytgpu_value* row, const u8* heap,
                                                          const KeyHead& h, const WordBounds& B, u32 b) {
    const u64* off = B.col_off + (u64)b * (L.ncols + 1);
    const u32 plen = B.plen[b];
    for (u32 c = 0; c < plen; ++c) {
        const KeyColLayout& k = L.col[c];
        const ytgpu_value v = c == 0 ? h.v0 : key_load(row + k.index);
        const u32 nk = c == 0 ? h.n0 : key_col_words(k, v);
        const u64* bw = B.words + off[c];
        const u32 nb = (u32)(off[c + 1] - off[c]);
        const u32 nw = nk < nb ? nk : nb;
        u32 w = 0;
        if (c == 0) {
#pragma unroll
            for (u32 i = 0; i < kHeadWords; ++i)
                if (i < nw && h.w[i] != bw[i]) return h.w[i] < bw[i] ? -1 : 1;
            w = kHeadWords;
        }
        for (; w < nw; ++w) {
            const u64 kw = key_col_word(k, v, heap, w), x = bw[w];
            if (kw != x) return kw < x ? -1 : 1;
        }
        if (nk != nb) return nk < nb ? -1 : 1;  // E_c is prefix-free: equal words up to here mean equal lengths
    }
    return 0;
}

// std::upper_bound(bounds, key, !TestKey) - 1   (partitioner.cpp:46-56), over key words.
__host__ __device__ __forceinline__ i32 ordered_index_words(const KeyLayout& L, const ytgpu_value* row, const u8* heap,
                                                            const WordBounds& B) {
    const KeyHead h = key_head(L, row, heap);
    u32 lo = 0, cnt = B.count;
    while (cnt > 0) {
        const u32 step = cnt >> 1, mid = lo + step;
        const int cmp = compare_key_bound(L, row, heap, h, B, mid);
        if (cmp > 0 || (cmp == 0 && B.inclusive[mid])) {
            lo = mid + 1;
            cnt -= step + 1;
        } else {
            cnt = step;
        }
    }
    return (i32)lo - 1;
}

// The same outputs and error bits as partition_index_kernel<false> for YTGPU_PARTITION_ORDERED.
__global__ void __launch_bounds__(256) partition_words_kernel(const PartParams P, const WordBounds B) {
    extern __shared__ u32 s_hist[];
    const bool smem_hist = P.histogram && P.partition_count <= (u32)kMaxSmemPartitions;
    if (smem_hist) {
        for (u32 i = threadIdx.x; i < P.partition_count; i += blockDim.x) s_hist[i] = 0;
        __syncthreads();
    }
    u32 err = 0;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < P.n; i += (u64)gridDim.x * blockDim.x) {
        const ytgpu_value* row = P.values + i * P.value_count;
        for (u32 c = 0; c < P.layout.ncols; ++c) err |= key_value_errors(P.layout.col[c], load_value(row + P.layout.col[c].index));
        i32 idx = ordered_index_words(P.layout, row, P.heap, B);
        if (idx < 0) { err |= DE_PART_OUT_OF_BOUNDS; idx = 0; }
        if (P.out_index) P.out_index[i] = idx;
        if (P.out_chunk) P.out_chunk[i] = (u64)(u32)idx;
        if (P.histogram) {
            if (smem_hist) atomicAdd(&s_hist[idx], 1u);
            else atomicAdd(&P.histogram[idx], 1ull);
        }
    }
    if (err) atomicOr(P.err_word, err);
    if (smem_hist) {
        __syncthreads();
        for (u32 i = threadIdx.x; i < P.partition_count; i += blockDim.x) {
            u32 c = s_hist[i];
            if (c) atomicAdd(&P.histogram[i], (unsigned long long)c);
        }
    }
}

// ---- host side: lower bounds -> normalised bytes (same encoding as the keys) ----
struct HostBounds {
    std::vector<u64> words;
    std::vector<u32> nbytes;
    std::vector<u8> inclusive;
};

void pack_be(const std::vector<u8>& bytes, u64* out, u32 nchunks) {
    for (u32 c = 0; c < nchunks; ++c) {
        u64 w = 0;
        for (u32 b = 0; b < 8; ++b) {
            size_t i = (size_t)c * 8 + b;
            w = (w << 8) | (i < bytes.size() ? bytes[i] : 0);
        }
        out[c] = w;
    }
}

Status normalize_bounds(const ytgpu_partition_spec* spec, const KeyLayout& L, HostBounds* hb) {
    const u32 P = (u32)spec->partition_count;
    hb->words.assign((size_t)P * L.nchunks, 0);
    hb->nbytes.assign(P, 0);
    hb->inclusive.assign(P, 0);
    for (u32 b = 0; b < P; ++b) {
        u32 plen = spec->bound_prefix_length ? spec->bound_prefix_length[b] : 0;
        if (plen > L.ncols || plen > spec->bound_value_count)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "Comparator is used with longer key bound (bound %u has %u values, comparator length %u)", b, plen, L.ncols);
        u32 nb = plen == L.ncols ? L.total_bytes : L.col[plen].byte_offset;
        bool incl = spec->bound_inclusive ? spec->bound_inclusive[b] != 0 : true;
        std::vector<u8> bytes;
        bytes.reserve(nb);
        bool terminated = false;
        auto terminate = [&](int sign_key_vs_bound) {
            // keys equal to the bound so far are all greater (sign>0) or all smaller (sign<0) than it
            bytes.resize(nb, sign_key_vs_bound > 0 ? 0x00 : 0xff);
            incl = sign_key_vs_bound > 0;
            terminated = true;
        };
        for (u32 c = 0; c < plen && !terminated; ++c) {
            const KeyColLayout& kc = L.col[c];
            const ytgpu_value& v = spec->bounds[(size_t)b * spec->bound_value_count + c];
            const int ord = kc.descending ? -1 : 1;
            if (v.type == YTGPU_TYPE_ANY || v.type == YTGPU_TYPE_COMPOSITE)
                return make_status(YTGPU_ERR_UNSUPPORTED, "partition bound %u holds an Any/Composite value", b);
            if (!kc.has_type_byte && v.type != kc.type) {
                terminate(((int)kc.type > (int)v.type ? 1 : -1) * ord);
                break;
            }
            std::vector<u8> colbytes;
            const u8 inv = kc.descending ? 0xff : 0x00;
            auto put = [&](u8 x) { colbytes.push_back((u8)(x ^ inv)); };
            if (kc.has_type_byte) put(v.type);
            bool type_matches = kc.type == 0 || v.type == kc.type;
            u32 payload_done = 0;
            int pending_sign = 0;
            if (type_matches || L.fixed_rows) {
                switch (v.type) {
                    case YTGPU_TYPE_INT64:
                    case YTGPU_TYPE_UINT64:
                    case YTGPU_TYPE_DOUBLE: {
                        u64 x = v.data;
                        if (v.type == YTGPU_TYPE_INT64) x ^= 0x8000000000000000ull;
                        else if (v.type == YTGPU_TYPE_DOUBLE) x = normalize_double_bits(x);
                        if (kc.payload_bytes >= 8) {
                            for (int s = 56; s >= 0; s -= 8) put((u8)(x >> s));
                            payload_done = 8;
                        }
                        break;
                    }
                    case YTGPU_TYPE_BOOLEAN:
                        if (kc.payload_bytes >= 1) { put((v.data & 0xff) != 0); payload_done = 1; }
                        break;
                    case YTGPU_TYPE_STRING: {
                        const u8* s = spec->bounds_heap + v.data;
                        u32 len = v.length;
                        u32 w = kc.width;
                        u32 take = len < w ? len : w;
                        for (u32 i = 0; i < take; ++i) put(s[i]);
                        for (u32 i = take; i < w; ++i) put(0);
                        payload_done = w;
                        if (len > w) {
                            pending_sign = -1 * ord;  // keys equal on W bytes are proper prefixes: key < bound
                        } else if (L.fixed_rows && len < w) {
                            pending_sign = 1 * ord;   // keys are exactly W long: key > shorter bound
                        } else if (!L.fixed_rows) {
                            for (int k = (int)kc.len_bytes - 1; k >= 0; --k) put((u8)(len >> (8 * k)));
                            payload_done += kc.len_bytes;
                        }
                        break;
                    }
                    default:
                        break;
                }
            }
            bytes.insert(bytes.end(), colbytes.begin(), colbytes.end());
            if (pending_sign) {
                terminate(pending_sign);
                break;
            }
            for (u32 i = payload_done; i < kc.payload_bytes; ++i) bytes.push_back(inv);  // zero payload, inverted if desc
        }
        bytes.resize(nb, 0);
        pack_be(bytes, hb->words.data() + (size_t)b * L.nchunks, L.nchunks);
        hb->nbytes[b] = nb;
        hb->inclusive[b] = incl ? 1 : 0;
    }
    return Status{};
}

// ---- host side: lower bounds -> key words (keys.cuh; the encoder the keys use) ----
struct HostWordBounds {
    std::vector<u64> words, col_off;
    std::vector<u32> plen;
    std::vector<u8> inclusive;
    WordBounds view() const { return WordBounds{words.data(), col_off.data(), plen.data(), inclusive.data(), (u32)plen.size()}; }
};

// The rules of normalize_bounds that do not depend on a width.  A bound string needs no width: prefix-free words order
// it against keys of any length.
Status encode_bounds_words(const ytgpu_partition_spec* spec, const KeyLayout& L, HostWordBounds* hb) {
    const u32 P = (u32)spec->partition_count;
    hb->words.clear();
    hb->col_off.clear();
    hb->plen.assign(P, 0);
    hb->inclusive.assign(P, 0);
    for (u32 b = 0; b < P; ++b) {
        u32 plen = spec->bound_prefix_length ? spec->bound_prefix_length[b] : 0;
        if (plen > L.ncols || plen > spec->bound_value_count)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "Comparator is used with longer key bound (bound %u has %u values, comparator length %u)", b, plen, L.ncols);
        bool incl = spec->bound_inclusive ? spec->bound_inclusive[b] != 0 : true;
        u32 eff = plen;
        hb->col_off.push_back(hb->words.size());
        for (u32 c = 0; c < plen; ++c) {
            const KeyColLayout& kc = L.col[c];
            const ytgpu_value& v = spec->bounds[(size_t)b * spec->bound_value_count + c];
            if (v.type == YTGPU_TYPE_ANY || v.type == YTGPU_TYPE_COMPOSITE)
                return make_status(YTGPU_ERR_UNSUPPORTED, "partition bound %u holds an Any/Composite value", b);
            if (!kc.has_type_byte && v.type != kc.type) {
                // every key equal to the bound so far holds the declared type here: type order decides
                eff = c;
                incl = ((int)kc.type > (int)v.type ? 1 : -1) * (kc.descending ? -1 : 1) > 0;
                break;
            }
            for (u32 w = 0, nw = key_col_words(kc, v); w < nw; ++w) hb->words.push_back(key_col_word(kc, v, spec->bounds_heap, w));
            hb->col_off.push_back(hb->words.size());
        }
        hb->col_off.resize((size_t)(b + 1) * (L.ncols + 1), hb->words.size());
        hb->plen[b] = eff;
        hb->inclusive[b] = incl ? 1 : 0;
    }
    if (hb->words.empty()) hb->words.push_back(0);  // every bound universal: keep the upload non-empty
    return Status{};
}

struct PartitionRun {
    DevBuf<u64> bwords;
    DevBuf<u32> bnbytes;     // key-word bounds: effective prefix length in columns
    DevBuf<u8> bincl;
    DevBuf<u64> boff;        // key-word bounds: per-column word offsets
    bool key_words = false;  // the layout does not fit kMaxKeyChunks: partition_words_kernel over `wbounds`
    WordBounds wbounds{};
    DevBuf<unsigned long long> hist;
    OutBuf<i32> index;
    DevBuf<u64> chunk;
};

Status launch_partition(Context* ctx, PartParams& P, bool fixed, const WordBounds* words = nullptr) {
    if (P.n == 0) return Status{};
    KernelTimer t(ctx, KC_PARTITION);
    u32 blocks = (u32)std::min<u64>((P.n + 255) / 256, (u64)kNumSms * 8);
    size_t smem = (P.histogram && P.partition_count <= (u32)kMaxSmemPartitions) ? (size_t)P.partition_count * 4 : 0;
    if (words) partition_words_kernel<<<blocks, 256, smem, ctx->stream>>>(P, *words);
    else if (fixed) partition_index_kernel<true><<<blocks, 256, smem, ctx->stream>>>(P);
    else partition_index_kernel<false><<<blocks, 256, smem, ctx->stream>>>(P);
    YTGPU_CUDA_TRY(cudaGetLastError());
    return Status{};
}

Status prepare_params(Context* ctx, const ytgpu_partition_spec* spec, bool fixed, u32 value_count,
                      const ytgpu_value* vals_dev, u64 n, PartParams* P, PartitionRun* run) {
    if (!spec) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null partition spec");
    if (spec->partition_count <= 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "partition_count must be positive");
    *P = PartParams{};
    P->kind = spec->kind;
    P->partition_count = (u32)spec->partition_count;
    P->err_word = ctx->dev_err;
    if (spec->kind == YTGPU_PARTITION_ORDERED) {
        std::vector<ytgpu_key_column> cols(spec->key.columns, spec->key.columns + spec->key.column_count);
        if (!fixed) {
            bool need = false;
            for (auto& k : cols) {
                if (k.index >= value_count) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key column index out of range");
                if ((k.type == YTGPU_TYPE_STRING || k.type == 0) && k.width == 0) need = true;
            }
            if (need) {
                u32 mx[kMaxKeyColumns];
                ytgpu_sort_spec tmp{cols.data(), (u32)cols.size()};
                YTGPU_TRY(measure_string_widths(ctx, &tmp, vals_dev, value_count, n, mx));
                for (size_t c = 0; c < cols.size(); ++c)
                    if ((cols[c].type == YTGPU_TYPE_STRING || cols[c].type == 0) && cols[c].width == 0) cols[c].width = mx[c];
            }
        }
        ytgpu_sort_spec ks{cols.data(), (u32)cols.size()};
        const Status s = build_key_layout(&ks, fixed, false, &P->layout);
        run->key_words = !fixed && s.code == YTGPU_ERR_UNSUPPORTED && P->layout.nchunks > (u32)kMaxKeyChunks;
        if (!run->key_words) YTGPU_TRY(s);
        if (!spec->bounds && spec->partition_count > 1)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "ordered partitioner needs bounds");
        if (run->key_words) {
            HostWordBounds hw;
            YTGPU_TRY(encode_bounds_words(spec, P->layout, &hw));
            const u32 Pn = P->partition_count;
            YTGPU_TRY(run->bwords.allocate(ctx, hw.words.size()));
            YTGPU_TRY(run->boff.allocate(ctx, hw.col_off.size()));
            YTGPU_TRY(run->bnbytes.allocate(ctx, Pn));
            YTGPU_TRY(run->bincl.allocate(ctx, Pn));
            YTGPU_CUDA_TRY(cudaMemcpyAsync(run->bwords.p, hw.words.data(), hw.words.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
            YTGPU_CUDA_TRY(cudaMemcpyAsync(run->boff.p, hw.col_off.data(), hw.col_off.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
            YTGPU_CUDA_TRY(cudaMemcpyAsync(run->bnbytes.p, hw.plen.data(), Pn * 4, cudaMemcpyHostToDevice, ctx->stream));
            YTGPU_CUDA_TRY(cudaMemcpyAsync(run->bincl.p, hw.inclusive.data(), Pn, cudaMemcpyHostToDevice, ctx->stream));
            YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));  // hw goes out of scope
            run->wbounds = WordBounds{run->bwords.p, run->boff.p, run->bnbytes.p, run->bincl.p, Pn};
            return Status{};
        }
        HostBounds hb;
        YTGPU_TRY(normalize_bounds(spec, P->layout, &hb));
        const u32 Pn = P->partition_count;
        YTGPU_TRY(run->bwords.allocate(ctx, hb.words.size()));
        YTGPU_TRY(run->bnbytes.allocate(ctx, Pn));
        YTGPU_TRY(run->bincl.allocate(ctx, Pn));
        YTGPU_CUDA_TRY(cudaMemcpyAsync(run->bwords.p, hb.words.data(), hb.words.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
        YTGPU_CUDA_TRY(cudaMemcpyAsync(run->bnbytes.p, hb.nbytes.data(), Pn * 4, cudaMemcpyHostToDevice, ctx->stream));
        YTGPU_CUDA_TRY(cudaMemcpyAsync(run->bincl.p, hb.inclusive.data(), Pn, cudaMemcpyHostToDevice, ctx->stream));
        YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));  // hb goes out of scope
        P->bounds = DeviceBounds{run->bwords.p, run->bnbytes.p, run->bincl.p, Pn, P->layout.nchunks};
    } else if (spec->kind == YTGPU_PARTITION_HASH) {
        if (spec->key_column_count < 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "negative key_column_count");
        P->key_column_count = (u32)spec->key_column_count;
        P->salt_hash = fh::fingerprint_u64(spec->salt);
        if (fixed) {
            if (!spec->key.columns) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "fixed-row hash partitioning needs key columns");
            YTGPU_TRY(build_key_layout(&spec->key, true, false, &P->layout));
        }
    } else if (spec->kind == YTGPU_PARTITION_COLUMN) {
        if (fixed) return make_status(YTGPU_ERR_UNSUPPORTED, "column-based partitioning needs a rowset");
        P->column_id = spec->partition_column_id;
    } else {
        return make_status(YTGPU_ERR_INVALID_ARGUMENT, "unknown partitioner kind %d", spec->kind);
    }
    return Status{};
}

Status finish_outputs(Context* ctx, PartitionRun& run, u64 n, u32 Pn, i32* out_index, u64* out_histogram, int out_mem) {
    YTGPU_TRY(run.index.download(ctx, n));
    // the kernels count into a zeroed scratch histogram, which is copied out in either memory space
    if (out_histogram) YTGPU_TRY(copy_out(ctx, out_histogram, run.hist.p, (size_t)Pn * 8, out_mem));
    return Status{};
}

Status partition_rowset_impl(Context* ctx, const ytgpu_rowset_view* in, const ytgpu_partition_spec* spec,
                             i32* out_index, u64* out_histogram, int out_mem, ytgpu_value* out_slab_values = nullptr,
                             u32* out_slab_perm = nullptr) {
    ctx->last_partition_key_words = false;
    if (!in) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null rowset");
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    const u64 n = in->row_count;
    StagedRowset staged;
    YTGPU_TRY(staged.stage(ctx, in, n ? in->mem : YTGPU_MEM_DEVICE));  // no rows: the caller's pointers stay
    const ytgpu_value* vals = staged.values.p;
    PartParams P;
    PartitionRun run;
    YTGPU_TRY(prepare_params(ctx, spec, false, in->value_count, vals, n, &P, &run));
    ctx->last_partition_key_words = run.key_words;
    P.values = vals;
    P.value_count = in->value_count;
    P.heap = staged.heap.p;
    P.n = n;
    const u32 Pn = P.partition_count;
    if (out_histogram) {
        YTGPU_TRY(run.hist.allocate(ctx, Pn));
        YTGPU_CUDA_TRY(cudaMemsetAsync(run.hist.p, 0, (size_t)Pn * 8, ctx->stream));
        P.histogram = run.hist.p;
    }
    YTGPU_TRY(run.index.prepare(ctx, out_index, n, out_mem));
    P.out_index = run.index.p;
    const bool slabs = (out_slab_values || out_slab_perm) && n;
    if (slabs) {
        YTGPU_TRY(run.chunk.allocate(ctx, n));
        P.out_chunk = run.chunk.p;
    }
    YTGPU_TRY(launch_partition(ctx, P, false, run.key_words ? &run.wbounds : nullptr));
    if (slabs) {
        // variable-length rows: the 16-byte values of a row are fixed width and the strings stay where they are (their
        // offsets still point into the input heap), so the slab scatter is the fixed-row one over value_count * 16 bytes
        SortScratch scratch;
        PermRef perm;
        const u64* cptr[1] = {run.chunk.p};
        YTGPU_TRY(radix_sort_chunks(ctx, cptr, 1, n, &scratch, &perm));
        const u32 rb = in->value_count * 16;
        OutBuf<u8> vout;
        OutBuf<u32> pout;
        if (out_slab_values) {
            YTGPU_TRY(vout.prepare(ctx, reinterpret_cast<u8*>(out_slab_values), n * rb, out_mem));
            YTGPU_TRY(gather_rows(ctx, reinterpret_cast<const u8*>(vals), perm, vout.p, n, rb));
            YTGPU_TRY(vout.download(ctx, n * rb));
        }
        if (out_slab_perm) {
            YTGPU_TRY(pout.prepare(ctx, out_slab_perm, n, out_mem));
            YTGPU_TRY(materialize_perm(ctx, perm, n, pout.p));
            YTGPU_TRY(pout.download(ctx, n));
        }
        if (out_mem == YTGPU_MEM_HOST) YTGPU_CUDA_TRY(cudaStreamSynchronize(ctx->stream));  // the staging buffers die here
    }
    YTGPU_TRY(finish_outputs(ctx, run, n, Pn, out_index, out_histogram, out_mem));
    return check_device_errors(ctx);
}

Status partition_fixed_impl(Context* ctx, const ytgpu_fixed_rows_view* in, const ytgpu_partition_spec* spec,
                            i32* out_index, u64* out_histogram, u8* out_slab_rows, int out_mem) {
    if (!in) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null rows");
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    const u64 n = in->row_count;
    const u32 rb = in->row_bytes;
    if (rb == 0 || rb % 16 != 0) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "row_bytes (%u) must be a positive multiple of 16", rb);
    InBuf<u8> rows;
    YTGPU_TRY(rows.stage(ctx, in->rows, n * rb, n ? in->mem : YTGPU_MEM_DEVICE));  // no rows: the caller's pointer stays
    OutBuf<u8> slabs;
    PartParams P;
    PartitionRun run;
    YTGPU_TRY(prepare_params(ctx, spec, true, 0, nullptr, n, &P, &run));
    for (u32 c = 0; c < P.layout.ncols; ++c)
        if ((u64)P.layout.col[c].index + P.layout.col[c].payload_bytes > rb)
            return make_status(YTGPU_ERR_INVALID_ARGUMENT, "key column %u exceeds the row", c);
    P.rows = rows.p;
    P.row_bytes = rb;
    P.n = n;
    const u32 Pn = P.partition_count;
    if (out_histogram) {
        YTGPU_TRY(run.hist.allocate(ctx, Pn));
        YTGPU_CUDA_TRY(cudaMemsetAsync(run.hist.p, 0, (size_t)Pn * 8, ctx->stream));
        P.histogram = run.hist.p;
    }
    YTGPU_TRY(run.index.prepare(ctx, out_index, n, out_mem));
    P.out_index = run.index.p;
    if (out_slab_rows) {
        YTGPU_TRY(run.chunk.allocate(ctx, n));
        P.out_chunk = run.chunk.p;
    }
    YTGPU_TRY(launch_partition(ctx, P, true));
    if (out_slab_rows && n) {
        // stable scatter into partition-contiguous slabs = stable sort by partition index + gather
        SortScratch scratch;
        PermRef perm;
        const u64* cptr[1] = {run.chunk.p};
        YTGPU_TRY(radix_sort_chunks(ctx, cptr, 1, n, &scratch, &perm));
        YTGPU_TRY(slabs.prepare(ctx, out_slab_rows, n * rb, out_mem));
        YTGPU_TRY(gather_rows(ctx, rows.p, perm, slabs.p, n, rb));
        YTGPU_TRY(slabs.download(ctx, n * rb));
    }
    YTGPU_TRY(finish_outputs(ctx, run, n, Pn, out_index, out_histogram, out_mem));
    return check_device_errors(ctx);
}

__global__ void __launch_bounds__(256) fingerprint_rows_kernel(const ytgpu_value* __restrict__ values, u32 value_count,
                                                               const u8* __restrict__ heap, u64 n, u32 k,
                                                               u64* __restrict__ out, u32* err_word) {
    u32 err = 0;
    for (u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (u64)gridDim.x * blockDim.x) {
        const ytgpu_value* row = values + i * value_count;
        u64 h = 0xdeadc0deULL;
        for (u32 c = 0; c < k; ++c) {
            u64 f;
            err |= fh::value_fingerprint(load_value(row + c), heap, &f);
            h = fh::fingerprint_u128(h, f);
        }
        out[i] = h ^ (u64)k;
    }
    if (err) atomicOr(err_word, err);
}

Status fingerprint_impl(Context* ctx, const ytgpu_rowset_view* in, u32 k, u64* out, int out_mem) {
    if (!in || !out) return make_status(YTGPU_ERR_INVALID_ARGUMENT, "null argument");
    YTGPU_CUDA_TRY(cudaSetDevice(ctx->device));
    const u64 n = in->row_count;
    if (n == 0) return Status{};
    k = std::min(k, in->value_count);
    StagedRowset staged;
    OutBuf<u64> dst;
    YTGPU_TRY(staged.stage(ctx, in, in->mem));
    YTGPU_TRY(dst.prepare(ctx, out, n, out_mem));
    {
        KernelTimer t(ctx, KC_PARTITION);
        u32 blocks = (u32)std::min<u64>((n + 255) / 256, (u64)kNumSms * 8);
        fingerprint_rows_kernel<<<blocks, 256, 0, ctx->stream>>>(staged.values.p, in->value_count, staged.heap.p, n, k, dst.p, ctx->dev_err);
        YTGPU_CUDA_TRY(cudaGetLastError());
    }
    YTGPU_TRY(dst.download(ctx, n));
    return check_device_errors(ctx);
}

}  // namespace

extern "C" {

int ytgpu_partition_rowset(ytgpu_context* h, const ytgpu_rowset_view* in, const ytgpu_partition_spec* spec,
                           int32_t* out_index, uint64_t* out_histogram, int out_mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, partition_rowset_impl(as_context(h), in, spec, out_index, out_histogram, out_mem));
}

int ytgpu_partition_rowset_slabs(ytgpu_context* h, const ytgpu_rowset_view* in, const ytgpu_partition_spec* spec, int32_t* out_index,
                                 uint64_t* out_histogram, ytgpu_value* out_slab_values, uint32_t* out_slab_perm, int out_mem,
                                 ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, partition_rowset_impl(as_context(h), in, spec, out_index, out_histogram, out_mem, out_slab_values, out_slab_perm));
}

int ytgpu_partition_fixed_rows(ytgpu_context* h, const ytgpu_fixed_rows_view* in, const ytgpu_partition_spec* spec,
                               int32_t* out_index, uint64_t* out_histogram, uint8_t* out_slab_rows, int out_mem,
                               ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, partition_fixed_impl(as_context(h), in, spec, out_index, out_histogram, out_slab_rows, out_mem));
}

int ytgpu_farm_fingerprint_rowset(ytgpu_context* h, const ytgpu_rowset_view* in, uint32_t key_column_count,
                                  uint64_t* out, int out_mem, ytgpu_error* err) {
    if (!h) return fill_error(err, make_status(YTGPU_ERR_INVALID_ARGUMENT, "null context"));
    CtxLock lock(h);
    return fill_error(err, fingerprint_impl(as_context(h), in, key_column_count, out, out_mem));
}

// ---- host-side self checks of the __host__ __device__ logic (CPU tests; not part of ytgpu.h) ----
int ytgpu_hostcheck_normalize_rowset(const ytgpu_value* values, uint32_t value_count, const uint8_t* heap,
                                     uint64_t n, const ytgpu_sort_spec* spec, uint64_t* out_words,
                                     uint32_t* out_nchunks, uint32_t* out_err) {
    KeyLayout L;
    Status s = build_key_layout(spec, false, false, &L);
    if (!s.ok()) return s.code;
    *out_nchunks = L.nchunks;
    u32 err = 0;
    for (u64 i = 0; i < n; ++i) {
        u64 words[kMaxKeyChunks + 1] = {0};
        ChunkWriter w(words);
        for (u32 c = 0; c < L.ncols; ++c) err |= normalize_value(L.col[c], values[i * value_count + L.col[c].index], heap, w);
        w.finish();
        for (u32 c = 0; c < L.nchunks; ++c) out_words[i * L.nchunks + c] = words[c];
    }
    *out_err = err;
    return YTGPU_OK;
}

int ytgpu_hostcheck_partition_ordered(const ytgpu_value* values, uint32_t value_count, const uint8_t* heap, uint64_t n,
                                      const ytgpu_partition_spec* spec, int32_t* out_index) {
    KeyLayout L;
    Status s = build_key_layout(&spec->key, false, false, &L);
    if (!s.ok()) return s.code;
    HostBounds hb;
    s = normalize_bounds(spec, L, &hb);
    if (!s.ok()) return s.code;
    for (u64 i = 0; i < n; ++i) {
        u64 key[kMaxKeyChunks + 1] = {0};
        ChunkWriter w(key);
        for (u32 c = 0; c < L.ncols; ++c) normalize_value(L.col[c], values[i * value_count + L.col[c].index], heap, w);
        w.finish();
        u32 lo = 0, cnt = (u32)spec->partition_count;
        while (cnt > 0) {
            u32 step = cnt >> 1, mid = lo + step;
            const u64* bw = hb.words.data() + (size_t)mid * L.nchunks;
            u32 nb = hb.nbytes[mid], full = nb >> 3, rem = nb & 7;
            int cmp = 0;
            for (u32 k = 0; k < full && !cmp; ++k)
                if (key[k] != bw[k]) cmp = key[k] > bw[k] ? 1 : -1;
            if (!cmp && rem) {
                u64 mask = ~0ull << (8 * (8 - rem));
                u64 a = key[full] & mask, b = bw[full] & mask;
                if (a != b) cmp = a > b ? 1 : -1;
            }
            bool t = cmp > 0 || (cmp == 0 && hb.inclusive[mid]);
            if (t) { lo = mid + 1; cnt -= step + 1; } else cnt = step;
        }
        out_index[i] = (i32)lo - 1;
    }
    return YTGPU_OK;
}

// The key-word partitioner (the bound encoding and the __host__ __device__ search partition_words_kernel runs) for keys
// of any width, the ones that fit the normalised form included.  out_index[i] = -1 for a key below the first bound.
int ytgpu_hostcheck_partition_ordered_words(const ytgpu_value* values, uint32_t value_count, const uint8_t* heap, uint64_t n,
                                            const ytgpu_partition_spec* spec, int32_t* out_index) {
    KeyLayout L;
    Status s = build_key_layout(&spec->key, false, false, &L);
    if (!s.ok() && !(s.code == YTGPU_ERR_UNSUPPORTED && L.nchunks > (u32)kMaxKeyChunks)) return s.code;
    HostWordBounds hb;
    s = encode_bounds_words(spec, L, &hb);
    if (!s.ok()) return s.code;
    const WordBounds B = hb.view();
    for (u64 i = 0; i < n; ++i) out_index[i] = ordered_index_words(L, values + i * value_count, heap, B);
    return YTGPU_OK;
}

uint64_t ytgpu_hostcheck_fingerprint_bytes(const uint8_t* s, uint64_t n) { return fh::fingerprint_bytes(s, n); }

int ytgpu_hostcheck_row_fingerprints(const ytgpu_value* values, uint32_t value_count, const uint8_t* heap, uint64_t n,
                                     uint32_t k, uint64_t* out) {
    u32 err = 0;
    for (u64 i = 0; i < n; ++i) err |= fh::row_fingerprint(values + i * value_count, k < value_count ? k : value_count, heap, &out[i]);
    return err ? YTGPU_ERR_UNSUPPORTED : YTGPU_OK;
}

}  // extern "C"
