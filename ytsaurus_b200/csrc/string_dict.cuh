// string_dict.cuh — a device string dictionary (see string_column_writer.cu): the distinct values of one string column,
// held in device memory the dictionary owns, and the lookup of other strings in it.  The join table keys its string
// components on it (join.cu).
#pragma once

#include "context.cuh"

namespace ytgpu {

// One column of `rows` rows, after string_dicts_build.  heap: every non-NULL value's bytes, compacted in row order; value
// g is lengths[g] bytes at heap + starts[g] (a NULL row has length 0; starts has rows + 1 entries).  slots: the
// open-addressing table of the string column writer's value-ids insert, kept as the insert leaves it: a power of two >= 2
// x rows (at least 8) of words (fingerprint << 32) | the first row holding the value, ~0 when empty.
struct StringDict {
    DevBuf<u8> heap;
    DevBuf<u64> starts;
    DevBuf<u32> lengths;
    DevBuf<u64> slots;
};

// The id of a value no dictionary row holds.  Dictionary ids are rows below 2^30.
constexpr u64 kStringDictMiss = ~0ull;

// For each of `count` string columns of `rows` rows (HOST or DEVICE, checked by the caller): dicts[c], and the column's
// ids: ids[c][g] = the first row of column c holding row g's bytes, 0 for NULL; null_bits[c], a YT null bitmap (1 = NULL)
// in ceil(rows / 32) 4-byte words, only for a column with a null bytemap.  A non-NULL value outside its heap is
// INVALID_ARGUMENT, and no byte outside the heap is read.  Synchronises once: the heap sizes and the device error word.
Status string_dicts_build(Context* ctx, const ytgpu_string_column* cols, u32 count, u64 rows, StringDict* dicts, DevBuf<u64>* ids,
                          DevBuf<u32>* null_bits);

// ids[g] = the dictionary id of row g of `col` (`rows` rows, HOST or DEVICE): the first dictionary row holding the same
// bytes, else kStringDictMiss; 0 for NULL, with its bit set in null_bits (written only when col has a null bytemap, in
// the layout above).  A non-NULL value outside its heap sets DE_STRING_OUT_OF_HEAP in the device error word and reads
// nothing; the caller reads that word.  No synchronisation.
Status string_dict_lookup(Context* ctx, const StringDict& dict, const ytgpu_string_column& col, u64 rows, u64* ids, u32* null_bits);

// A growing dictionary (the GROUP BY table's, groupby_table.cu) uses the same layout with dense ids: value id is
// lengths[id] bytes at heap + starts[id] for id < *count, *bytes heap bytes are in use, and the slot words are
// (fingerprint << 32) | id; string_dict_lookup reads it as it reads a built one.  An empty one has 8 empty slots.
// string_dict_append adds the values of `col` (n rows, HOST or DEVICE, every non-NULL value inside its heap: the caller
// looked the column up first and read the device error word) that the dictionary lacks, in first-row order, growing its
// buffers by doubling and rehashing its slots from the kept bytes.  ids: in, string_dict_lookup's result over col; out,
// every non-NULL row's id (NULL rows keep 0).  Synchronises once, for the count and bytes of the new values.
Status string_dict_append(Context* ctx, StringDict* dict, u64* count, u64* bytes, const ytgpu_string_column& col, u64 n, u64* ids);

}  // namespace ytgpu
