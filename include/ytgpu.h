/* ytgpu.h — C ABI of the H100-native sort/shuffle + scan→filter→group-by hot path.
 *
 * This is the drop-in boundary a YTsaurus job proxy / CHYT instance binds to
 * (INTEGRATION.md shows the C++ adapters).  Plain pointers and sizes only; no
 * torch / CUDA types in signatures (a CUDA stream travels as void*).
 *
 * Every entry point cites the reference interface it replaces (paths relative
 * to the YTsaurus tree).  All calls are asynchronous with respect to the
 * context's stream unless they return data to HOST memory, in which case they
 * synchronise that stream before returning.  Calls never fall back to a CPU
 * implementation: if the device cannot run the request the call fails with
 * YTGPU_ERR_UNSUPPORTED / YTGPU_ERR_CUDA.
 */
#ifndef YTGPU_H_
#define YTGPU_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define YTGPU_ABI_VERSION 2

/* ---- status / errors (replaces TErrorException, THROW_ERROR_EXCEPTION) ---- */
typedef enum ytgpu_status {
    YTGPU_OK = 0,
    YTGPU_ERR_INVALID_ARGUMENT = 1,
    YTGPU_ERR_UNSUPPORTED = 2,      /* e.g. Any/Composite key columns (need the YSON comparer) */
    YTGPU_ERR_CUDA = 3,
    YTGPU_ERR_OUT_OF_MEMORY = 4,
    YTGPU_ERR_SCHEMA_VIOLATION = 5, /* value type differs from the declared key column type */
    YTGPU_ERR_PARTITION_BAD_TYPE = 10,     /* partitioner.cpp:143-149 */
    YTGPU_ERR_PARTITION_NEGATIVE = 11,     /* partitioner.cpp:151-156 */
    YTGPU_ERR_PARTITION_OUT_OF_BOUNDS = 12,/* partitioner.cpp:158-163 */
    YTGPU_ERR_PARTITION_NO_COLUMN = 13     /* partitioner.cpp:167 */
} ytgpu_status;

typedef struct ytgpu_error {
    int32_t code;       /* ytgpu_status */
    int32_t cuda_error; /* cudaError_t when code == YTGPU_ERR_CUDA */
    char message[248];
} ytgpu_error;

/* ---- memory spaces ---- */
typedef enum ytgpu_mem { YTGPU_MEM_DEVICE = 0, YTGPU_MEM_HOST = 1 } ytgpu_mem;

/* ---- per-device context (explicit; no thread-local CUDA state is assumed, YT fibers migrate) ----
 * Calls made on ONE context are serialised by the library (each entry point locks the context), so readers,
 * partitioners and writers living on different threads may share it; use one context per job slot / stream for
 * concurrency.  A process may own contexts on several devices. */
typedef struct ytgpu_context ytgpu_context;

/* cuda_stream: a cudaStream_t to run on (e.g. torch's current stream; pass cudaStreamLegacy == (void*)1
 * for the legacy default stream), or NULL for a private non-blocking stream. */
int ytgpu_context_create(int device, void* cuda_stream, ytgpu_context** out, ytgpu_error* err);
void ytgpu_context_destroy(ytgpu_context* ctx);
int ytgpu_context_synchronize(ytgpu_context* ctx, ytgpu_error* err);
/* Number of kernel launches issued through this context since creation (bench.py's gpu_launches). */
uint64_t ytgpu_context_launch_count(const ytgpu_context* ctx);
/* Device time (ms) of the dominant kernel class measured with CUDA events on the context stream,
 * accumulated since the last reset: which = 0 radix passes that moved data (timed launch by launch), 1 row
 * gather / peer scatter, 2 key extraction, 3 histogram / tie fix-up, 4 partition, 5 group-by, 6 decode / block
 * codec, 7 radix pass launches that were skipped on the device (inactive digit), 8 the in-box
 * shuffle's row scatter over NVLink, 9 its sampling / pivot selection / count exchange / peer barriers (includes the
 * time spent WAITING for the other ranks), 10 sorted-input segmented reduce, 11 hash join: build, probe, pair write and
 * gathers.
 * launches (nullable) receives the number of launches behind the returned time. */
double ytgpu_context_kernel_ms(ytgpu_context* ctx, int which, uint64_t* launches);
void ytgpu_context_reset_timers(ytgpu_context* ctx);
/* Radix passes that actually moved data in the most recent sort on this context (digits whose
 * histogram has a single bin are skipped); synchronises the stream. */
uint64_t ytgpu_context_last_sort_passes(ytgpu_context* ctx);
void ytgpu_context_enable_timers(ytgpu_context* ctx, int enabled);
/* Tuning / experiment switches of one context (defaults are the measured-best settings):
 *   "sort_hybrid"  1 (default): single-chunk keys are sorted by their most significant active digits first and short
 *                  runs of equal prefixes are fixed up; 0: always the full LSD schedule.
 *   "merge_path"   1 (default): ytgpu_merge_sorted_runs merges up to 16 sorted runs pairwise (merge path); 0: always the
 *                  stable sort of the concatenated runs.
 * Returns INVALID_ARGUMENT for an unknown name. */
int ytgpu_context_set_option(ytgpu_context* ctx, const char* name, int64_t value, ytgpu_error* err);
/* Reads an option back, or one of the read-only counters:
 *   "last_merge_used_merge_path"  1 when the most recent ytgpu_merge_sorted_runs took the merge-path rounds, 0 when it
 *                                 sorted (many runs, an unsorted run, a key of more than 256 normalised bytes, or the
 *                                 option switched off).
 *   "last_sort_refine_rounds"     refinement rounds the most recent ytgpu_sort_rowset / ytgpu_merge_sorted_runs /
 *                                 ytgpu_join_sorted_runs ran: >= 1 when its key did not fit the 256-byte normalised form
 *                                 and took the width-free key words (the first round counts even when every key is
 *                                 equal), 0 when it took the normalised-key path.
 *   "last_sort_refine_rows.<r>"   rows that round r (from 0) of that call sorted (0 past its last round).
 *   "last_partition_key_words"    1 when the most recent ytgpu_partition_rowset / ytgpu_partition_rowset_slabs
 *                                 compared width-free key words (an ordered partitioner whose key did not fit the
 *                                 256-byte normalised form), 0 otherwise. */
int ytgpu_context_get_option(ytgpu_context* ctx, const char* name, int64_t* value, ytgpu_error* err);

/* Completion notification without blocking a thread: `fn(user)` runs on a driver thread once everything enqueued on the
 * context's stream so far has finished (cudaLaunchHostFunc).  The adapters set the TFuture<void> behind GetReadyEvent()
 * from it, so a YT fiber never sits in cudaStreamSynchronize (SURVEY §8b "Threading"; sorting_reader.cpp:53-55 runs
 * DoOpen via AsyncVia for the same reason).  DEVICE-flavour calls are asynchronous; enqueue the call(s), then the
 * notification.  The callback must not call back into the library. */
typedef void (*ytgpu_callback)(void* user);
int ytgpu_context_notify(ytgpu_context* ctx, ytgpu_callback fn, void* user, ytgpu_error* err);

/* Pinned host buffers for the HOST-memory flavour of the calls (cudaHostAlloc). */
void* ytgpu_host_alloc(size_t bytes);
void ytgpu_host_free(void* p);

int ytgpu_abi_version(void);

/* ---- row model ---- */
/* EValueType, yt/yt/client/table_client/row_base.h:11-28 */
enum {
    YTGPU_TYPE_MIN = 0x00, YTGPU_TYPE_BOTTOM = 0x01, YTGPU_TYPE_NULL = 0x02, YTGPU_TYPE_INT64 = 0x03,
    YTGPU_TYPE_UINT64 = 0x04, YTGPU_TYPE_DOUBLE = 0x05, YTGPU_TYPE_BOOLEAN = 0x06, YTGPU_TYPE_STRING = 0x10,
    YTGPU_TYPE_ANY = 0x11, YTGPU_TYPE_COMPOSITE = 0x12, YTGPU_TYPE_MAX = 0xef
};

/* TUnversionedValue, yt/yt/client/table_client/unversioned_value.h:37-62 (same 16-byte layout).
 * For string-like types `data` is a byte OFFSET into the rowset's string heap. */
typedef struct ytgpu_value {
    uint16_t id;
    uint8_t type;
    uint8_t flags;
    uint32_t length;
    uint64_t data;
} ytgpu_value;

/* A drained TRange<TUnversionedRow> (unversioned_row.h:272-352): row_count rows of value_count values. */
typedef struct ytgpu_rowset_view {
    const ytgpu_value* values;
    uint64_t row_count;
    uint32_t value_count;
    uint32_t reserved;
    const uint8_t* string_heap;
    uint64_t string_heap_bytes;
    int32_t mem; /* ytgpu_mem of values and string_heap */
} ytgpu_rowset_view;

/* Fixed-width packed rows: schemaful rows whose columns are all required fixed-size scalars or
 * fixed-length strings (the benchmark's "64-byte row": uint64 key + string[56]). */
typedef struct ytgpu_fixed_rows_view {
    const uint8_t* rows;
    uint64_t row_count;
    uint32_t row_bytes; /* multiple of 16 */
    int32_t mem;
} ytgpu_fixed_rows_view;

/* One key column: TColumnSortSchema{Name, SortOrder} + the type information of TColumnSchema.
 *  rowset:     `index` = position of the value in the row; `type` = declared EValueType or 0 for "any
 *              scalar" (schemaless keys); `required` drops the type byte (TColumnSchema::Required());
 *              `width` = maximum string length (0 = measure it on the device).
 *  fixed rows: `index` = byte offset in the row; `type` one of INT64/UINT64/DOUBLE/BOOLEAN/STRING;
 *              `width` = exact string length. */
typedef struct ytgpu_key_column {
    uint32_t index;
    uint32_t width;
    uint8_t type;
    uint8_t descending; /* ESortOrder::Descending, comparator.cpp:56-58 */
    uint8_t required;
    uint8_t reserved;
} ytgpu_key_column;

typedef struct ytgpu_sort_spec {
    const ytgpu_key_column* columns; /* host memory */
    uint32_t column_count;           /* == TComparator::GetLength() */
} ytgpu_sort_spec;

/* ---- sort ----
 * Replaces TSortingReader::DoOpen's std::sort (yt/yt/ytlib/table_client/sorting_reader.cpp:163-188,
 * factory sorting_reader.h:15-20) and TPartitionSortReader's bucket sort + merge
 * (partition_sort_reader.cpp:384-529).  The sort is STABLE (rows with equal keys keep input order),
 * which is one of the orders the reference's unstable std::sort may produce.
 * out_perm[i] = input index of the i-th output row.
 * Keys of any length: a key whose normalised form (strings padded to the longest one, or to the declared `width`) fits
 * in 256 bytes is radix-sorted as such; a longer one is sorted by refinement rounds over width-free key words (see
 * "last_sort_refine_rounds").  A string longer than a declared `width` is YTGPU_ERR_SCHEMA_VIOLATION on both paths;
 * Any/Composite key values are YTGPU_ERR_UNSUPPORTED. */
int ytgpu_sort_rowset(ytgpu_context* ctx, const ytgpu_rowset_view* in, const ytgpu_sort_spec* spec,
                      uint32_t* out_perm, ytgpu_value* out_values /* nullable: rows gathered in sorted order */,
                      int out_mem, ytgpu_error* err);

int ytgpu_sort_fixed_rows(ytgpu_context* ctx, const ytgpu_fixed_rows_view* in, const ytgpu_sort_spec* spec,
                          uint8_t* out_rows /* nullable */, uint32_t* out_perm /* nullable */, int out_mem,
                          ytgpu_error* err);

/* Replaces CreateSortedMergingReader (sorted_merging_reader.cpp:771-788; order = CompareStreams :395-409):
 * `in` is the concatenation of run_count sorted runs, run r = rows [run_offsets[r], run_offsets[r+1]).
 * Ties are broken by run index, then by position in the run.  Keys of any length, as ytgpu_sort_rowset; a key that does
 * not fit the 256-byte normalised form always takes the stable sort of the concatenated runs. */
int ytgpu_merge_sorted_runs(ytgpu_context* ctx, const ytgpu_rowset_view* in, const ytgpu_sort_spec* spec,
                            const uint64_t* run_offsets /* host */, uint32_t run_count, uint32_t* out_perm,
                            int out_mem, ytgpu_error* err);

/* Replaces CreateSortedJoiningReader / TSortedJoiningReader::Read (sorted_merging_reader.cpp:566-760, factory :790-815):
 * run 0 of `in` is the PRIMARY stream (the already merged primary readers), runs 1.. are the FOREIGN streams; every run
 * is sorted by the join key = the first join_key_column_count columns of `spec`.  The remaining spec columns only break
 * ties between streams: the reference's heap orders streams with equal keys by their table index (CompareStreams
 * :395-409; one index per stream, taken from its first row :101-104), so the adapters append that index as the last
 * key column.  The result is the stable order by all spec columns in which a foreign row survives iff its join key
 * occurs in the primary stream (:722-738: it equals the last primary key consumed or the next one).
 * out_perm (capacity row_count) receives the input indices of the emitted rows, *out_row_count (host) their number.
 * Keys of any length, as ytgpu_sort_rowset. */
int ytgpu_join_sorted_runs(ytgpu_context* ctx, const ytgpu_rowset_view* in, const ytgpu_sort_spec* spec,
                           uint32_t join_key_column_count, const uint64_t* run_offsets /* host */, uint32_t run_count,
                           uint32_t* out_perm, uint64_t* out_row_count, int out_mem, ytgpu_error* err);

/* ---- partition ----
 * Replaces the per-row IPartitioner::GetPartitionIndex loop of TPartitionMultiChunkWriter::WriteRow
 * (yt/yt/ytlib/table_client/partitioner.h:14-19, partitioner.cpp:41-57,99-107,122-173,
 * schemaless_chunk_writer.cpp:1604-1623) and CreatePartitioner (ytlib/job_proxy/helpers.cpp:113-147). */
typedef enum ytgpu_partitioner_kind {
    YTGPU_PARTITION_ORDERED = 0, YTGPU_PARTITION_HASH = 1, YTGPU_PARTITION_COLUMN = 2
} ytgpu_partitioner_kind;

typedef struct ytgpu_partition_spec {
    int32_t kind;
    int32_t partition_count;          /* ordered: number of lower bounds incl. the universal bound 0 */
    /* ordered: */
    ytgpu_sort_spec key;              /* comparator */
    const ytgpu_value* bounds;        /* host; partition_count rows of bound_value_count values */
    const uint8_t* bounds_heap;       /* host */
    uint64_t bounds_heap_bytes;
    uint32_t bound_value_count;
    const uint32_t* bound_prefix_length; /* host; values of the prefix used by bound b (0 = universal) */
    const uint8_t* bound_inclusive;      /* host */
    /* hash: */
    int32_t key_column_count;         /* reduce_key_column_count */
    uint64_t salt;                    /* partition_task_level; Salt_ = FarmHash(salt), partitioner.cpp:88-91 */
    /* column: */
    uint16_t partition_column_id;
} ytgpu_partition_spec;

/* out_index (nullable) gets the partition of every row; out_histogram (nullable, partition_count
 * entries) the rows per partition.  Both live in out_mem.
 * Ordered partitioner, keys of any length: a key whose normalised form (strings padded to the longest one, or to the
 * declared `width`) fits in 256 bytes is compared as such; a longer one is compared with the bounds over width-free key
 * words, with the same indices (see "last_partition_key_words").  A string longer than a declared `width` is
 * YTGPU_ERR_SCHEMA_VIOLATION and Any/Composite key or bound values are YTGPU_ERR_UNSUPPORTED on both paths; a key
 * below the first bound is YTGPU_ERR_PARTITION_OUT_OF_BOUNDS. */
int ytgpu_partition_rowset(ytgpu_context* ctx, const ytgpu_rowset_view* in, const ytgpu_partition_spec* spec,
                           int32_t* out_index, uint64_t* out_histogram, int out_mem, ytgpu_error* err);

/* The same with the rows scattered into partition-contiguous slabs (stable inside a partition) for VARIABLE-length rows:
 * out_slab_values (nullable, row_count * value_count values) receives the rows' values grouped by partition — string
 * values keep their offsets into the INPUT heap, which therefore serves all slabs — and out_slab_perm (nullable,
 * row_count entries) the input row index of every slab row.  Partition p's rows are [sum(hist[0..p)), +hist[p]).
 * This is what the P per-partition block writers of TPartitionMultiChunkWriter accumulate
 * (schemaless_chunk_writer.cpp:1604-1623) before FlushBlock encodes a partition's rows.  Keys of any length, as
 * ytgpu_partition_rowset. */
int ytgpu_partition_rowset_slabs(ytgpu_context* ctx, const ytgpu_rowset_view* in, const ytgpu_partition_spec* spec,
                                 int32_t* out_index, uint64_t* out_histogram, ytgpu_value* out_slab_values,
                                 uint32_t* out_slab_perm, int out_mem, ytgpu_error* err);

/* Fixed-row flavour used by the in-box shuffle: additionally scatters the rows into
 * partition-contiguous slabs (stable inside a partition) — the GPU equivalent of the P per-partition
 * block writers (schemaless_chunk_writer.cpp:1609-1616).  out_slab_rows nullable. */
int ytgpu_partition_fixed_rows(ytgpu_context* ctx, const ytgpu_fixed_rows_view* in,
                               const ytgpu_partition_spec* spec, int32_t* out_index, uint64_t* out_histogram,
                               uint8_t* out_slab_rows, int out_mem, ytgpu_error* err);

/* ---- in-box shuffle over NVLink peer memory ----
 * Inside one 8-GPU box the reference's materialised shuffle (partition jobs tag blocks with partition_index,
 * schemaless_chunk_writer.cpp:1650-1667; sort jobs fetch them by tag, partition_chunk_reader.cpp:82-86) becomes one
 * kernel that writes each destination's slab straight into that GPU's receive buffer.  One process per GPU:
 * receive buffers are shared through CUDA IPC handles (64 opaque bytes, exchanged by the host plumbing). */
#define YTGPU_IPC_HANDLE_BYTES 64
int ytgpu_peer_buffer_create(ytgpu_context* ctx, uint64_t bytes, void** out_dev_ptr, uint8_t* out_handle /*[64]*/,
                             ytgpu_error* err);
int ytgpu_peer_buffer_destroy(ytgpu_context* ctx, void* dev_ptr, ytgpu_error* err);
int ytgpu_peer_buffer_open(ytgpu_context* ctx, const uint8_t* handle /*[64]*/, void** out_dev_ptr, ytgpu_error* err);
int ytgpu_peer_buffer_close(ytgpu_context* ctx, void* dev_ptr, ytgpu_error* err);
/* Fused slab scatter + exchange.  `in` (DEVICE) holds the rows, partition_index (DEVICE) their partitions as returned
 * by ytgpu_partition_fixed_rows, partition_rows (host) the rows per partition.  Partition p's rows are written in
 * stable order to dest_base[p] (host array of device pointers: local memory or peer-mapped receive buffers).
 * partition_count is in [1, 4096]; in->rows and every dest_base[p] are 16-byte aligned.  An index outside
 * [0, partition_count) or partition_rows that disagree with the index fail with YTGPU_ERR_INVALID_ARGUMENT before any
 * row is written.  Returns after the kernel completed on this GPU; a cross-rank barrier makes the data visible to its
 * readers. */
int ytgpu_scatter_rows_to_peers(ytgpu_context* ctx, const ytgpu_fixed_rows_view* in, const int32_t* partition_index,
                                int32_t partition_count, const uint64_t* partition_rows, void* const* dest_base,
                                ytgpu_error* err);

/* ---- in-box distributed sort: the whole Partition -> Sort hand-off of the sort controller for the GPUs of one box ----
 * Reference shape: samples -> BuildPartitionKeysFromSamples (yt/yt/server/controller_agent/helpers.cpp:263-425) ->
 * partition jobs with the ordered partitioner (partitioner.cpp:41-57) -> sort jobs per partition
 * (sort_controller.cpp:3444-3456).  One process (or thread) per GPU makes the same calls; rank r ends up with key range
 * r sorted (stable: ties keep (source rank, input position) order), so the concatenation over ranks is the sorted
 * table.  Ranks communicate only through peer-mapped device memory over NVLink: sample keys, the g x g row-count
 * matrix, device-side barriers and the rows themselves (fused slab scatter) — no NCCL, no host barrier; the host reads
 * the count matrix once per sort.  Pivot selection handles skew like the reference (weighted samples, maniac
 * partitions for heavily duplicated keys).
 * Setup: every rank creates its shuffle (receive buffer of capacity_rows rows) and obtains a 64-byte CUDA IPC handle;
 * the caller's own plumbing (job proxy RPC / torch.distributed in bench.py) gathers the handles of all ranks, in rank
 * order, and every rank passes the array to ytgpu_shuffle_connect. */
#define YTGPU_MAX_SHUFFLE_RANKS 32
typedef struct ytgpu_shuffle ytgpu_shuffle;
typedef struct ytgpu_shuffle_stats {
    uint64_t rows_in;                             /* rows this rank contributed */
    uint64_t rows_out;                            /* rows of this rank's key range */
    uint64_t sent[YTGPU_MAX_SHUFFLE_RANKS];       /* rows sent to every rank */
    uint64_t received[YTGPU_MAX_SHUFFLE_RANKS];   /* rows received from every rank */
    uint32_t world;
    uint32_t maniac;                              /* this rank's partition holds a single key (no sort was needed) */
} ytgpu_shuffle_stats;
int ytgpu_shuffle_create(ytgpu_context* ctx, int world, int rank, uint64_t capacity_rows, uint32_t row_bytes,
                         ytgpu_shuffle** out, uint8_t* out_handle /*[64]*/, ytgpu_error* err);
int ytgpu_shuffle_connect(ytgpu_shuffle* shuffle, const uint8_t* handles /*[world][64], rank order*/, ytgpu_error* err);
/* Collective: every rank calls it with its shard (`in`, DEVICE memory) and the same spec.  out_rows (DEVICE, nullable)
 * receives the rank's sorted key range, *out_row_count its size; INVALID_ARGUMENT when it exceeds out_capacity_rows or
 * when any rank's range exceeds its receive buffer (all ranks fail together).  Synchronises the stream once. */
int ytgpu_shuffle_sort(ytgpu_shuffle* shuffle, const ytgpu_fixed_rows_view* in, const ytgpu_sort_spec* spec,
                       uint8_t* out_rows, uint64_t out_capacity_rows, uint64_t* out_row_count, ytgpu_shuffle_stats* stats,
                       ytgpu_error* err);
int ytgpu_shuffle_destroy(ytgpu_shuffle* shuffle, ytgpu_error* err);

/* GetFarmFingerprint(row.FirstNElements(k)), unversioned_row.cpp:586-594, farm_hash.h:51-59. */
int ytgpu_farm_fingerprint_rowset(ytgpu_context* ctx, const ytgpu_rowset_view* in, uint32_t key_column_count,
                                  uint64_t* out, int out_mem, ytgpu_error* err);

/* ---- horizontal (schemaless) block codec: the intermediate-chunk wire format of partition / sort jobs ----
 * block = ui32 offsets[row_count] ++ rows; row = varuint32 value_count, then per value varuint32 id, varuint32 type,
 * payload (Int64 zig-zag varint, Uint64 varint, Double 8 raw bytes, Boolean 1 byte, String/Any varuint32 length +
 * bytes; Composite is written as Any).
 * Decode replaces THorizontalBlockReader::JumpToRowIndex/GetRow + ReadRowValue
 * (yt/yt/ytlib/table_client/schemaless_block_reader.cpp:187-246,323-349; unversioned_row.cpp:208-280): the first
 * value_count values of every row (short rows padded with Null, id 0xffff); a string value's `data` is the byte
 * offset of its payload INSIDE THE BLOCK (pass the block as the string heap of the resulting rowset).
 * out_row_value_counts (nullable) receives each row's real value count.  Malformed input -> INVALID_ARGUMENT. */
int ytgpu_decode_horizontal_block(ytgpu_context* ctx, const uint8_t* block, uint64_t block_bytes, uint32_t row_count,
                                  uint32_t value_count, ytgpu_value* out_values, uint32_t* out_row_value_counts,
                                  int mem, ytgpu_error* err);
/* Encode replaces THorizontalBlockWriter::WriteRow/FlushBlock + WriteRowValue
 * (schemaless_block_writer.cpp:40-86; unversioned_row.cpp:159-206).  row_value_counts (nullable, same memory space
 * as `rows`) gives the values actually present in each row.  *out_block_bytes is always set to the size the block
 * needs; the call fails with INVALID_ARGUMENT when out_capacity is smaller. */
int ytgpu_encode_horizontal_block(ytgpu_context* ctx, const ytgpu_rowset_view* rows, const uint32_t* row_value_counts,
                                  uint8_t* out_block, uint64_t out_capacity, uint64_t* out_block_bytes, int out_mem,
                                  ytgpu_error* err);

/* ---- columnar batches ----
 * Mirrors IUnversionedColumnarRowBatch::TColumn (yt/yt/client/table_client/row_batch.h:49-191) so a
 * MaterializeColumns() result can be described without copying semantics.  All pointers of one
 * view share `mem`.  Integer/double/boolean columns only (strings: offsets helper below). */
#define YTGPU_COLUMN_ARROW_VALIDITY 1u
typedef struct ytgpu_column_view {
    int64_t start_index;            /* TColumn::StartIndex */
    int64_t value_count;            /* TColumn::ValueCount */
    uint8_t value_type;             /* YTGPU_TYPE_INT64 / UINT64 / DOUBLE / BOOLEAN */
    uint8_t has_values;             /* TColumn::Values present (else: all null) */
    uint8_t zigzag;                 /* TValueBuffer::ZigZagEncoded */
    uint8_t bit_width;              /* 8/16/32/64, 0 when `values` is a TBitPackedUnsignedVector, 1 when it is a plain
                                       TBitmap (boolean columns: boolean_column_reader.cpp:134-172) */
    uint32_t reserved;              /* flags; bit 0 (YTGPU_COLUMN_ARROW_VALIDITY): null_bitmap is an Arrow validity
                                       bitmap (bit set = VALID), so an Arrow block — the input of YQL's
                                       BlockCombineHashed — is described without rewriting its bitmap */
    uint64_t base_value;            /* TValueBuffer::BaseValue */
    const void* values;             /* value vector of the (leaf) value column: dictionary values when
                                       dictionary-encoded, RLE values when RLE-encoded, else direct */
    uint64_t values_count;
    const uint8_t* null_bitmap;     /* nullable; bit i set = value i of the value vector is null */
    const uint32_t* dictionary_indexes; /* nullable; 1-based, 0 = null (ZeroMeansNull) */
    uint64_t dictionary_index_count;
    const uint64_t* rle_indexes;    /* nullable; start index of each run; rle_indexes[0] == 0 */
    uint64_t rle_count;
    int32_t mem;
} ytgpu_column_view;

/* DecodeIntegerVector + BuildNullBytemapForCHColumn (columnar-inl.h:355-376,
 * yt/chyt/server/columnar_conversion.cpp:204-234,948-999; bit unpack
 * yt/yt/core/misc/bit_packed_unsigned_vector-inl.h:115-173).  out_values gets value_count 64-bit
 * values (nulls decode to 0), out_null_bytemap (nullable) value_count bytes (1 = null). */
int ytgpu_decode_column(ytgpu_context* ctx, const ytgpu_column_view* column, uint64_t* out_values,
                        uint8_t* out_null_bytemap, int out_mem, ytgpu_error* err);

/* The same decode into a ClickHouse ColumnVector<T>: ConvertIntegerYTColumnToCHColumn (yt/chyt/server/
 * columnar_conversion.cpp:204-234,1001-1050) assigns the decoded 64-bit value to the column's element type (Int8 .. UInt64,
 * Date = UInt16, Date32 = Int32, Datetime = UInt32, DateTime64 = Int64: element_bytes 1 / 2 / 4 / 8, narrowed by truncation);
 * ConvertFloatingPointYTColumnToCHColumn (:341-369): a value vector of 32-bit floats (value_type Double, bit_width 32)
 * read with element_bytes 8 is widened to doubles, with element_bytes 4 copied; doubles are copied with element_bytes 8. */
int ytgpu_decode_column_typed(ytgpu_context* ctx, const ytgpu_column_view* column, uint32_t element_bytes, void* out_values,
                              uint8_t* out_null_bytemap, int out_mem, ytgpu_error* err);

/* DecodeStringOffsets, columnar.cpp:654-684: out[k-start] = offset(k) - offset(start), k in [start,end]. */
int ytgpu_decode_string_offsets(ytgpu_context* ctx, const uint32_t* encoded, uint32_t avg_length,
                                int64_t start_index, int64_t end_index, uint32_t* out, int mem,
                                ytgpu_error* err);

/* DecodeStringPointersAndLengths, columnar.cpp:686-707 (the string column reader's dense / dictionary value decode,
 * string_column_reader.cpp:266-520): value i of a string segment starts at out_start[i] inside the segment's string data
 * and is out_length[i] bytes long; end(i) = avg_length * (i + 1) + ZigZagDecode(encoded[i]).  `count` values. */
int ytgpu_decode_string_pointers_and_lengths(ytgpu_context* ctx, const uint32_t* encoded, uint32_t avg_length, uint64_t count,
                                             uint32_t* out_start, int32_t* out_length, int mem, ytgpu_error* err);

/* ---- null / dictionary-index helpers of the column readers (client/table_client/columnar.h:13-200) ----
 * The reference builds Arrow validity bitmaps, ClickHouse null bytemaps and Arrow dictionary indexes out of two kinds of
 * per-value flags: "the 1-based dictionary index is 0" (ZeroMeansNull) and "the bit of a TBitmap is set", either
 * addressed directly by the row or through RLE run starts.  One flag source + three consumers cover the family:
 *
 *   reference function (columnar.cpp)                                  entry point                      source     rle  negate
 *   BuildValidityBitmapFromDictionaryIndexesWithZeroNull    :286-331   ytgpu_build_bitmap_from_flags    DICT_ZERO  no   1
 *   BuildValidityBitmapFromRleDictionaryIndexesWithZeroNull :333-348   ytgpu_build_bitmap_from_flags    DICT_ZERO  yes  1
 *   BuildValidityBitmapFromRleNullBitmap                    :623-636   ytgpu_build_bitmap_from_flags    BITMAP     yes  1
 *   CopyBitmapRangeToBitmap / ...Negated                    :577-601   ytgpu_build_bitmap_from_flags    BITMAP     no   0 / 1
 *   BuildNullBytemapFromDictionaryIndexesWithZeroNull       :350-364   ytgpu_build_bytemap_from_flags   DICT_ZERO  no   0
 *   BuildNullBytemapFromRleDictionaryIndexesWithZeroNull    :366-382   ytgpu_build_bytemap_from_flags   DICT_ZERO  yes  0
 *   BuildNullBytemapFromRleNullBitmap                       :638-652   ytgpu_build_bytemap_from_flags   BITMAP     yes  0
 *   DecodeBytemapFromBitmap                                 :603-621   ytgpu_build_bytemap_from_flags   BITMAP     no   0
 *   CountNullsInDictionaryIndexesWithZeroNull               :454-466   ytgpu_count_flags                DICT_ZERO  no
 *   CountNullsInRleDictionaryIndexesWithZeroNull            :468-493   ytgpu_count_flags                DICT_ZERO  yes
 *   CountOnesInBitmap                                       :495-548   ytgpu_count_flags                BITMAP     no
 *   CountOnesInRleBitmap                                    :550-575   ytgpu_count_flags                BITMAP     yes
 *   BuildDictionaryIndexesFromDictionaryIndexesWithZeroNull :384-398   ytgpu_build_dictionary_indexes   (rle_indexes NULL)
 *   BuildDictionaryIndexesFromRleDictionaryIndexesWithZeroNull :400-420 ytgpu_build_dictionary_indexes
 *   BuildIotaDictionaryIndexesFromRleIndexes                :422-452   ytgpu_build_dictionary_indexes   (dictionary_indexes NULL)
 *   CountTotalStringLengthInRleDictionaryIndexesWithZeroNull :709-735  ytgpu_count_total_string_length
 *   TranslateRleIndex / ...StartIndex / ...EndIndex         :737-768   ytgpu_translate_rle_indexes
 *
 * Rows [start_index, end_index) are produced.  Bitmaps are written as GetBitmapByteSize(end - start) bytes, the unused
 * bits of the last byte zero; bytes behind them are not touched.  Bytemap bytes are 0 / 1.  YT_VERIFY conditions of the
 * reference (negative or reversed ranges, rle_indexes[0] != 0, ranges past the data) come back as
 * YTGPU_ERR_INVALID_ARGUMENT. */
typedef enum ytgpu_flag_kind {
    YTGPU_FLAGS_DICTIONARY_ZERO = 0, /* flag(i) = (dictionary_indexes[k(i)] == 0); data = uint32 indexes */
    YTGPU_FLAGS_BITMAP = 1           /* flag(i) = bit k(i) of a TBitmap; data = bitmap bytes */
} ytgpu_flag_kind;

typedef struct ytgpu_flag_source {
    int32_t kind;                /* ytgpu_flag_kind */
    int32_t reserved;
    const void* data;
    uint64_t data_count;         /* number of dictionary indexes | number of BITS in the bitmap */
    const uint64_t* rle_indexes; /* nullable: k(i) = i; else k(i) = TranslateRleIndex(rle_indexes, i), rle_indexes[0] == 0 */
    uint64_t rle_count;
} ytgpu_flag_source;

/* `mem` names the space of every buffer of the call (source data, rle indexes, dst); counts are returned to the host. */
int ytgpu_build_bitmap_from_flags(ytgpu_context* ctx, const ytgpu_flag_source* source, int64_t start_index, int64_t end_index,
                                  int negate, uint8_t* dst, int mem, ytgpu_error* err);
int ytgpu_build_bytemap_from_flags(ytgpu_context* ctx, const ytgpu_flag_source* source, int64_t start_index, int64_t end_index,
                                   int negate, uint8_t* dst, int mem, ytgpu_error* err);
int ytgpu_count_flags(ytgpu_context* ctx, const ytgpu_flag_source* source, int64_t start_index, int64_t end_index,
                      int64_t* out_count, int mem, ytgpu_error* err);
/* dst[i - start] = dictionary_indexes[k(i)] - 1 (a null becomes 0xFFFFFFFF); dictionary_indexes == NULL: the number of
 * the run holding row i, counted from the run holding start_index (rle_indexes required). */
int ytgpu_build_dictionary_indexes(ytgpu_context* ctx, const uint32_t* dictionary_indexes, uint64_t dictionary_index_count,
                                   const uint64_t* rle_indexes, uint64_t rle_count, int64_t start_index, int64_t end_index,
                                   uint32_t* dst, int mem, ytgpu_error* err);
/* sum over rows [start, end) of string_lengths[dictionary_indexes[k(i)] - 1], nulls counting 0. */
int ytgpu_count_total_string_length(ytgpu_context* ctx, const uint32_t* dictionary_indexes, const uint64_t* rle_indexes,
                                    uint64_t rle_count, const int32_t* string_lengths, uint64_t string_count,
                                    int64_t start_index, int64_t end_index, int64_t* out_total, int mem, ytgpu_error* err);
/* out[j] = TranslateRleIndex(rle_indexes, indexes[j]) (end_flavour 0; also TranslateRleStartIndex) or
 * TranslateRleEndIndex(rle_indexes, indexes[j]) (end_flavour 1). */
int ytgpu_translate_rle_indexes(ytgpu_context* ctx, const uint64_t* rle_indexes, uint64_t rle_count, const int64_t* indexes,
                                uint64_t count, int end_flavour, int64_t* out, int mem, ytgpu_error* err);

/* ---- scan -> filter -> GROUP BY key: SUM(val), COUNT(*) ----
 * Replaces the scan loop + hash aggregation of
 *   CHYT: TSecondaryQuerySourceBase::generate (yt/chyt/server/secondary_query_source.cpp:293-400) feeding
 *         DB::Aggregator::executeOnBlock (key64, AggregateFunctionSum/Count), and
 *   YT QL: ScanOpHelper/GroupOpHelper/InsertGroupRow (library/query/engine/cg_routines/registry.cpp:315-438,
 *         1783-1920) with the `sum` aggregate (engine/udf/sum.c:12-36).
 * Semantics: NULL key is its own group; SUM skips nulls and is NULL when no non-null value was seen;
 * integer SUM wraps mod 2^64; COUNT(*) counts every row that passes the filter. */
typedef enum ytgpu_cmp_op {
    YTGPU_CMP_NONE = 0, YTGPU_CMP_LT = 1, YTGPU_CMP_LE = 2, YTGPU_CMP_GT = 3, YTGPU_CMP_GE = 4,
    YTGPU_CMP_EQ = 5, YTGPU_CMP_NE = 6
} ytgpu_cmp_op;

typedef struct ytgpu_predicate {
    int32_t op;        /* compares the VALUE column with `constant`; a null value never passes */
    int32_t reserved;
    uint64_t constant; /* bit pattern in the column's value type */
} ytgpu_predicate;

typedef struct ytgpu_groupby_result {
    uint64_t group_count;
    uint64_t* keys;          /* [capacity] */
    uint8_t* key_null;       /* [capacity] */
    uint64_t* sums;          /* [capacity] bit patterns in the value type */
    uint8_t* sum_null;       /* [capacity] */
    uint64_t* counts;        /* [capacity] */
    uint64_t capacity;       /* in: allocated groups; YTGPU_ERR_INVALID_ARGUMENT if exceeded */
    uint64_t* first_rows;    /* [capacity], nullable: index (inside the batch) of the first row of every group.
                                YT QL emits groups in first-seen order (InsertGroupRow, cg_routines/registry.cpp:
                                1571-1655): sort the result by first_rows to reproduce it */
    uint64_t* mins;          /* [capacity], nullable: MIN(value) / MAX(value) of every group over its non-NULL values that */
    uint64_t* maxs;          /* passed the predicate, bit patterns in the value type; 0 where sum_null is set (the
                                aggregate is NULL: udf/min.c:21-56, max.c).  Integers: exact.  Doubles are ordered like
                                AggLess (mkql_block_agg_minmax.cpp:20-31): NaN is the biggest value (returned as the
                                canonical quiet NaN); -0.0 orders below +0.0 (the reference keeps whichever zero its row
                                order met last).  Either pointer may be given alone. */
} ytgpu_groupby_result;

/* Groups are emitted ordered by (key_null, key) — ClickHouse's order is hash-table order (unspecified), QL's is
 * first-seen: pass out->first_rows to get every group's first row index and order by it.
 * group_count_hint is a HINT (expected number of groups, 0 = unknown): it sizes the hash table; when the table turns
 * out too small the pass is repeated with a doubled table, it never fails because of the hint.  Hints up to 2048 use a
 * shared-memory front table per CTA. */
int ytgpu_scan_filter_groupby(ytgpu_context* ctx, const ytgpu_column_view* key_column,
                              const ytgpu_column_view* value_column, const ytgpu_predicate* predicate,
                              uint64_t group_count_hint, ytgpu_groupby_result* out, int out_mem,
                              ytgpu_error* err);

/* ---- GROUP BY over a key TUPLE with a LIST of aggregates (the general form of the call above) ----
 * Replaces GroupOpHelper / InsertGroupRow with several group items and aggregate items (registry.cpp:1571-1655,1783-1920;
 * aggregates of library/query/base/builtin_function_types.cpp:201-254: sum, min, max — engine/udf/sum.c, min.c, max.c —,
 * avg, argmin, argmax — engine/builtin_function_profiler.cpp:1300-1620 —, first — registry.cpp:3633-3693 — and count),
 * ClickHouse's Aggregator over a multi-column key and YQL's BlockCombineHashed over tuple keys
 * (mkql_block_agg.cpp:1234-1400).  Semantics, per aggregate, over the rows of a group that passed the predicate:
 *   SUM    skips NULLs, NULL when no value was seen; integers wrap mod 2^64; doubles are added in arbitrary order
 *   MIN / MAX  skip NULLs, NULL without values; doubles ordered like AggLess (NaN is the biggest, -0.0 < +0.0)
 *   COUNT  number of non-NULL values of the column (COUNT(*) is out->counts)
 *   AVG    double(sum) / double(count of non-NULL values), NULL without values; result bits are a double
 *   ARGMIN / ARGMAX  value of `column` in the FIRST row (smallest index) that attains MIN / MAX of `by_column` among the
 *          rows where both are non-NULL (the reference replaces its state only on a strict comparison)
 *   FIRST  the first non-NULL value of the column
 * Key columns are compared as (is-null, 64-bit payload) tuples — doubles by bit pattern.  Groups are emitted in
 * FIRST-SEEN order (QL's order; ClickHouse's is unspecified).  At most 8 key columns, 32 aggregates, 2^30 rows per call. */
typedef enum ytgpu_agg_op {
    YTGPU_AGG_SUM = 0, YTGPU_AGG_MIN = 1, YTGPU_AGG_MAX = 2, YTGPU_AGG_COUNT = 3, YTGPU_AGG_AVG = 4,
    YTGPU_AGG_ARGMIN = 5, YTGPU_AGG_ARGMAX = 6, YTGPU_AGG_FIRST = 7
} ytgpu_agg_op;

typedef struct ytgpu_aggregate {
    int32_t op;         /* ytgpu_agg_op */
    int32_t column;     /* index into value_columns (++ string_columns, see ytgpu_scan_filter_groupby_multi_strings):
                           the aggregated (argmin / argmax: the returned) column */
    int32_t by_column;  /* argmin / argmax: the column that is minimised / maximised */
    int32_t reserved;
} ytgpu_aggregate;

typedef struct ytgpu_groupby_multi_result {
    uint64_t group_count;        /* out */
    uint64_t capacity;           /* in: entries of every output array; INVALID_ARGUMENT if exceeded */
    uint64_t* const* keys;       /* host array of key_count arrays [capacity] */
    uint8_t* const* key_null;    /* host array of key_count arrays [capacity] */
    uint64_t* const* values;     /* host array of aggregate_count arrays [capacity]: bit patterns in the result type */
    uint8_t* const* value_null;  /* host array of aggregate_count arrays [capacity] */
    uint64_t* counts;            /* [capacity], nullable: COUNT(*) */
    uint64_t* first_rows;        /* [capacity], nullable: index of the group's first row (ascending in the output) */
} ytgpu_groupby_multi_result;

/* predicate (nullable) compares value_columns[predicate_column]; a NULL there never passes.  All columns hold the
 * same number of rows.  group_count_hint as above (0 = unknown). */
int ytgpu_scan_filter_groupby_multi(ytgpu_context* ctx, const ytgpu_column_view* key_columns, uint32_t key_count,
                                    const ytgpu_column_view* value_columns, uint32_t value_count,
                                    const ytgpu_aggregate* aggregates, uint32_t aggregate_count,
                                    const ytgpu_predicate* predicate, int32_t predicate_column, uint64_t group_count_hint,
                                    ytgpu_groupby_multi_result* out, int out_mem, ytgpu_error* err);

/* A flat string column, as ytgpu_extract_column, ytgpu_string_value_ids and ytgpu_encode_string_column take it: value i is
 * the lengths[i] bytes at heap + starts[i]; a NULL row (null_bytemap[i] != 0) ignores its start and length. */
typedef struct ytgpu_string_column {
    const uint8_t* heap;          /* string bytes */
    uint64_t heap_bytes;
    const uint64_t* starts;       /* row_count entries: byte offset of the value in heap */
    const uint32_t* lengths;      /* row_count entries */
    const uint8_t* null_bytemap;  /* nullable; 1 = NULL (start / length ignored) */
    uint64_t row_count;
    int32_t mem;                  /* ytgpu_mem of every pointer above */
    int32_t reserved;
} ytgpu_string_column;

/* ytgpu_scan_filter_groupby_multi with string-valued aggregates (YT QL's min / max / first / argmin / argmax / count over
 * strings: builtin_function_types.cpp:201-254, the string branches of engine/udf/min.c and max.c,
 * builtin_function_profiler.cpp:1442-1482).  An aggregate's `column` and `by_column` index value_columns ++ string_columns:
 * index value_count + i is string_columns[i].  The predicate column must be a value column; a string GROUP BY key is passed
 * as the ids of ytgpu_string_value_ids in key_columns.  Strings are ordered as in QL: unsigned bytes over the common prefix,
 * then the shorter value first.  Over a string column:
 *   MIN / MAX  skip NULLs, NULL without values
 *   COUNT      number of non-NULL values
 *   FIRST      the first non-NULL value
 *   ARGMIN / ARGMAX  `column`, `by_column` or both may be strings; the first row (smallest index) that attains the bound wins
 *   SUM / AVG  YTGPU_ERR_UNSUPPORTED
 * A string-valued result (MIN, MAX, FIRST of a string column; ARGMIN / ARGMAX whose `column` is a string) is a ROW INDEX:
 * values[a][g] is the row that holds the group's result (read starts / lengths there); value_null as for scalars.  For
 * MIN / MAX it is the smallest row index that holds the value, so the output is deterministic.
 * INVALID_ARGUMENT: a string column whose row_count differs from the key columns, a null starts / lengths, a null heap
 * with heap_bytes > 0, a mem that is neither DEVICE nor HOST, a
 * non-NULL value whose [start, start + length) leaves the heap (checked on the device for the columns the aggregates
 * read; no byte outside the heap is read).  With string_count = 0 this is ytgpu_scan_filter_groupby_multi. */
int ytgpu_scan_filter_groupby_multi_strings(ytgpu_context* ctx, const ytgpu_column_view* key_columns, uint32_t key_count,
                                            const ytgpu_column_view* value_columns, uint32_t value_count,
                                            const ytgpu_aggregate* aggregates, uint32_t aggregate_count,
                                            const ytgpu_predicate* predicate, int32_t predicate_column,
                                            uint64_t group_count_hint, ytgpu_groupby_multi_result* out, int out_mem,
                                            const ytgpu_string_column* string_columns, uint32_t string_count,
                                            ytgpu_error* err);

/* ---- GROUP BY table: kept on the device and updated block by block ----
 * The one-shot GROUP BY above needs every row of a query in one call.  A GROUP BY table accumulates blocks instead: it is
 * created with the key and value types and the aggregate list, each _update folds one block of rows into it, and _result
 * returns the groups so far.  The contract: updates over blocks B1 .. Bm, each with its own predicate, then _result, give
 * exactly what ytgpu_scan_filter_groupby_multi_strings gives over the rows of B1 ++ .. ++ Bm with each block's predicate
 * applied to its own rows: the same groups, the same first-seen order, first_rows as GLOBAL row numbers (the rows of the
 * earlier updates plus the row's index in its block, 64-bit), COUNT(*) and every aggregate with the semantics stated above
 * (NULLs, wrap-around, AggLess for doubles, the first row winning an ARGMIN / ARGMAX tie).  Two exceptions, as for the
 * one-shot call: double SUM / AVG add in any order, and a +-0 MIN / MAX compares by value.
 * Keys.  The key tuple is the key_count numeric keys (INT64 / UINT64 / DOUBLE / BOOLEAN, any encoding the GROUP BY calls
 * take) followed by the string_key_count string keys (flat string columns, HOST or DEVICE): 1 .. 8 components, key_count
 * may be 0.  Keys compare as GROUP BY keys: (is-null, payload), doubles by bit pattern, NULL equals NULL; strings by length
 * and bytes, "" is not NULL.  The table owns its keys: the caller may free a block's buffers once _update returns.
 * Create.  value_types: the types of the value_count value columns every update passes; aggregates over them only (at most
 * 32; string-valued aggregates are UNSUPPORTED here and take ytgpu_groupby_table_create_strings below).  group_count_hint sizes the table (0 = unknown); it grows by doubling.
 * Update.  At most 2^30 rows, checked from the views before any access (UNSUPPORTED); all columns of one length; key and
 * value counts and types must be the table's (INVALID_ARGUMENT); predicate as for the one-shot call.  The table holds fewer
 * than 2^30 groups: an update whose new groups would reach 2^30 together with the table's is UNSUPPORTED.  A refused
 * update leaves the groups and states as they were (a non-NULL string outside its heap is INVALID_ARGUMENT, with no byte
 * outside the heap read, and is found before anything changes).  Updates may follow a refusal.  The string dictionaries
 * keep every distinct non-NULL value an update passed, including the values of rows its predicate dropped and of a block
 * refused for its group count: their memory is bounded by the distinct values seen, not by the groups, and no result
 * shows the extra values.
 * Result.  out as for the one-shot call, with out->keys / key_null for the numeric keys only; string_out[s] per string
 * key: starts / lengths / null_bytemap [capacity] and a heap of heap_capacity bytes, value o at heap + starts[o] (a NULL
 * key has start, length 0).  Capacity protocol: group_count and every heap_bytes are written; a capacity below the group
 * count, or a heap_capacity below heap_bytes, is INVALID_ARGUMENT with nothing written to the outputs, so capacity 0 is
 * the count query.  _result does not
 * change the table: updates may continue after it.  The outputs are in out_mem.
 * Memory.  Per group: 8 B per key component, 4 B of null mask, 16 B of COUNT(*) and first row and 32 B per aggregate, in
 * arrays whose capacity doubles (so up to twice that per group held), and 8 to 16 B of slot table; per string value
 * kept: its bytes, 12 B of start and length (capacity doubling too) and 16 to 32 B of slots.
 * Synchronisations.  Update: one for the block's group count, one for its count of new groups (which sizes the growth),
 * and a closing one; with string keys, one for the bounds checks and one per string key for the number and bytes of new
 * values; the assign step's error word as in the one-shot call.  Result: one for the sort's plan (from 2^18 groups), one for the byte totals and group
 * count, and a closing one.  Errors: a table of another context is INVALID_ARGUMENT; destroy(NULL) is a no-op; destroy a
 * table before its context. */
typedef struct ytgpu_groupby_table ytgpu_groupby_table;

typedef struct ytgpu_groupby_string_keys {
    uint8_t* heap;           /* [heap_capacity]: the emitted values' bytes, in output order */
    uint64_t heap_capacity;  /* in */
    uint64_t heap_bytes;     /* out: bytes the values need */
    uint64_t* starts;        /* [capacity] */
    uint32_t* lengths;       /* [capacity] */
    uint8_t* null_bytemap;   /* [capacity]: 1 = NULL */
} ytgpu_groupby_string_keys;

int ytgpu_groupby_table_create(ytgpu_context* ctx, const uint8_t* key_types, uint32_t key_count, uint32_t string_key_count,
                               const uint8_t* value_types, uint32_t value_count, const ytgpu_aggregate* aggregates,
                               uint32_t aggregate_count, uint64_t group_count_hint, ytgpu_groupby_table** out, ytgpu_error* err);
int ytgpu_groupby_table_update(ytgpu_context* ctx, ytgpu_groupby_table* table, const ytgpu_column_view* key_columns,
                               uint32_t key_count, const ytgpu_string_column* string_keys, uint32_t string_key_count,
                               const ytgpu_column_view* value_columns, uint32_t value_count, const ytgpu_predicate* predicate,
                               int32_t predicate_column, ytgpu_error* err);
int ytgpu_groupby_table_result(ytgpu_context* ctx, const ytgpu_groupby_table* table, ytgpu_groupby_multi_result* out,
                               ytgpu_groupby_string_keys* string_out, uint32_t string_key_count, int out_mem, ytgpu_error* err);
int ytgpu_groupby_table_destroy(ytgpu_groupby_table* table, ytgpu_error* err);

/* GROUP BY tables with string-valued aggregates: MIN / MAX / FIRST / COUNT of a string column and ARGMIN / ARGMAX whose
 * `column`, `by_column` or both are strings, with the semantics of ytgpu_scan_filter_groupby_multi_strings (QL string
 * order, the first row winning a tie).  The table keeps the bytes of every selected string, so the caller may free a
 * block once _update returns.  The calls above are these with string_value_count = 0.
 * Create.  An aggregate's `column` and `by_column` index value_types ++ string_value_count string value columns (index
 * value_count + i is string value i).  SUM / AVG of a string is UNSUPPORTED; an index past both is INVALID_ARGUMENT.
 * Update.  string_values: string_value_count flat string columns (HOST or DEVICE) of the block's length; a count that
 * differs from the table's is INVALID_ARGUMENT.  Every non-NULL value of a string column the aggregates read is
 * bounds-checked, the rows the predicate drops included: one outside its heap is INVALID_ARGUMENT, no byte outside the
 * heap is read, and it is found before the table (its string key dictionaries included) changes.  The predicate column
 * is a value column.
 * Result.  values[a] of a string-valued aggregate (MIN, MAX or FIRST of a string, ARGMIN / ARGMAX whose `column` is a
 * string) is the GLOBAL row number of the selected row, exactly the row index the one-shot call returns over the
 * concatenated blocks (MIN / MAX: the smallest row holding the value); value_null as for scalars.  value_string_out[j],
 * one per string-valued aggregate in aggregate order (string_aggregate_count of them, else INVALID_ARGUMENT), carries the
 * values' bytes in the layout of string_out, under the same capacity protocol: every heap_bytes is written, and a short
 * capacity is INVALID_ARGUMENT with nothing written.
 * Memory.  Per group and string-valued aggregate, 12 B of start and length per kept string (one for MIN / MAX / FIRST,
 * one or two for ARGMIN / ARGMAX: the value and a string bound) in the group-indexed arrays, and the strings' bytes in the
 * aggregate's own heap.  A replaced string's bytes stay there until the heap's used bytes exceed 2 x its live bytes (and
 * 1 MiB): it is then compacted in group-id order into a buffer of the live bytes.  After every update an aggregate's heap
 * holds at most max(2 x live bytes, 1 MiB); during an update, that plus the update's replacements, in a buffer of up to
 * twice its used bytes, plus the compacted copy.
 * Synchronisations.  None more per update: the bytes the replacements append and free are read in the same copy as the
 * count of new groups (string values alone add the bounds-check synchronisation of string keys).  Result: the value
 * heaps' byte totals are read in the same copy as the key heaps'. */
int ytgpu_groupby_table_create_strings(ytgpu_context* ctx, const uint8_t* key_types, uint32_t key_count, uint32_t string_key_count,
                                       const uint8_t* value_types, uint32_t value_count, uint32_t string_value_count,
                                       const ytgpu_aggregate* aggregates, uint32_t aggregate_count, uint64_t group_count_hint,
                                       ytgpu_groupby_table** out, ytgpu_error* err);
int ytgpu_groupby_table_update_strings(ytgpu_context* ctx, ytgpu_groupby_table* table, const ytgpu_column_view* key_columns,
                                       uint32_t key_count, const ytgpu_string_column* string_keys, uint32_t string_key_count,
                                       const ytgpu_column_view* value_columns, uint32_t value_count,
                                       const ytgpu_string_column* string_values, uint32_t string_value_count,
                                       const ytgpu_predicate* predicate, int32_t predicate_column, ytgpu_error* err);
int ytgpu_groupby_table_result_strings(ytgpu_context* ctx, const ytgpu_groupby_table* table, ytgpu_groupby_multi_result* out,
                                       ytgpu_groupby_string_keys* string_out, uint32_t string_key_count,
                                       ytgpu_groupby_string_keys* value_string_out, uint32_t string_aggregate_count, int out_mem,
                                       ytgpu_error* err);

/* ---- hash JOIN: inner, left, left semi and left only equi-joins over key tuples ----
 * The join of YT QL's JoinOpHelper (library/query/engine/cg_routines/registry.cpp), which collects the primary rows' join
 * keys, fetches the foreign rows and joins them row by row through a hash lookup keyed on the join key.  Here the foreign
 * side is always the built one: its key tuples go into the open-addressing table of the GROUP BY calls, every primary row
 * probes it, and the result is a list of (primary row, foreign row) PAIRS; ytgpu_gather_column and
 * ytgpu_gather_string_column turn the pairs into columns every other call takes.
 * Keys.  Key k of the two sides has one value_type: INT64, UINT64, DOUBLE or BOOLEAN, in any encoding the GROUP BY calls take.
 * There is no implicit widening: different types are INVALID_ARGUMENT, the caller casts.  Tuples compare exactly as the GROUP
 * BY calls compare them, as (is-null, 64-bit payload) per column: doubles by bit pattern, so -0.0 does not match +0.0 and a
 * NaN matches only the same NaN bits; NULL EQUALS NULL.  That rule is shared with GROUP BY and with the unversioned value
 * comparator; that YT QL's join lookup treats NULL keys this way is recalled, not read.  The SQL rule of ClickHouse and YQL,
 * where NULL never matches, is the join table's YTGPU_JOIN_NULLS_NEVER_MATCH (below); ytgpu_hash_join keeps the rule above.
 * String keys go through ytgpu_string_value_ids: call it ONCE over one string column holding the F foreign values followed
 * by the P primary values.  Then ids[0, F) is the foreign key column and ids[F, F + P) the primary one, both UINT64 with the
 * null bytemap as their NULLs: equal strings on either side get the same first-row id.  The join itself is numeric only.
 * A join table takes string keys itself (ytgpu_join_table_build_strings, below).
 * Pairs.  INNER: one pair (p, f) for every primary row p and foreign row f with equal key tuples.  LEFT: in addition one pair
 * (p, YTGPU_JOIN_NO_ROW) for every primary row without a match.  The pairs are ordered by ascending primary row, then
 * ascending foreign row, the LEFT pair of an unmatched row at its place: the row-by-row order of JoinOpHelper when the
 * foreign rows come in their fetched order (that order is recalled, not read).  The output is fully deterministic.
 * Capacity protocol (that of ytgpu_evaluate_filter's out_rows): *out_pair_count is always written once the call gets that
 * far.  Both outputs NULL is a count query and launches no write pass; exactly one NULL is INVALID_ARGUMENT.  A
 * pairs_capacity below the count fails with INVALID_ARGUMENT, the count still written.  Outputs are in out_mem.
 * Limits and errors: 1 .. YTGPU_JOIN_MAX_KEYS key columns; at most 2^30 primary rows and 2^30 - 1 foreign rows (slots and
 * rows are 32-bit, and the foreign rows go through the radix sort, which takes fewer than 2^30), checked before any access
 * (UNSUPPORTED); the key columns of one side have one length (INVALID_ARGUMENT); an unknown kind is
 * INVALID_ARGUMENT; a key type other than the four scalars is UNSUPPORTED.
 * ytgpu_hash_join takes INNER and LEFT only (any other kind is INVALID_ARGUMENT); it is the join table below built, probed
 * once and destroyed, with every argument check of both sides made before the first launch.
 * Launches: the build (a decode pass of the foreign keys, one assign pass of the GROUP BY calls, sized for the foreign row count so that no retry is expected,
 * and a read of its error word), one probe kernel over the primary rows, a three-kernel scan of the per-row pair counts and
 * a read of the total; with outputs, a three-kernel scan of the per-key counts and one stable radix sort of the foreign rows
 * by their slot (which reads its plan back once from 2^18 foreign rows) before the probe, the output-partitioned pair write and a closing
 * synchronisation of the context's stream: the outputs are complete when the call returns, whichever stream the caller
 * reads them on (a context may run on a private stream), as with the GROUP BY calls.  HOST inputs are copied to the device
 * first. */
typedef enum ytgpu_join_kind {
    YTGPU_JOIN_INNER = 0,
    YTGPU_JOIN_LEFT = 1,
    YTGPU_JOIN_SEMI = 2,  /* LEFT SEMI: each primary row with at least one match, once (join table only) */
    YTGPU_JOIN_ANTI = 3   /* LEFT ONLY: each primary row without a match, once (join table only) */
} ytgpu_join_kind;
#define YTGPU_JOIN_NO_ROW 0xffffffffu
#define YTGPU_JOIN_MAX_KEYS 8

int ytgpu_hash_join(ytgpu_context* ctx, const ytgpu_column_view* primary_keys, const ytgpu_column_view* foreign_keys,
                    uint32_t key_count, int kind, uint32_t* out_primary_rows, uint32_t* out_foreign_rows,
                    uint64_t pairs_capacity, uint64_t* out_pair_count /* host */, int out_mem, ytgpu_error* err);

/* Join table: the foreign (right) side built once and probed any number of times, one block of primary rows at a time.
 * Build.  foreign_keys as ytgpu_hash_join takes them (1 .. YTGPU_JOIN_MAX_KEYS columns of one length, INT64 / UINT64 / DOUBLE /
 * BOOLEAN in any encoding the GROUP BY calls take, fewer than 2^30 rows, HOST or DEVICE memory).  The table owns a device
 * copy of the foreign key tuples, decoded to 64-bit payloads plus a null mask per row: the caller may free or overwrite the
 * foreign key buffers as soon as the build returns, and no probe reads them.  The build also runs every step that depends
 * on the foreign side only (the assign step of the GROUP BY calls, the per-key counts and their scan, the stable radix
 * sort of the foreign rows by slot), so no probe repeats them.  The table records its context, key count and key types; it
 * is immutable, may be probed from any thread that may use its context, and must be destroyed before its context.
 * NULL rules.  YTGPU_JOIN_NULLS_EQUAL: NULL equals NULL, exactly as ytgpu_hash_join (YT QL).  YTGPU_JOIN_NULLS_NEVER_MATCH:
 * the SQL rule of YQL and ClickHouse, a key tuple with any NULL component matches nothing: such a foreign row does not
 * enter the table, and such a primary row gives no INNER pair, the LEFT pair (p, YTGPU_JOIN_NO_ROW), no SEMI row and an
 * ANTI row.  DOUBLE keys compare by bit pattern under both rules (-0.0 does not match +0.0, a NaN matches only the same
 * NaN bits).  SQL value equality of doubles is not offered; what YQL's map join does with -0.0 and NaN keys is not known
 * here, so a YQL caller with such keys sees this difference: a known limit.
 * Probe.  primary_keys: key_count columns of the table's key count and types, at most 2^30 rows; primary row indexes are
 * the rows of these columns, foreign row indexes the rows of the build's columns.  INNER and LEFT give exactly the pairs
 * and the order of ytgpu_hash_join (ascending primary row, then ascending foreign row; a LEFT miss as (p,
 * YTGPU_JOIN_NO_ROW) at its place) into out_primary_rows / out_foreign_rows.  SEMI and ANTI give ascending primary row
 * indexes in out_primary_rows; out_foreign_rows must be NULL.  Capacity protocol of ytgpu_hash_join: *out_count is
 * written once the call gets that far; no outputs is a count query; a capacity below the count is INVALID_ARGUMENT with the
 * count written.  A SEMI / ANTI count is at most the primary row count, so that capacity always suffices.
 * Errors.  INVALID_ARGUMENT: a null context, table or argument; a table of another context; a key count or key type
 * other than the table's; an unknown kind or NULL rule; a SEMI / ANTI probe with out_foreign_rows, an INNER / LEFT one
 * with exactly one output.  UNSUPPORTED: a side over its row limit (checked from the views, before any access) or a key
 * type other than the four scalars.  ytgpu_join_table_destroy(NULL) is a no-op.
 * Synchronisations.  Build: the read of the assign step's error word (again when a full table doubles), the sort's plan
 * read from 2^18 foreign rows, and a closing synchronisation.  SEMI / ANTI probe: one read-back (the row count, after the
 * rows are listed), and a copy after it when out_mem is HOST or the capacity is below the primary row count.  INNER /
 * LEFT probe: the read of the pair count and, with outputs, a closing synchronisation.  Bit-packed DEVICE columns cost one
 * more read of their header word, as in every call. */
typedef enum ytgpu_join_nulls {
    YTGPU_JOIN_NULLS_EQUAL = 0,       /* QL: NULL equals NULL, exactly as ytgpu_hash_join */
    YTGPU_JOIN_NULLS_NEVER_MATCH = 1  /* SQL: a key tuple with any NULL component matches nothing */
} ytgpu_join_nulls;
typedef struct ytgpu_join_table ytgpu_join_table;

int ytgpu_join_table_build(ytgpu_context* ctx, const ytgpu_column_view* foreign_keys, uint32_t key_count, int nulls,
                           ytgpu_join_table** out, ytgpu_error* err);
int ytgpu_join_table_probe(ytgpu_context* ctx, const ytgpu_join_table* table, const ytgpu_column_view* primary_keys,
                           uint32_t key_count, int kind, uint32_t* out_primary_rows, uint32_t* out_foreign_rows,
                           uint64_t capacity, uint64_t* out_count /* host */, int out_mem, ytgpu_error* err);
int ytgpu_join_table_destroy(ytgpu_join_table* table, ytgpu_error* err);

/* Join tables with string keys.  The key tuple is the key_count numeric keys followed by the string_key_count string keys
 * (flat string columns, HOST or DEVICE, each with its own heap): 1 .. YTGPU_JOIN_MAX_KEYS components in all, key_count may
 * be 0.  With string_key_count = 0 these are exactly ytgpu_join_table_build / _probe.  Two string values are equal when
 * they have the same length and the same bytes: no collation, and "" is not NULL.  Both NULL rules apply per component, as
 * for numbers.  Pairs, rows, their order, the kinds and the capacity protocol are those of ytgpu_join_table_probe.
 * Build.  The table owns its string keys: the caller may free or overwrite the foreign heaps, starts, lengths and null
 * bytemaps once the build returns.  Per string key it keeps a dictionary in device memory: the bytes of the non-NULL
 * values, compacted; 12 B per foreign row of starts and lengths; and a hash table of a power of two >= 2 x the foreign
 * rows (at least 8) 8-byte slots, 16 to 32 B per row.  Each foreign value becomes the id of the first foreign row with
 * its bytes, and the numeric build runs on those ids.
 * Probe.  primary_keys and primary_string_keys must have the table's numeric key count and types and its string key count.
 * Each primary string value is looked up in its key's dictionary (FNV-1a + mix64 hash, fingerprint, then length and
 * bytes); a value no foreign row holds matches nothing.  Key columns without NULLs (string columns without a null
 * bytemap) keep the probe's fast path.
 * Errors: as ytgpu_join_table_build / _probe, and INVALID_ARGUMENT for a string count other than the table's, string
 * columns whose row_count differs from the other keys', a null starts or lengths, a null heap with heap_bytes > 0, a mem
 * that is neither DEVICE nor HOST, and a non-NULL value whose [start, start + length) leaves its heap (checked on the
 * device for every value on either side: no byte outside a heap is read).  Row limits are checked from the views
 * (row_count without numeric keys), before any access.  After such a refusal the context and the table stay usable.
 * Synchronisations.  Build: one more than ytgpu_join_table_build, which reads the dictionaries' byte totals and the bounds
 * checks together.  Probe: none more; the bounds checks are read with the count. */
int ytgpu_join_table_build_strings(ytgpu_context* ctx, const ytgpu_column_view* foreign_keys, uint32_t key_count,
                                   const ytgpu_string_column* foreign_string_keys, uint32_t string_key_count, int nulls,
                                   ytgpu_join_table** out, ytgpu_error* err);
int ytgpu_join_table_probe_strings(ytgpu_context* ctx, const ytgpu_join_table* table, const ytgpu_column_view* primary_keys,
                                   uint32_t key_count, const ytgpu_string_column* primary_string_keys, uint32_t string_key_count,
                                   int kind, uint32_t* out_primary_rows, uint32_t* out_foreign_rows, uint64_t capacity,
                                   uint64_t* out_count /* host */, int out_mem, ytgpu_error* err);

/* Gathers.  ytgpu_gather_column decodes `column` at rows[i] into out_values[i] and bit i of out_null_bitmap, for i < count,
 * in the layout of ytgpu_evaluate_expression: out_values count 64-bit bit patterns (a NULL row holds 0), out_null_bitmap
 * 8 * ceil(count / 64) bytes (LSB first, the bits past count zero), *out_null_count (host, nullable) the NULL rows.  So
 * {value_type = column->value_type, bit_width = 64, has_values = 1, values = out_values, values_count = count, value_count
 * = count, null_bitmap = out_null_bitmap} is a column every other call takes.  rows[i] = YTGPU_JOIN_NO_ROW gives NULL: that
 * is how the missing foreign side of a LEFT join becomes NULL.
 * ytgpu_gather_string_column gathers starts, lengths and the null bytemap (count entries each; a NULL row gets start 0,
 * length 0, null byte 1).  The heap is not copied: {column->heap, column->heap_bytes, out_starts, out_lengths,
 * out_null_bytemap, count, out_mem} is the gathered column.  rows, like the outputs, are in out_mem; the column in its own.
 * INVALID_ARGUMENT: a row index neither below the column's length (value_count / row_count) nor YTGPU_JOIN_NO_ROW (checked
 * on the device: no byte outside the column is read), a null output, a column as the other calls refuse it.  UNSUPPORTED: a
 * value_type other than INT64, UINT64, DOUBLE or BOOLEAN.  One gather kernel, then one read of the error word (and the NULL
 * count).  out_null_bitmap is written in 4-byte words: 4-byte aligned in DEVICE memory. */
int ytgpu_gather_column(ytgpu_context* ctx, const ytgpu_column_view* column, const uint32_t* rows /* out_mem */,
                        uint64_t count, uint64_t* out_values, uint8_t* out_null_bitmap,
                        uint64_t* out_null_count /* host, nullable */, int out_mem, ytgpu_error* err);

int ytgpu_gather_string_column(ytgpu_context* ctx, const ytgpu_string_column* column, const uint32_t* rows /* out_mem */,
                               uint64_t count, uint64_t* out_starts, uint32_t* out_lengths, uint8_t* out_null_bytemap,
                               int out_mem, ytgpu_error* err);

/* ---- ORDER BY ... OFFSET ... LIMIT over typed columns ----
 * The order of YT QL's OrderOpHelper (library/query/engine/cg_routines/registry.cpp:1948) and its TTopCollector
 * (engine_api/top_collector.h), computed as ONE stable sort of the rows being ordered followed by a window.
 * Inputs.  Item k names columns[column] (INT64, UINT64, DOUBLE or BOOLEAN, in any encoding the GROUP BY calls take:
 * plain widths, bit-packed, dictionary, RLE, boolean bitmap, Arrow validity, start_index windows) or, with is_string,
 * string_columns[column] (flat string columns; each may have its own heap).  Every item column holds the same number of
 * rows L.  Columns not named by an item are not read.
 * Order.  Items are compared in turn, each in the unversioned value order of ytgpu_sort_rowset (compare-inl.h:49-66):
 * NULL below every value; false below true; a NaN above +inf, all NaNs equal; -0.0 equal to +0.0; strings as unsigned
 * bytes, a prefix first.  `descending` reverses one item, its NULLs then come last.  Rows equal on every item keep their
 * order in `rows` (ascending row index when `rows` is NULL): the sort is stable, which is one of the orders the
 * reference's heap may produce.  That QL's generated ORDER BY comparer orders NaN and NULL this way is recalled, not read.
 * Output.  out_rows[i] is the ROW INDEX (not the position in `rows`) of the row at position offset + i of that order,
 * for i < *out_count = min(limit, row_count - min(offset, row_count)).  out_rows NULL is a count query: *out_count is
 * written and nothing is launched; so is a window of 0 rows (limit == 0, offset >= row_count).
 * Limits and errors.  row_count < 2^30 (the radix sort's bound), checked before any access: UNSUPPORTED otherwise.
 * 1 .. 32 items.  INVALID_ARGUMENT: a row index >= L (checked on the device, no byte outside a column is read); item
 * columns of different lengths; an item naming a missing column; a non-zero `reserved`; a null out_count; a string
 * value whose [start, start + length) leaves its heap (checked on the device).  UNSUPPORTED: another value type.
 * Memory and launches.  `rows` and out_rows are in out_mem, each column in its own mem (HOST columns are copied to the
 * device first).  One kernel writes the rows in `rows` order as a device rowset of item_count values each (numeric
 * items decoded, string starts rebased into one heap: the string heaps concatenated), the stable sort of
 * ytgpu_sort_rowset runs over it (keys of any length, "last_sort_refine_rounds" as there), one kernel writes the window.
 * The call synchronises the context's stream before returning. */
typedef struct ytgpu_order_item {
    uint32_t column;     /* index into columns[], or into string_columns[] when is_string */
    uint8_t is_string;
    uint8_t descending;
    uint16_t reserved;   /* 0 */
} ytgpu_order_item;

int ytgpu_order_rows(ytgpu_context* ctx, const ytgpu_column_view* columns, uint32_t column_count,
                     const ytgpu_string_column* string_columns, uint32_t string_column_count,
                     const ytgpu_order_item* items /* host */, uint32_t item_count,
                     const uint32_t* rows /* out_mem, nullable: rows 0 .. row_count - 1 */, uint64_t row_count,
                     uint64_t offset, uint64_t limit, uint32_t* out_rows, uint64_t* out_count /* host */,
                     int out_mem, ytgpu_error* err);

/* ---- WHERE expressions: a selection over several columns ----
 * The filter of YT QL's ScanOpHelper / FilterOpHelper (the WHERE clause compiled by the query evaluator) and of
 * ClickHouse's FilterTransform, for expressions built of comparisons, IN lists, NULL tests, prefix and substring tests and
 * LIKE patterns joined by AND / OR / NOT.  A filter is a PROGRAM of nodes in POSTFIX order; a row is selected iff the program evaluates to TRUE
 * under three-valued (Kleene) logic:
 *   COMPARE(column, cmp, constant)        NULL if the value is NULL; otherwise the comparison of the built-in predicate:
 *                                         INT64 signed, UINT64 unsigned, DOUBLE by IEEE (a NaN operand makes every op false
 *                                         except NE; -0.0 == +0.0), BOOLEAN 0 < 1.  STRING: unsigned bytes over the common
 *                                         prefix, then the shorter value first (QL's string order).
 *   COMPARE_COLUMNS(column, cmp, column2) NULL if either value is NULL, otherwise as above.  Both columns have the same
 *                                         type (both strings, or the same value_type).
 *   IN(column, list)                      NULL if the value is NULL; TRUE if it equals an entry by the EQ rule above (a NaN
 *                                         entry never matches), else FALSE.  The list holds no NULL: write
 *                                         is_null(c) OR c IN (...) instead.
 *   STARTS_WITH(column, prefix)           string columns only (QL is_prefix, ClickHouse startsWith): NULL if the value is
 *                                         NULL, else whether its first len(prefix) bytes are the prefix.  An empty prefix
 *                                         matches every non-NULL value.
 *   CONTAINS(column, needle)              string columns only (QL is_substr(needle, s), ClickHouse position(s, needle) > 0):
 *                                         NULL if the value is NULL, else whether the needle occurs in the value as a
 *                                         contiguous byte sequence.  An empty needle matches every non-NULL value.
 *   LIKE(column, pattern, escape)         string columns only: NULL if the value is NULL, else whether the WHOLE value
 *                                         matches the pattern.  NOT LIKE is LIKE followed by NOT.  Pattern bytes:
 *                                           %  matches any byte sequence, including the empty one;
 *                                           _  matches one character: one byte outside 0x80..0xBF, followed by any number
 *                                              of bytes in 0x80..0xBF;
 *                                           any other byte matches itself;
 *                                           with an escape byte E (column2 = 0..255; -1: no escape), E followed by any
 *                                           byte X matches X literally.  A pattern that ends in a lone E is an error.
 *                                         A match exists iff some split of the value satisfies the pattern: as a regular
 *                                         expression over bytes, fully matched, % is [\x00-\xff]*, _ is
 *                                         [^\x80-\xbf][\x80-\xbf]* and every other byte is itself.  Newlines are ordinary
 *                                         bytes and matching is case-sensitive.  When the value and the pattern are valid
 *                                         UTF-8 this is exactly "_ = one code point, % = any code-point sequence", the rule
 *                                         ClickHouse documents for LIKE.  YT QL's like compiles to an RE2 expression; how
 *                                         that treats _ on multibyte input and whether % / _ cross a newline (RE2's dot_nl)
 *                                         was not read in the reference, so those two rules are unverified against YT QL.
 *                                         Work per row is bounded: the pattern is split at % into segments, each segment is
 *                                         an NFA run bit-parallel (Shift-And) over ceil(positions / 64) 64-bit words, and
 *                                         every middle segment takes its earliest end (the next % absorbs any gap).  Each
 *                                         value byte is consumed by at most one segment scan, so a row costs at most
 *                                         (value length) * ceil(positions / 64) + segments steps, whatever the pattern: no
 *                                         backtracking.  CONTAINS(x) is compiled as the pattern %x% without wildcards.
 *   IS_NULL(column), IS_NOT_NULL(column)  never NULL.  NULL is what the group-by calls take as NULL: a dictionary index of
 *                                         0, a null bit or Arrow validity bit, has_values = 0; the null bytemap of a string
 *                                         column.
 *   AND, OR, NOT                          Kleene: F AND x = F, T OR x = T, NOT N = N; every other combination with a NULL
 *                                         operand is NULL.
 * A one-node COMPARE program selects exactly the rows the built-in ytgpu_predicate passes.  These NULL rules are the
 * SQL ones; they were not checked against YT QL's own evaluator.
 *
 * Node fields by op:
 *   column     index into columns ++ string_columns (column_count + i is string_columns[i]), as ytgpu_aggregate::column
 *   cmp        ytgpu_cmp_op, LT .. NE (COMPARE, COMPARE_COLUMNS)
 *   column2    COMPARE_COLUMNS: the right-hand column; LIKE: the escape byte 0..255, or -1 for none
 *   constant   COMPARE on a scalar column: the bit pattern in the column's type (length must be 0);
 *              COMPARE / STARTS_WITH / CONTAINS / LIKE on a string column: byte offset of the constant (prefix, needle,
 *              pattern) in string_constants, `length` bytes;
 *              IN: index of the first entry in list_values, `length` entries.  A scalar column's entries are bit patterns
 *              in its type; a string column's are (offset << 32) | length into string_constants.
 * Limits: 1 .. 64 nodes and a stack depth of at most 16; at most 65536 IN entries over all IN nodes of a call; at most
 * 1 MiB of string_constants; fewer than 2^32 rows, and every column (value_count) and string column (row_count) holds
 * the same number of rows.  Scalar columns are INT64, UINT64, DOUBLE or BOOLEAN.
 * Pattern limits (CONTAINS and LIKE): at most YTGPU_FILTER_MAX_PATTERN_POSITIONS (256) positions per pattern, a position
 * being one literal byte (an escaped byte included) or one _, so a pattern state is at most 4 words; a CONTAINS needle has
 * one position per byte.  The patterns of a call compile to at most YTGPU_FILTER_MAX_PATTERN_BYTES (32 KiB), all staged
 * in shared memory; a pattern with W = ceil(positions / 64) words (W = 1 when it has no position), S non-empty segments
 * and C byte classes takes 272 + 8 * S + 8 * W * (C + 1) bytes, where C is the number of distinct literal bytes, plus one
 * if some byte outside 0x80..0xBF is not among them, plus one if some byte in 0x80..0xBF is not among them.  A realistic
 * 200-byte URL pattern of 40 distinct bytes takes about 2.6 KB.
 * Outputs, each nullable, in out_mem:
 *   out_bitmap   8 * ceil(n / 64) bytes; bit i (LSB first) = row i selected, the bits past n zero.  So
 *                {value_type = BOOLEAN, bit_width = 1, has_values = 1, values = out_bitmap, values_count = n, value_count = n}
 *                is a column the GROUP BY calls aggregate the selected rows of with the predicate {YTGPU_CMP_EQ, 1}.
 *   out_bytemap  n bytes of 0 / 1: ClickHouse's IColumn::Filter, also the filter_hint of the string column conversion.
 *   out_rows     the selected row indexes in ascending order, rows_capacity entries.
 *   *out_selected (host) the number of selected rows; always written when the call gets that far.
 * Launches: without out_rows one evaluation kernel and one read of the count and the error word; with out_rows four
 * more (an exclusive scan of the per-32-row counts and the row write).  HOST inputs are copied to the device first.
 * YTGPU_ERR_INVALID_ARGUMENT: a malformed program (stack underflow, other than one value left, an unknown op or cmp, a
 * column out of range), STARTS_WITH, CONTAINS, LIKE or a non-zero `length` on a scalar column, COMPARE_COLUMNS over
 * different types, a constant or list range outside its buffer, a LIKE escape outside -1..255, a LIKE pattern that ends in
 * a lone escape byte, a limit above, rows_capacity below the selected count (the count is still in
 * *out_selected), a non-NULL string that leaves its heap (checked on the device for the string columns the program reads;
 * no byte outside the heap is read).  YTGPU_ERR_UNSUPPORTED: a scalar column of another type. */
typedef enum ytgpu_filter_op {
    YTGPU_FILTER_COMPARE = 1, YTGPU_FILTER_COMPARE_COLUMNS = 2, YTGPU_FILTER_IN = 3, YTGPU_FILTER_STARTS_WITH = 4,
    YTGPU_FILTER_IS_NULL = 5, YTGPU_FILTER_IS_NOT_NULL = 6, YTGPU_FILTER_AND = 7, YTGPU_FILTER_OR = 8, YTGPU_FILTER_NOT = 9,
    YTGPU_FILTER_CONTAINS = 10, YTGPU_FILTER_LIKE = 11
} ytgpu_filter_op;

#define YTGPU_FILTER_MAX_NODES 64
#define YTGPU_FILTER_MAX_DEPTH 16
#define YTGPU_FILTER_MAX_IN_ENTRIES 65536
#define YTGPU_FILTER_MAX_STRING_CONSTANT_BYTES (1u << 20)
#define YTGPU_FILTER_MAX_PATTERN_POSITIONS 256
#define YTGPU_FILTER_MAX_PATTERN_BYTES 32768

typedef struct ytgpu_filter_node {
    int32_t op;         /* ytgpu_filter_op */
    int32_t cmp;        /* ytgpu_cmp_op: COMPARE, COMPARE_COLUMNS */
    int32_t column;     /* index into columns ++ string_columns */
    int32_t column2;    /* COMPARE_COLUMNS: a column; LIKE: the escape byte or -1 */
    uint64_t constant;  /* see above */
    uint32_t length;    /* string constant: bytes; IN: number of entries */
    uint32_t reserved;
} ytgpu_filter_node;

int ytgpu_evaluate_filter(ytgpu_context* ctx, const ytgpu_column_view* columns, uint32_t column_count,
                          const ytgpu_string_column* string_columns, uint32_t string_count,
                          const ytgpu_filter_node* program /* host */, uint32_t node_count,
                          const uint64_t* list_values /* host */, uint64_t list_value_count,
                          const uint8_t* string_constants /* host */, uint64_t string_constant_bytes,
                          uint8_t* out_bitmap, uint8_t* out_bytemap, uint32_t* out_rows, uint64_t rows_capacity,
                          uint64_t* out_selected /* host */, int out_mem, ytgpu_error* err);

/* ---- computed columns: arithmetic, bitwise, cast, if_null and conditional expressions ----
 * The projections of YT QL's expression compiler (cg_fragment_compiler.cpp) that a GROUP BY key (`group by a % 2`), an
 * aggregate argument (`sum(price * qty)`) or a WHERE leaf (`a + b > 10`) may hold.  An expression is a PROGRAM of nodes in
 * POSTFIX order, evaluated row by row into a computed column.  The program is typed: the type of every node follows from the
 * column types, the constants' types and the CAST targets, and is checked before the launch.
 *   COLUMN(column)           the row's value of columns[column]: INT64, UINT64, DOUBLE or BOOLEAN, in any encoding the
 *                            GROUP BY calls take (a BOOLEAN payload other than 0 is read as 1)
 *   CONSTANT(type, constant) the bit pattern `constant` of type INT64, UINT64, DOUBLE or BOOLEAN (0 / 1)
 *   ADD, SUB, MUL, DIV       two operands of one type INT64, UINT64 or DOUBLE; the result has that type
 *   MOD                      two operands of one type INT64 or UINT64
 *   NEG                      one operand INT64, UINT64 or DOUBLE
 *   BIT_AND, BIT_OR, BIT_XOR two operands of one type INT64 or UINT64; BIT_NOT one
 *   CAST(type)               one operand of any of the four types to INT64, UINT64 or DOUBLE
 *   IF_NULL                  two operands of one type, any of the four
 * There is no implicit widening (QL has none between int64 and uint64): binary operands of different types are an error,
 * the caller inserts CAST.  Semantics:
 *   NULL     a NULL operand makes the result NULL, except IF_NULL(a, b), which is a when a is not NULL and b otherwise.  NULL
 *            is what the GROUP BY calls take as NULL: a null bit, an Arrow validity bit, a dictionary index of 0,
 *            has_values = 0.
 *   integers ADD, SUB, MUL and NEG wrap mod 2^64 (NEG of INT64_MIN is INT64_MIN).  DIV truncates toward zero and MOD has the
 *            sign of the dividend, as C's / and %.  BIT_* act on the 64-bit pattern.
 *   division an integer DIV or MOD by 0 fails the call with YTGPU_ERR_INVALID_ARGUMENT and the message "Division by zero";
 *            INT64_MIN / -1 and INT64_MIN % -1 fail it with "Division INT_MIN by -1".  A row whose divisor or dividend is
 *            NULL, and a row outside the selection, never fails.  After a failure the outputs' contents are unspecified.
 *   doubles  IEEE-754 with round to nearest (x / 0 is +-inf, 0 / 0 is NaN); every operation is rounded on its own, never
 *            contracted into an FMA.  NEG flips the sign bit.  The sign and payload of a NaN that ADD, SUB, MUL or DIV
 *            produces are unspecified (the GPU returns a canonical NaN, not an operand's payload).
 *   CAST     INT64 <-> UINT64 keeps the bits (two's complement); an integer to DOUBLE rounds to nearest; DOUBLE to an integer
 *            truncates toward zero, and an out-of-range value follows PTX's saturating cvt.rzi: a value below / above the
 *            range becomes the type's minimum / maximum.  NaN becomes 0 (tested for explicitly: on sm_90 the 64-bit
 *            cvt.rzi.s64.f64 returns INT64_MIN for it).  The reference compiles this cast with
 *            LLVM fptosi / fptoui, whose result for those inputs is poison, so this rule has no counterpart there.  BOOLEAN
 *            becomes 0 / 1 or 0.0 / 1.0; a cast to the operand's own type is the identity.
 * These rules were not checked against YT QL's own evaluator; in particular the two division-error messages and the
 * INT64_MIN / -1 check are recalled from cg_fragment_compiler.cpp, not read there.
 *
 * Conditional expressions (`sum(if(status = 200, 1, 0))`, `sum(if(b = 0, 0, a / b))`, `group by if(latency > 1000, 'slow',
 * 'fast')`, `group by lower(host) = 'example.com'`), taken by both entry points; STRING operands by
 * ytgpu_evaluate_expression_strings only:
 *   COMPARE(cmp)             two operands of one type, any of the four or STRING, -> BOOLEAN; `column` holds the
 *                            ytgpu_cmp_op LT .. NE.  No implicit widening: the caller casts.  The comparison is the filter's
 *                            COMPARE rule: INT64 signed, UINT64 unsigned, DOUBLE by IEEE (a NaN operand makes every op false
 *                            except NE; -0.0 == +0.0), BOOLEAN 0 < 1, STRING as unsigned bytes, then the shorter value
 *                            first.  NULL if either operand is NULL (the filter's SQL rule).  A STRING operand may be any
 *                            string result (lower(x), concat(a, b), ...): the bytes are compared as they would be written.
 *   AND, OR                  two BOOLEANs -> BOOLEAN, Kleene logic as the filter: F AND x = F, T OR x = T, otherwise a NULL
 *                            operand makes the result NULL.
 *   NOT                      one BOOLEAN -> BOOLEAN; NOT NULL is NULL.
 *   IS_NULL, IS_NOT_NULL     one operand of any type, STRING included -> BOOLEAN, never NULL.
 *   IF                       postfix `c a b IF`: c a BOOLEAN, a and b of one type (STRING included) -> that type: a where c
 *                            is TRUE, b where it is FALSE, NULL where c is NULL.  That a NULL condition gives NULL is
 *                            recalled from QL's TIfFunctionCodegen (builtin_function_profiler.cpp), not read there.
 * Errors follow the data.  Each stack entry carries the errors its value met (a division error; in
 * ytgpu_evaluate_expression_strings also a non-ASCII LOWER / UPPER operand); every op passes on the union of its operands'
 * errors, and only the errors of the program's result fail the call.  The exceptions: IF keeps c's errors and those of the
 * branch it takes (c's alone when c is NULL); AND whose left operand is FALSE and OR whose left operand is TRUE drop the
 * right operand's errors.  So `if(b = 0, 0, a / b)` never fails, `if(b = 0, a / b, 0)` fails where b = 0, `FALSE AND (a /
 * 0 > 1)` never fails and `NULL AND (a / 0 > 1)` does.  A program without IF, AND or OR fails on exactly the rows where
 * any of its divisions (or case maps) fails, as it always has.  A string value outside its heap is an input error and
 * fails the call wherever it is read.
 *
 * selection (nullable, out_mem): a bitmap in the layout of ytgpu_evaluate_filter's out_bitmap.  A row whose bit is clear is
 * not evaluated: its result is NULL and it raises no division error (QL evaluates projections after WHERE, so a division by
 * zero in a row the WHERE drops must not fail the query).
 * Outputs, in out_mem:
 *   out_values      n 64-bit bit patterns in the result type; a NULL row holds 0.
 *   out_null_bitmap 8 * ceil(n / 64) bytes; bit i (LSB first) set when row i is NULL, the bits past n zero.  So
 *                   {value_type = *out_value_type, bit_width = 64, has_values = 1, values = out_values, values_count = n,
 *                   value_count = n, null_bitmap = out_null_bitmap} is a column the GROUP BY, filter and decode calls take.
 *   *out_value_type (host, nullable) the result type, written once the program is checked.
 *   *out_null_count (host, nullable) the number of NULL rows, so a caller may drop the bitmap from the view when it is 0.
 * Launches: one evaluation kernel and one read of the NULL count and the error word.  HOST inputs are copied to the device
 * first.
 * YTGPU_ERR_INVALID_ARGUMENT: a malformed program (stack underflow, other than one value left, a stack deeper than 16, more
 * than 64 nodes, an unknown op or type, a column out of range), operand types an op does not take, a BOOLEAN constant other
 * than 0 / 1, no columns (they give the row count), columns of different lengths, 2^32 rows or more, a division error
 * above.  YTGPU_ERR_UNSUPPORTED: a column of
 * another type (strings included). */
typedef enum ytgpu_expr_op {
    YTGPU_EXPR_COLUMN = 1, YTGPU_EXPR_CONSTANT = 2,
    YTGPU_EXPR_ADD = 3, YTGPU_EXPR_SUB = 4, YTGPU_EXPR_MUL = 5, YTGPU_EXPR_DIV = 6, YTGPU_EXPR_MOD = 7, YTGPU_EXPR_NEG = 8,
    YTGPU_EXPR_BIT_AND = 9, YTGPU_EXPR_BIT_OR = 10, YTGPU_EXPR_BIT_XOR = 11, YTGPU_EXPR_BIT_NOT = 12,
    YTGPU_EXPR_CAST = 13, YTGPU_EXPR_IF_NULL = 14,
    /* ytgpu_evaluate_expression_strings only */
    YTGPU_EXPR_CONCAT = 15, YTGPU_EXPR_LOWER = 16, YTGPU_EXPR_UPPER = 17, YTGPU_EXPR_FARM_HASH = 18,
    /* conditional expressions, both entry points (see below) */
    YTGPU_EXPR_COMPARE = 19, YTGPU_EXPR_AND = 20, YTGPU_EXPR_OR = 21, YTGPU_EXPR_NOT = 22, YTGPU_EXPR_IS_NULL = 23,
    YTGPU_EXPR_IS_NOT_NULL = 24, YTGPU_EXPR_IF = 25,
    /* predicates inside expressions, ytgpu_evaluate_expression_strings only (see there) */
    YTGPU_EXPR_IN = 26, YTGPU_EXPR_STARTS_WITH = 27, YTGPU_EXPR_CONTAINS = 28, YTGPU_EXPR_LIKE = 29,
    /* timestamps: TIMESTAMP_FLOOR both entry points, FORMAT_TIMESTAMP ytgpu_evaluate_expression_strings only (see there) */
    YTGPU_EXPR_TIMESTAMP_FLOOR = 30, YTGPU_EXPR_FORMAT_TIMESTAMP = 31
} ytgpu_expr_op;

/* TIMESTAMP_FLOOR's unit, in the node's `column` */
typedef enum ytgpu_timestamp_unit {
    YTGPU_TIMESTAMP_HOUR = 0, YTGPU_TIMESTAMP_DAY = 1, YTGPU_TIMESTAMP_WEEK = 2, YTGPU_TIMESTAMP_MONTH = 3, YTGPU_TIMESTAMP_YEAR = 4
} ytgpu_timestamp_unit;

#define YTGPU_EXPR_MAX_NODES 64
#define YTGPU_EXPR_MAX_DEPTH 16
#define YTGPU_EXPR_MAX_PIECES 16
#define YTGPU_EXPR_MAX_HASH_OPERANDS 16
#define YTGPU_EXPR_MAX_STRING_CONSTANT_BYTES (1u << 20)
#define YTGPU_EXPR_MAX_FORMATTED_BYTES 64

typedef struct ytgpu_expr_node {
    int32_t op;          /* ytgpu_expr_op */
    int32_t column;      /* COLUMN: index into columns (++ string_columns); FARM_HASH: its operand count;
                            COMPARE: the ytgpu_cmp_op; LIKE: the escape byte 0..255, or -1 for none;
                            TIMESTAMP_FLOOR: the ytgpu_timestamp_unit */
    uint8_t type;        /* CONSTANT: its value type; CAST: the target type (YTGPU_TYPE_*) */
    uint8_t reserved[7];
    uint64_t constant;   /* CONSTANT: the bit pattern in `type`; a STRING one: (offset << 32) | length into string_constants;
                            IN: (offset << 32) | count of its list in string_constants; STARTS_WITH, CONTAINS, LIKE: the
                            prefix, needle or pattern as (offset << 32) | length into string_constants; FORMAT_TIMESTAMP:
                            the format, likewise */
} ytgpu_expr_node;

int ytgpu_evaluate_expression(ytgpu_context* ctx, const ytgpu_column_view* columns, uint32_t column_count,
                              const ytgpu_expr_node* program /* host */, uint32_t node_count,
                              const uint8_t* selection /* nullable, out_mem */, uint64_t* out_values,
                              uint8_t* out_null_bitmap, uint8_t* out_value_type /* host, nullable */,
                              uint64_t* out_null_count /* host, nullable */, int out_mem, ytgpu_error* err);

/* ---- computed string columns: concat, lower, upper, if_null and farm_hash ----
 * ytgpu_evaluate_expression with string leaves and string results: `group by lower(host)`, `group by concat(region, '/',
 * city)`, `group by if_null(campaign, 'none')`, `group by farm_hash(user_id) % 64`, `where farm_hash(k) % 100 < 5`.  The
 * ops are QL's concat / lower / upper / if_null / farm_hash UDFs, recalled, not read.  With string_count = 0 and a program
 * of the ops above (COLUMN .. IF_NULL) this call is exactly ytgpu_evaluate_expression; the string ops and string leaves
 * are taken by this entry point only (ytgpu_evaluate_expression keeps refusing them).
 *   COLUMN(column)           column indexes columns ++ string_columns: column_count + i is string_columns[i], a STRING
 *   CONSTANT(STRING)         `constant` = (offset << 32) | length: the bytes string_constants[offset, offset + length)
 *   CONCAT                   two STRING operands -> STRING, the first one's bytes then the second's
 *   LOWER, UPPER             one STRING -> STRING: ASCII A-Z -> a-z (LOWER) or a-z -> A-Z (UPPER), every other byte kept.
 *                            QL's lower / upper are recalled to map UTF-8 with Unicode case tables, which this library does
 *                            not have; on pure-ASCII values any such mapping agrees with this one.  So an operand with a byte
 *                            >= 0x80 in a row that is evaluated (selected and non-NULL) fails the call with
 *                            YTGPU_ERR_UNSUPPORTED rather than yield a different string; a caller takes its CPU path then.
 *   IF_NULL                  also two STRING operands -> STRING
 *   FARM_HASH(k)             k = `column` in 1 .. YTGPU_EXPR_MAX_HASH_OPERANDS (16) operands of any type, STRING included ->
 *                            UINT64, never NULL: GetFarmFingerprint over the k values in order (the first pushed first),
 *                            bit-identical to ytgpu_farm_fingerprint_rowset over a row of those k values: each value's
 *                            fingerprint (a string's FarmHash Fingerprint64 of its bytes, a number's Fingerprint(uint64) of
 *                            its bits, BOOLEAN as 0 / 1, NULL as Fingerprint(0)) folded from 0xdeadc0de with
 *                            Fingerprint(uint128), then xor k.  That QL's farm_hash(a, b, ...) is GetFarmFingerprint of its
 *                            arguments is recalled from its UDF, not read.  A STRING operand must be a leaf, a constant or
 *                            IF_NULL of those; a CONCAT, LOWER or UPPER result under FARM_HASH is YTGPU_ERR_UNSUPPORTED.
 * NULL: a NULL operand makes CONCAT, LOWER and UPPER NULL; IF_NULL and FARM_HASH as above.  The numeric ops are those of
 * ytgpu_evaluate_expression, and they do not take strings (YTGPU_ERR_UNSUPPORTED).  The conditional ops above take
 * STRING operands here.  There is no substr.
 * Limits: those of ytgpu_evaluate_expression; at most YTGPU_EXPR_MAX_PIECES (16) string pieces on the stack at any node,
 * where a leaf or constant is one piece, CONCAT adds its operands' pieces, IF_NULL and IF take the larger count and
 * COMPARE, IS_NULL and IS_NOT_NULL leave none (so a program concatenates at most 16 values); at most 1 MiB of
 * string_constants; a result value of at most 2^32 - 1 bytes.
 * selection: as ytgpu_evaluate_expression; an unselected row is NULL and not evaluated, so a non-ASCII value or a value
 * outside its heap there does not fail the call.
 * Outputs, in out_mem:
 *   a numeric result  out_values / out_null_bitmap as ytgpu_evaluate_expression; the string outputs are not touched.
 *   a STRING result   out_values / out_null_bitmap are not touched, and
 *     *out_heap_bytes (host)  the bytes of all result values, always written once the program is checked and evaluated;
 *     out_heap                the values back to back in row order (out_heap_capacity bytes).  NULL: a size query that
 *                             writes *out_heap_bytes only, so a caller sizes the heap and calls again;
 *     out_starts (u64), out_lengths (u32), out_null_bytemap (u8), n entries each: value i is the out_lengths[i] bytes at
 *                             out_heap + out_starts[i]; a NULL row has length 0 and null byte 1.  So {out_heap,
 *                             *out_heap_bytes, out_starts, out_lengths, out_null_bytemap, n, out_mem} is the
 *                             ytgpu_string_column that ytgpu_evaluate_filter, ytgpu_string_value_ids and
 *                             ytgpu_scan_filter_groupby_multi_strings take.
 *   *out_value_type, *out_null_count as ytgpu_evaluate_expression.
 *   A first call with out_heap, out_values and out_null_bitmap all NULL is a type and size query: a numeric result is
 *   checked and typed but not evaluated (no launch), a STRING one is sized as above.  A caller that does not know the
 *   result type makes it, then allocates only the outputs that type needs; for a STRING result the second call runs the
 *   size pass again.
 * Launches: a numeric result: one evaluation kernel and one host read, as ytgpu_evaluate_expression (none for a type
 * query).  A STRING result: a
 * size pass and a three-kernel scan of the lengths, then one host read (NULL count, error bits, heap size); with out_heap
 * a fill pass follows (five launches).  HOST inputs are copied to the device first.
 * YTGPU_ERR_INVALID_ARGUMENT: everything ytgpu_evaluate_expression refuses; a new op over a type it does not take, FARM_HASH
 * with k outside 1 .. 16, more than 16 pieces, a string constant outside string_constants or more than 1 MiB of them, a
 * string column of another length, null starts / lengths, a null heap with heap_bytes > 0 or a mem that is neither DEVICE
 * nor HOST, a non-NULL value whose [start, start + length) leaves its heap (checked on the device for the string columns
 * the program reads; no byte outside the heap is read), a result value longer than 2^32 - 1 bytes, out_heap_capacity
 * below the heap size (which is still written), a null out_heap_bytes with a STRING result.  YTGPU_ERR_UNSUPPORTED: a
 * numeric op over a STRING, a non-ASCII LOWER / UPPER operand, a CONCAT / LOWER / UPPER result under FARM_HASH.  After a
 * failure the outputs' contents are unspecified.
 *
 * Predicates inside expressions (`sum(if(status in (200, 201, 204), 1, 0))`, `group by url like '%/api/%'`,
 * `group by if(is_prefix('https://', url), 'tls', 'plain')`, `lower(agent) like '%bot%'`), taken by this entry point only
 * (ytgpu_evaluate_expression refuses them as unknown ops), with or without string columns.  Each takes the value on top of
 * the stack and gives a BOOLEAN; a NULL operand gives NULL, any other TRUE or FALSE.
 *   IN                       one operand of type INT64, UINT64, DOUBLE, BOOLEAN or STRING: TRUE when it equals an entry of
 *                            the list.  `constant` = (offset << 32) | count: count 8-byte little-endian entries at an 8-aligned
 *                            offset of string_constants.  A number's entry is its bit pattern in the operand's type (a
 *                            BOOLEAN's 0 or 1); a STRING's is (offset << 32) | length of its bytes in string_constants.
 *                            Equality is COMPARE's EQ rule: a NaN operand or entry never matches, -0.0 equals +0.0; strings
 *                            are equal byte for byte.  The list holds no NULL: write is_null(x) OR x IN (...) instead.  An
 *                            empty list is FALSE for every non-NULL operand; duplicate entries are allowed.
 *   STARTS_WITH              one STRING (QL is_prefix(prefix, s)): whether its first len(prefix) bytes are the prefix given
 *                            by `constant` = (offset << 32) | length into string_constants.  An empty prefix matches
 *                            every non-NULL value.
 *   CONTAINS                 one STRING (QL is_substr(needle, s)): whether the needle, given as STARTS_WITH's prefix, occurs
 *                            in it as a contiguous byte sequence.  An empty needle matches every non-NULL value.
 *   LIKE                     one STRING: whether the WHOLE value matches the pattern given as STARTS_WITH's prefix, with the
 *                            escape byte in `column` (0..255; -1: no escape).  NOT LIKE is LIKE followed by NOT.  Pattern
 *                            bytes:
 *                              %  matches any byte sequence, including the empty one;
 *                              _  matches one character: one byte outside 0x80..0xBF, followed by any number of bytes in
 *                                 0x80..0xBF;
 *                              any other byte matches itself;
 *                              with an escape byte E, E followed by any byte X matches X literally.  A pattern that ends in
 *                              a lone E is an error.
 *                            As a regular expression over bytes, fully matched, % is [\x00-\xff]*, _ is
 *                            [^\x80-\xbf][\x80-\xbf]* and every other byte is itself.  Newlines are ordinary bytes and
 *                            matching is case-sensitive.  When the value and the pattern are valid UTF-8 this is exactly
 *                            "_ = one code point, % = any code-point sequence", the rule ClickHouse documents for LIKE.  YT
 *                            QL's like compiles to an RE2 expression; how that treats _ on multibyte input and whether % / _
 *                            cross a newline (RE2's dot_nl) was not read in the reference, so those two rules are unverified
 *                            against YT QL.  Work per row is bounded as in ytgpu_evaluate_filter: at most (value length) *
 *                            ceil(positions / 64) + segments steps, no backtracking.  CONTAINS(x) is the pattern %x% without
 *                            wildcards.
 * The STRING operand of IN, STARTS_WITH, CONTAINS and LIKE may be any string result (lower(concat(a, '/', b)) like 'x%'): it
 * is matched against the bytes it would be written as, case maps applied, as COMPARE does.  These ops pass on their
 * operand's errors, as every op but IF, AND and OR: `if(b = 0, 0, a / b) in (1, 2)` fails nowhere, `(a / b) in (1, 2)`
 * fails where b = 0.  They consume their operand's pieces and count none toward YTGPU_EXPR_MAX_PIECES.  CONTAINS and LIKE
 * match values shorter than 2^32 bytes: an operand of 2^32 bytes or more (a CONCAT of long values) in a row where the op
 * is evaluated fails the call with YTGPU_ERR_INVALID_ARGUMENT, "CONTAINS / LIKE over a value of 2^32 bytes or more".  Like
 * a value outside its heap this is an input check: it does not follow the data, so it fails in an IF branch not taken
 * and under FALSE AND too.  STARTS_WITH and IN take any length.
 * Limits, per call, those of ytgpu_evaluate_filter: at most YTGPU_FILTER_MAX_IN_ENTRIES (65536) IN entries over all IN
 * nodes, YTGPU_FILTER_MAX_PATTERN_POSITIONS (256) positions per CONTAINS needle or LIKE pattern and
 * YTGPU_FILTER_MAX_PATTERN_BYTES (32 KiB) of compiled patterns (sizes as stated there).  Lists, prefixes, needles and
 * patterns live in string_constants, so they count against its 1 MiB.
 * Launches: as above, one for a numeric or BOOLEAN result and five for a STRING one; the lists and compiled patterns travel
 * in the one upload of the program.
 * YTGPU_ERR_INVALID_ARGUMENT, besides the above: an operand type the op does not take (STARTS_WITH, CONTAINS, LIKE over a
 * non-STRING), an IN list that is not 8-byte aligned or leaves string_constants, a STRING entry outside string_constants, a
 * BOOLEAN entry other than 0 / 1, a prefix, needle or pattern outside string_constants, a LIKE escape outside -1..255, a
 * pattern that ends in a lone escape byte, a limit above, a CONTAINS / LIKE operand of 2^32 bytes or more.
 *
 * Timestamps (`group by timestamp_floor_day(ts)`, `group by format_timestamp(ts, '%Y-%m')`).  A timestamp is seconds since
 * the Unix epoch, UTC, proleptic Gregorian, no leap seconds, in an INT64 or UINT64 operand; a NULL operand gives NULL.
 *   TIMESTAMP_FLOOR(unit)    both entry points; `column` the ytgpu_timestamp_unit -> the operand's type: HOUR t - t % 3600,
 *                            DAY t - t % 86400, WEEK the Monday 00:00 of t's week ((d - (d + 3) % 7) * 86400 with
 *                            d = t / 86400), MONTH the first day of t's month at 00:00, YEAR January 1 of t's year at 00:00.
 *                            That QL's week starts on Monday is recalled, not read.
 *   FORMAT_TIMESTAMP         this entry point only (ytgpu_evaluate_expression refuses it as an unknown op) -> STRING: byte
 *                            for byte what C-locale strftime(format, gmtime(t)) writes.  `constant` = (offset << 32) |
 *                            length of the format in string_constants.  Conversions: %a %A %b %B %h %p (the C locale's
 *                            English names), %C %d %e %H %I %j %m %M %S %u %w %y %Y, %D %F %R %T, %U %W, the ISO %G %g %V,
 *                            %n %t %%; every other byte is itself; an empty format gives "".  That QL's format_timestamp
 *                            is the C library's strftime is recalled, not read.  The format is compiled when the program
 *                            is checked and travels in the program's one upload.  A formatted value is a STRING operand
 *                            like any other (CONCAT, COMPARE, IN, STARTS_WITH, CONTAINS, LIKE, IF, IF_NULL, LOWER, UPPER,
 *                            the result) and one piece toward YTGPU_EXPR_MAX_PIECES; under FARM_HASH it is
 *                            YTGPU_ERR_UNSUPPORTED, as a CONCAT result is.
 * A timestamp is accepted in [0, 253402300799] (9999-12-31T23:59:59Z).  An evaluated row outside it, or a WEEK floor whose
 * result would be negative (t before 1970-01-05), fails the call with YTGPU_ERR_UNSUPPORTED: the reference's result there
 * is not known (it is recalled to go through an unsigned instant).  This error follows the data as a division error does:
 * a row outside the selection, an IF branch not taken and FALSE AND x raise nothing.  YTGPU_ERR_UNSUPPORTED whatever the
 * data: another conversion (%c %x %X %r %Z %z %s %k %l %P %+ ...), an E / O modifier, a flag or width (%-d, %10Y), a lone %
 * at the end, a format whose longest output exceeds YTGPU_EXPR_MAX_FORMATTED_BYTES (64; a bound chosen to be safe, as the
 * reference's buffer size was not read).  YTGPU_ERR_INVALID_ARGUMENT: an operand other than INT64 / UINT64, a unit outside
 * 0 .. 4, a format outside string_constants.  Device scratch: 64 bytes per thread of the grid and FORMAT_TIMESTAMP node
 * (about 17 MB each on a 132-SM H100 at 10^6 rows or more). */
int ytgpu_evaluate_expression_strings(ytgpu_context* ctx, const ytgpu_column_view* columns, uint32_t column_count,
                                      const ytgpu_string_column* string_columns, uint32_t string_count,
                                      const uint8_t* string_constants /* host */, uint64_t string_constant_bytes,
                                      const ytgpu_expr_node* program /* host */, uint32_t node_count,
                                      const uint8_t* selection /* nullable, out_mem */, uint64_t* out_values,
                                      uint8_t* out_null_bitmap, uint8_t* out_heap, uint64_t out_heap_capacity,
                                      uint64_t* out_starts, uint32_t* out_lengths, uint8_t* out_null_bytemap,
                                      uint64_t* out_heap_bytes /* host */, uint8_t* out_value_type /* host, nullable */,
                                      uint64_t* out_null_count /* host, nullable */, int out_mem, ytgpu_error* err);

/* ---- segmented SUM / COUNT over rows ALREADY SORTED by the group key (the aggregate stage after a sort) ----
 * Consecutive rows with equal keys form a group; no hash table.  Replaces the per-group accumulation of a GROUP BY
 * over a sorted stream / a sorted reduce (yt/yt/library/query/engine/cg_routines/registry.cpp:1838-1920 for the
 * aggregation itself; sort_controller.cpp:3444-3456 produces the sorted partitions).  `in` (DEVICE) holds fixed-width
 * rows whose 8-byte key column at key_offset is non-decreasing (only equality of neighbours is used); the value column
 * at value_offset is INT64 / UINT64 (sums wrap mod 2^64) or DOUBLE.  out_* (DEVICE, `capacity` entries) receive one
 * entry per group in input order, *out_group_count (host) the number of groups; INVALID_ARGUMENT when it exceeds
 * capacity.  `in->rows` and out_* must be 8-byte aligned (INVALID_ARGUMENT otherwise).  Same sums / counts as
 * ytgpu_scan_filter_groupby over the same rows: double sums are added in arbitrary order starting from +0.0, so a
 * group of only -0.0 sums to +0.0, and a group holding a NaN, or both infinities, sums to a NaN. */
int ytgpu_reduce_sorted_fixed_rows(ytgpu_context* ctx, const ytgpu_fixed_rows_view* in, uint32_t key_offset,
                                   uint32_t value_offset, uint8_t value_type, uint64_t* out_keys, uint64_t* out_sums,
                                   uint64_t* out_counts, uint64_t capacity, uint64_t* out_group_count, ytgpu_error* err);

/* ---- YQL block aggregators over Arrow blocks, "combine all" form ----
 * A fixed-width arrow::ArrayData as TArrowBlock hands it to an aggregator: buffers[0] = validity (LSB bit order,
 * 1 = valid, NULL = no nulls), buffers[1] = 64-bit values; element i is values[offset + i], its validity bit is
 * bit (offset + i).  `nullable` = the YQL item type is Optional<T> (the aggregators' IsNullable template argument). */
typedef struct ytgpu_arrow_array {
    const void* values;
    const uint8_t* validity;
    int64_t offset;
    int64_t length;
    uint8_t value_type;   /* YTGPU_TYPE_INT64 / UINT64 / DOUBLE */
    uint8_t nullable;
    uint16_t reserved;
    int32_t mem;          /* ytgpu_mem of values / validity / the filter */
} ytgpu_arrow_array;

/* The states of the fixed-width aggregators side by side (TSumState, TAvgState, TState<IsNullable,TIn,IsMin>, count):
 * values are bit patterns in the column's type; *_valid mirror IsValid (always 1 for a non-optional column). */
typedef struct ytgpu_block_agg_state {
    uint64_t sum;         /* integers wrap mod 2^64 */
    uint64_t min_value;
    uint64_t max_value;
    uint64_t count;       /* Count(column) == Avg's Count: non-null rows that passed the filter */
    uint64_t count_all;   /* CountAll: rows that passed the filter */
    uint8_t sum_valid, min_valid, max_valid, value_type;
    uint32_t reserved;
} ytgpu_block_agg_state;

/* InitState: zero sums/counts, InitialStateValue for min/max (mkql_block_agg_minmax.cpp:76-101). */
void ytgpu_block_agg_state_init(ytgpu_block_agg_state* state, uint8_t value_type, uint8_t nullable);

/* IBlockAggregatorCombineAll::AddMany (yql/essentials/minikql/comp_nodes/mkql_block_agg_factory.h:34-45) of the sum /
 * avg / min / max / count / count_all aggregators (mkql_block_agg_sum.cpp:160-232,421-485, mkql_block_agg_minmax.cpp:
 * 697-770, mkql_block_agg_count.cpp) in ONE pass over the block: folds the batch into *state (host).  `filter`
 * (nullable) is the non-nullable bool filter column, one byte per row.  Same IsValid rules as the reference,
 * including its quirks (a filtered batch without nulls raises sum's IsValid even if no row passed).  Floating point:
 * the sum is a tree reduction (reproducible for a given length), min/max follow AggLess (NaN is the biggest, all NaNs
 * are equal, -0.0 == +0.0): of AggLess-equal values the last in row order stays, with its own bits, so the state is
 * the reference's bit for bit.  DEVICE `values` must be 8-byte aligned (INVALID_ARGUMENT otherwise). */
int ytgpu_block_combine_all(ytgpu_context* ctx, const ytgpu_arrow_array* column, const uint8_t* filter,
                            ytgpu_block_agg_state* state, ytgpu_error* err);

/* ---- columnar write side: rows -> columns -> scan-optimised integer segments ----
 * ytgpu_convert_integer_column replaces TIntegerColumnConverter<T>::Convert
 * (yt/yt/library/column_converters/integer_column_converter.cpp:69-161): value `column_index` of every row becomes
 * one 64-bit word (Int64 zig-zag encoded, Null -> 0) minus *out_base_value, plus a null bitmap (bit i of byte i/8,
 * 1 = null, 8*ceil(n/64) bytes).  The reference never lowers MinValue_ below its initial 2^64-1, so the base is
 * always 2^64-1 and the words are value+1 (mod 2^64); that is kept, the column decodes to the same values.
 * A value that is neither Null nor `value_type` (YTGPU_TYPE_INT64 / UINT64) -> YTGPU_ERR_SCHEMA_VIOLATION. */
int ytgpu_convert_integer_column(ytgpu_context* ctx, const ytgpu_rowset_view* rows, uint32_t column_index,
                                 uint8_t value_type, uint64_t* out_values, uint8_t* out_null_bitmap,
                                 uint64_t* out_base_value /* host */, int out_mem, ytgpu_error* err);

/* One segment of an unversioned integer column as TUnversionedIntegerColumnWriter<T>::DumpSegment emits it
 * (yt/yt/ytlib/table_chunk_format/integer_column_writer.cpp:353-538).  Data parts, in writer order:
 *   DirectDense     : bit-packed (value - min)            | null bitmap (1 bit per row)
 *   DictionaryDense : bit-packed dictionary (value - min) | bit-packed ids (0 = null, else 1-based first-seen id)
 *   DirectRle       : bit-packed run values               | null bitmap (1 bit per run) | bit-packed run starts
 *   DictionaryRle   : bit-packed dictionary               | bit-packed run ids          | bit-packed run starts
 * Bit-packed vectors are TBitPackedUnsignedVector: header word size | width << 56, then ceil(width*size/64) words
 * (yt/yt/core/misc/bit_packed_unsigned_vector-inl.h:31-90); bitmaps are 8*ceil(bits/64) bytes (bitmap.h:131-200). */
typedef struct ytgpu_integer_segment {
    uint32_t type;              /* EUnversionedIntegerSegmentType (table_chunk_format/private.h:25-30):
                                   0 DictionaryRle, 1 DictionaryDense, 2 DirectRle, 3 DirectDense */
    uint32_t row_count;         /* TSegmentMeta::row_count */
    uint64_t chunk_row_count;   /* rows of the chunk up to and including this segment */
    uint64_t min_value;         /* TIntegerSegmentMeta::min_value == TIntegerMeta::BaseValue (encoded domain) */
    uint64_t data_offset;       /* first byte of the segment's data in out_data */
    uint64_t data_bytes;
    uint64_t part_bytes[3];     /* sizes of the data parts in writer order (0 = absent) */
    uint32_t values_size;       /* TIntegerMeta::ValuesSize */
    uint32_t ids_size;          /* TIntegerMeta::IdsSize (dictionary types) */
    uint32_t row_indexes_size;  /* TKeyIndexMeta::RowIndexesSize (RLE types) */
    uint8_t values_width, ids_width, row_indexes_width;
    uint8_t direct;             /* TIntegerMeta::Direct */
} ytgpu_integer_segment;

/* Replaces AddValues + DumpSegment of the unversioned Int64/Uint64 column writer: `values` are the raw 64-bit
 * payloads (is_signed: zig-zag encoded first, integer_column_writer.cpp:24-33), null_bytemap (nullable) marks nulls.
 * A segment is cut every max_segment_value_count rows (config.cpp:130, default 131072) and encoded with whichever of
 * the four layouts the reference's size estimate makes smallest (first minimum in enum order).  chunk_row_offset =
 * rows already written to the chunk (it enters the RLE size estimate).  Segment descriptors go to HOST memory;
 * *out_data_bytes is always set, INVALID_ARGUMENT when out_capacity or segment_capacity is too small. */
int ytgpu_encode_integer_column(ytgpu_context* ctx, const uint64_t* values, const uint8_t* null_bytemap,
                                uint64_t row_count, int is_signed, uint32_t max_segment_value_count,
                                uint64_t chunk_row_offset, int mem, uint8_t* out_data, uint64_t out_capacity,
                                uint64_t* out_data_bytes, ytgpu_integer_segment* out_segments,
                                uint32_t segment_capacity, uint32_t* out_segment_count, ytgpu_error* err);

/* ---- floating-point and boolean column writers ----
 * One segment of an unversioned double / boolean column as the reference's writers dump it:
 *   TUnversionedFloatingPointColumnWriter<double>::DumpSegment (yt/yt/ytlib/table_chunk_format/
 *     floating_point_column_writer.cpp:213-240): ui64 value count | raw doubles (:21-31)  ||  null bitmap
 *   TUnversionedBooleanColumnWriter::DumpSegment (boolean_column_writer.cpp:196-216, DumpBooleanValues :18-28):
 *     ui64 value count  ||  value bitmap  ||  null bitmap
 * Bitmaps: bit i of byte i/8, 8*ceil(rows/64) bytes.  A NULL row stores a zero payload / a false bit (the payload of a
 * Null TUnversionedValue, AddValues :247-256 / :228-238).  Both segment metas are type 0, version 0. */
typedef struct ytgpu_plain_segment {
    uint32_t row_count;         /* TSegmentMeta::row_count */
    uint32_t reserved;
    uint64_t chunk_row_count;   /* rows of the chunk up to and including this segment */
    uint64_t data_offset;       /* first byte of the segment's data in out_data */
    uint64_t data_bytes;
    uint64_t part_bytes[3];     /* sizes of the data parts in writer order (0 = absent) */
} ytgpu_plain_segment;

/* `values`: raw 64-bit patterns of the doubles, null_bytemap (nullable) marks NULL rows.  A segment is cut every
 * max_segment_value_count rows (the reference finishes a segment once it holds at least that many values,
 * floating_point_column_writer.cpp:242-251).  Same capacity protocol as ytgpu_encode_integer_column. */
int ytgpu_encode_double_column(ytgpu_context* ctx, const uint64_t* values, const uint8_t* null_bytemap, uint64_t row_count,
                               uint32_t max_segment_value_count, uint64_t chunk_row_offset, int mem, uint8_t* out_data,
                               uint64_t out_capacity, uint64_t* out_data_bytes, ytgpu_plain_segment* out_segments,
                               uint32_t segment_capacity, uint32_t* out_segment_count, ytgpu_error* err);
/* `values`: one byte per row (non-zero = true).  The reference cuts boolean segments only at block boundaries; the
 * caller chooses max_segment_value_count (pass row_count for one segment). */
int ytgpu_encode_boolean_column(ytgpu_context* ctx, const uint8_t* values, const uint8_t* null_bytemap, uint64_t row_count,
                                uint32_t max_segment_value_count, uint64_t chunk_row_offset, int mem, uint8_t* out_data,
                                uint64_t out_capacity, uint64_t* out_data_bytes, ytgpu_plain_segment* out_segments,
                                uint32_t segment_capacity, uint32_t* out_segment_count, ytgpu_error* err);

/* Rows -> one flat column: the AddValues loops of the column converters / writers for Double, Boolean and String columns
 * (yt/yt/library/column_converters/floating_point_column_converter.cpp:117-127, boolean_column_converter.cpp,
 * string_column_converter.cpp:288-296; floating_point_column_writer.cpp:247-256, boolean_column_writer.cpp:228-238,
 * string_column_writer.cpp:689-705).  out_payload[i] = bit pattern of the double / 0 or 1 / the integer / the string's
 * offset in the rowset's heap; out_lengths (strings; nullable otherwise) its length; out_null_bytemap (nullable) 1 for a
 * Null value, whose payload and length are 0.  The outputs are the inputs of ytgpu_encode_double_column /
 * _boolean_column (one byte per row: narrow the 0 / 1 payloads) / _string_column (starts = payload, heap = the rowset's heap) and of
 * ytgpu_string_value_ids.  A value of another type -> YTGPU_ERR_SCHEMA_VIOLATION. */
int ytgpu_extract_column(ytgpu_context* ctx, const ytgpu_rowset_view* rows, uint32_t column_index, uint8_t value_type,
                         uint64_t* out_payload, uint32_t* out_lengths, uint8_t* out_null_bytemap, int out_mem, ytgpu_error* err);

/* ---- YT string column -> ClickHouse ColumnString (the string path of the CHYT scan) ----
 * ConvertStringLikeYTColumnToCHColumn (yt/chyt/server/columnar_conversion.cpp:429-648,907-912): rows
 * [start_index, start_index + value_count) of a string column in any of its encodings — direct, dictionary (1-based
 * indexes, 0 = null), RLE, dictionary + RLE — become ColumnString's `chars` (every value followed by a zero byte) and
 * `offsets` (offsets[i] = end of value i including that zero byte).  A null row and, with a filter hint
 * (:506-541, CountTotalStringLengthWithFilterHint :397-427), a row whose hint byte is 0 become empty strings; nulls
 * themselves travel in the separate null bytemap (ytgpu_build_bytemap_from_flags).  String i of the value column spans
 * [offset(i), offset(i + 1)) of `chars` with offset(0) = 0, offset(k) = avg_length * k + ZigZagDecode32(offsets[k - 1])
 * (DecodeStringRange, client/table_client/columnar-inl.h:20-50).
 * Two calls per batch: out_chars == NULL returns the exact size in *out_chars_bytes (the reference pre-computes it the
 * same way for the RLE and filter-hint shapes, :506-518,:566-575, and grows its buffer otherwise); then the call with a
 * buffer of at least that many bytes fills out_chars and out_offsets (value_count entries).  A too small capacity is
 * YTGPU_ERR_INVALID_ARGUMENT with the needed size in *out_chars_bytes. */
typedef struct ytgpu_string_column_view {
    const uint32_t* offsets;            /* TStrings: zig-zag encoded differences from avg_length * k (BitWidth 32) */
    uint64_t string_count;              /* strings in the value column (dictionary size when dictionary-encoded) */
    uint32_t avg_length;
    int32_t mem;                        /* ytgpu_mem of every input buffer (and of filter_hint) */
    const uint8_t* chars;
    uint64_t chars_bytes;
    const uint32_t* dictionary_indexes; /* nullable */
    uint64_t dictionary_index_count;
    const uint64_t* rle_indexes;        /* nullable; rle_indexes[0] == 0 */
    uint64_t rle_count;
    int64_t start_index;                /* TColumn::StartIndex */
    int64_t value_count;                /* TColumn::ValueCount */
} ytgpu_string_column_view;

int ytgpu_convert_string_column_to_ch(ytgpu_context* ctx, const ytgpu_string_column_view* column, const uint8_t* filter_hint,
                                      uint8_t* out_chars, uint64_t out_chars_capacity, uint64_t* out_offsets,
                                      uint64_t* out_chars_bytes /* host */, int out_mem, ytgpu_error* err);

/* ---- ClickHouse column -> unversioned values (the write-back side of CHYT) ----
 * TCHToYTConverter::ConvertColumnToUnversionedValues (yt/chyt/server/ch_to_yt_converter.cpp:970-1040) for the types whose
 * logical type is a "V1" simple type, i.e. TSimpleValueConverter::FillValueRange (:131-215) under an optional
 * TNullableConverter (:374-386): every row becomes one 16-byte value with id 0.
 *   INT8..INT64 -> Int64 (sign extended); UINT8..UINT64 -> Uint64; FLOAT32 (widened) / FLOAT64 -> Double;
 *   BOOL: a UInt8 that must be 0 or 1 -> Boolean, anything else fails the call ("Cannot convert value ... to YT boolean",
 *         :183-186; checked for every row, as the reference fills the nested column before it applies the null map);
 *   STRING: ColumnString (chars + offsets, offsets[i] = END of value i INCLUDING its terminating zero byte,
 *         contrib/clickhouse/src/Columns/ColumnString.h:46-53,122-126) -> String values that point into `chars`
 *         (data = offset of the first byte, length = size without the zero byte) — zero copy, as in the reference;
 *   DATE (UInt16) / DATETIME (UInt32) -> Uint64, DATE32 (Int32) / DATETIME64 (Int64) -> Int64, each after adding
 *         time_adjustment and casting back to the ClickHouse type (:150-155, :203-206); TIMESTAMP (DateTime64 mapped to
 *         the YT timestamp type) -> Uint64, a negative adjusted value fails the call (:189-195).
 * null_map (nullable): ColumnNullable's byte map; a non-zero byte turns the row into Null (MakeUnversionedNullValue).
 * Composite / decimal / enum / low-cardinality columns are YSON- or string-building paths and stay on the CPU. */
typedef enum ytgpu_ch_type {
    YTGPU_CH_INT8 = 1, YTGPU_CH_INT16 = 2, YTGPU_CH_INT32 = 3, YTGPU_CH_INT64 = 4,
    YTGPU_CH_UINT8 = 5, YTGPU_CH_UINT16 = 6, YTGPU_CH_UINT32 = 7, YTGPU_CH_UINT64 = 8,
    YTGPU_CH_FLOAT32 = 9, YTGPU_CH_FLOAT64 = 10, YTGPU_CH_BOOL = 11, YTGPU_CH_STRING = 12,
    YTGPU_CH_DATE = 13, YTGPU_CH_DATE32 = 14, YTGPU_CH_DATETIME = 15, YTGPU_CH_DATETIME64 = 16, YTGPU_CH_TIMESTAMP = 17
} ytgpu_ch_type;

typedef struct ytgpu_ch_column {
    int32_t type;              /* ytgpu_ch_type */
    int32_t mem;               /* ytgpu_mem of data, offsets, null_map */
    const void* data;          /* row_count fixed-width elements; STRING: the chars */
    const uint64_t* offsets;   /* STRING only: row_count end offsets */
    uint64_t chars_bytes;      /* STRING only */
    const uint8_t* null_map;   /* nullable */
    int64_t time_adjustment;   /* TimezoneAdjustmentSeconds_ (date / time types), normally 0 */
    uint64_t row_count;
} ytgpu_ch_column;

int ytgpu_convert_ch_column_to_values(ytgpu_context* ctx, const ytgpu_ch_column* column, ytgpu_value* out_values, int out_mem,
                                      ytgpu_error* err);

/* ---- string column writer ----
 * One segment of an unversioned string column as TUnversionedStringColumnWriter<String>::DumpSegment emits it
 * (yt/yt/ytlib/table_chunk_format/string_column_writer.cpp:589-636).  Data parts, in writer order:
 *   DirectDense     : bit-packed offsets | null bitmap (1 bit per row) | string bytes of all rows        (:201-229)
 *   DictionaryDense : bit-packed ids (0 = null, else 1-based first-seen id) | bit-packed dictionary offsets | dictionary bytes (:152-199)
 *   DirectRle       : bit-packed run starts | bit-packed offsets | null bitmap (1 bit per run) | string bytes of the runs (:496-537)
 *   DictionaryRle   : bit-packed run starts | bit-packed run ids | bit-packed dictionary offsets | dictionary bytes      (:539-586)
 * Offsets are END offsets stored as zig-zag differences from (i + 1) * expected_length (PrepareDiffFromExpected,
 * yt/yt/core/misc/bit_packed_unsigned_vector.cpp:11-33); DecodeStringPointersAndLengths reads them back. */
typedef struct ytgpu_string_segment {
    uint32_t type;              /* EUnversionedStringSegmentType (table_chunk_format/private.h:32-37):
                                   0 DictionaryRle, 1 DictionaryDense, 2 DirectRle, 3 DirectDense */
    uint32_t row_count;         /* TSegmentMeta::row_count */
    uint64_t chunk_row_count;   /* rows of the chunk up to and including this segment */
    uint64_t data_offset;       /* first byte of the segment's data in out_data (8-byte aligned) */
    uint64_t data_bytes;
    uint64_t part_bytes[4];     /* sizes of the data parts in writer order (0 = absent) */
    uint32_t expected_length;   /* TStringSegmentMeta::expected_length */
    uint32_t offsets_size;      /* TBlobMeta::OffsetsSize */
    uint32_t ids_size;          /* TBlobMeta::IdsSize (dictionary types) */
    uint32_t row_indexes_size;  /* TKeyIndexMeta::RowIndexesSize (RLE types) */
    uint8_t offsets_width, ids_width, row_indexes_width;
    uint8_t direct;             /* TBlobMeta::Direct */
    uint32_t reserved;
} ytgpu_string_segment;

/* Replaces AddValues + DumpSegment of the unversioned String column writer: value i is the lengths[i] bytes at
 * string_heap + starts[i]; null_bytemap (nullable) marks NULL rows (their starts / lengths are ignored).  A segment ends
 * once it holds max_segment_value_count values or more than max_buffer_bytes string bytes (0 = the reference's 32 MB,
 * string_column_writer.cpp:25,:701-703) and is encoded with whichever of the four layouts the reference's size estimate
 * makes smallest (first minimum in enum order, :589-593,:646-676).  Same capacity protocol as
 * ytgpu_encode_integer_column; out_data needs 8-byte alignment in DEVICE memory. */
int ytgpu_encode_string_column(ytgpu_context* ctx, const uint8_t* string_heap, uint64_t string_heap_bytes, const uint64_t* starts,
                               const uint32_t* lengths, const uint8_t* null_bytemap, uint64_t row_count,
                               uint32_t max_segment_value_count, uint64_t max_buffer_bytes, uint64_t chunk_row_offset, int mem,
                               uint8_t* out_data, uint64_t out_capacity, uint64_t* out_data_bytes,
                               ytgpu_string_segment* out_segments, uint32_t segment_capacity, uint32_t* out_segment_count,
                               ytgpu_error* err);

/* String GROUP BY keys: out_ids[i] = index of the FIRST row whose string equals row i's (so equal strings get equal ids and
 * the id of a group names a row that holds its key); NULL rows get id 0 and out_null_bytemap[i] = 1 (nullable output).
 * Feed out_ids (+ the bytemap as a null bitmap) to ytgpu_scan_filter_groupby[_multi] as a UINT64 key column: that is the
 * hashed aggregation over string keys of YT QL (GroupOpHelper with a string group item, cg_routines/registry.cpp:1571-1655:
 * the reference hashes and compares the string bytes per row) and of YQL's BlockCombineHashed over string keys
 * (mkql_block_agg.cpp:1234-1400).  Inputs as for ytgpu_encode_string_column; at most 2^30 rows per call. */
int ytgpu_string_value_ids(ytgpu_context* ctx, const uint8_t* string_heap, uint64_t string_heap_bytes, const uint64_t* starts,
                           const uint32_t* lengths, const uint8_t* null_bytemap, uint64_t row_count, uint64_t* out_ids,
                           uint8_t* out_null_bytemap, int mem, ytgpu_error* err);

/* Replaces the value extraction of the four unversioned string segment readers (string_column_reader.cpp: extractors
 * :39-71,:84-97,:130-143, readers :266-520): for every row of the segment the position of its string — out_start[i] bytes
 * from the segment's first byte, out_length[i] bytes long, so `segment_data` serves as the heap of the resulting values —
 * and out_null_bytemap[i] (nullable; a NULL row gets start 0, length 0).  `segment` (host) carries type, row_count,
 * expected_length, data_bytes and part_bytes; `segment_data` points at the segment's data_bytes bytes (8-byte aligned in
 * DEVICE memory).  Inconsistent sizes -> INVALID_ARGUMENT. */
int ytgpu_decode_string_segment(ytgpu_context* ctx, const ytgpu_string_segment* segment, const uint8_t* segment_data,
                                uint32_t* out_start, uint32_t* out_length, uint8_t* out_null_bytemap, int mem, ytgpu_error* err);

#ifdef __cplusplus
}
#endif
#endif /* YTGPU_H_ */
