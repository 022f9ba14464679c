/*
 * ybgpu_compaction.h — C ABI of the H100-native DocDB compaction engine.
 *
 * This is the drop-in boundary for the one hot path this repository replaces: the loop inside
 * rocksdb::CompactionJob::ProcessKeyValueCompaction (reference
 * src/yb/rocksdb/db/compaction_job.cc:664-895) together with everything that loop pulls through
 * per entry — MergingIterator/BlockIter (table/merger.cc:406-430, table/block.cc:348-447),
 * CompactionIterator (db/compaction_iterator.cc:139-483), DocDBCompactionFeed::Feed
 * (docdb/docdb_compaction_context.cc:941-1311) and BlockBasedTableBuilder::Add
 * (table/block_based_table_builder.cc:498-541).
 *
 * Plain pointers and sizes only; no C++/torch types.  Every entry point returns a ybgpu_status
 * (numerically equal to yb::Status::Code, util/status_codes.h; the C++ adapter casts) and fills the job's
 * error string on failure.  There is no CPU fallback: if no CUDA device is usable, create fails
 * with YBGPU_RUNTIME_ERROR.
 *
 * Threading: a job handle is used by one thread at a time (the reference runs one
 * PriorityThreadPool worker per CompactionJob, db_impl.cc:397-403); different jobs may run
 * concurrently on the same or different devices.
 */
#ifndef YBGPU_COMPACTION_H_
#define YBGPU_COMPACTION_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* yb::Status::Code values (src/yb/util/status_codes.h:14-43) used on this path; the numbers are the
 * reference's, so the adapter's static_cast<Status::Code>(s) is exact (tests/golden/status_codes_table.json holds the
 * table extracted from the reference header; tests/test_abi_cpu.py checks this enum against it). */
typedef enum ybgpu_status {
  YBGPU_OK = 0,
  YBGPU_NOT_FOUND = 1,
  YBGPU_CORRUPTION = 2,            /* bad block / entry / key encoding */
  YBGPU_NOT_SUPPORTED = 3,         /* e.g. compressed output, packed row without schema provider */
  YBGPU_INVALID_ARGUMENT = 4,
  YBGPU_IO_ERROR = 5,
  YBGPU_RUNTIME_ERROR = 7,         /* CUDA failure, out of device memory (status_codes.h:22) */
  YBGPU_ILLEGAL_STATE = 9,         /* (status_codes.h:24) */
  YBGPU_TRY_AGAIN = 25,            /* whole-subcompaction retry if no output was kept (compaction_job.cc:830-840) */
  YBGPU_SHUTDOWN_IN_PROGRESS = 27  /* shutting_down flag observed (compaction_job.cc:820-824; status_codes.h:43) */
} ybgpu_status;

/* rocksdb::KeyValueEncodingFormat (rocksdb/types.h:50-56); per input file from the table
 * property kDataBlockKeyValueEncodingFormat (block_based_table_reader.cc:759-765). */
enum { YBGPU_KEY_ENCODING_SHARED_PREFIX = 1, YBGPU_KEY_ENCODING_THREE_SHARED_PARTS = 2 };
enum { YBGPU_FILTER_NONE = 0, YBGPU_FILTER_DOCKEY_V3 = 1 };
enum { YBGPU_COMPRESSION_NONE = 0, YBGPU_COMPRESSION_SNAPPY = 1, YBGPU_COMPRESSION_LZ4 = 4 };   /* rocksdb::CompressionType (options.h:92-101) */

#define YBGPU_HT_MIN      0ull
#define YBGPU_HT_MAX      0xffffffffffffffffull
#define YBGPU_HT_INVALID  0xfffffffffffffffeull   /* HybridTime::kInvalid (common/hybrid_time.h:58) */
#define YBGPU_TTL_MAX_NS  0x7fffffffffffffffll    /* ValueControlFields::kMaxTtl = MonoDelta::kMax */
#define YBGPU_MAX_SEQUENCE 0x00ffffffffffffffull  /* kMaxSequenceNumber (db/dbformat.h:75) */
#define YBGPU_STREAM_PRIVATE ((void*)(intptr_t)-1) /* ybgpu_job_options::cuda_stream: job-owned stream */

/* Everything CompactionJob / DocDBCompactionContext know when the loop starts. */
typedef struct ybgpu_job_options {
  int32_t device;                    /* CUDA device ordinal */

  /* --- rocksdb::Compaction / CompactionIterator inputs --- */
  int32_t bottommost_level;          /* Compaction::bottommost_level() (db/compaction.cc:168-200) */
  uint64_t last_sequence;            /* VersionSet::LastSequence(): earliest_snapshot_ when there are
                                        no snapshots (compaction_iterator.cc:56-65) */
  const uint8_t* largest_user_key;   /* Compaction::GetLargestUserKey() (db/compaction.cc:318);  */
  uint64_t largest_user_key_len;     /* NULL/has=0 => engine derives it from the inputs          */
  int32_t has_largest_user_key;

  /* --- DocDB retention (docdb/docdb_compaction_context.h:57-111,178-196) ---
   * retention_enabled = 0 reproduces a DB without compaction_context_factory (plain RocksDB). */
  int32_t retention_enabled;
  uint64_t history_cutoff_ht;        /* HistoryCutoff::primary_cutoff_ht (HybridTime repr) */
  uint64_t cotables_cutoff_ht;       /* HistoryCutoff::cotables_cutoff_ht or YBGPU_HT_INVALID */
  int64_t table_ttl_ns;              /* HistoryRetentionDirective::table_ttl, YBGPU_TTL_MAX_NS = none */
  int32_t retain_delete_markers_in_major_compaction;
  uint64_t other_min_ht;             /* CompactionHybridTimeConstraints::other_min; HT_MAX = "major" */
  const uint8_t* key_bounds_lower;   /* docdb::KeyBounds (docdb/key_bounds.h); len 0 = unbounded */
  uint64_t key_bounds_lower_len;
  const uint8_t* key_bounds_upper;
  uint64_t key_bounds_upper_len;

  /* --- output table (rocksdb::BlockBasedTableOptions, table.h:107-217) --- */
  uint32_t block_size;               /* 32 KB in DocDB (dockv/packed_row.cc:39) */
  int32_t block_restart_interval;    /* 16 (docdb_rocksdb_util.cc:74,188) */
  int32_t block_size_deviation;      /* 10 (table.h:144) */
  int32_t output_key_encoding;       /* YBGPU_KEY_ENCODING_* */
  uint32_t index_block_size;         /* 32 KB */
  uint32_t min_keys_per_index_block; /* 100 */

  int32_t verify_checksums;          /* verify input block CRC32C (version_set.cc:3788-3849) */

  /* --- key-range sharding of one oversized compaction (SURVEY.md 8e; the GPU analogue of
   * subcompaction boundaries, rocksdb/db/compaction_job.cc:409-519,771-788): only entries with
   * range_lower <= user_key < range_upper take part; the others are invisible (not counted). */
  const uint8_t* range_lower; uint64_t range_lower_len;   /* len 0 = unbounded */
  const uint8_t* range_upper; uint64_t range_upper_len;
  void* cuda_stream;                 /* cudaStream_t to launch on; NULL = the legacy default stream;
                                        YBGPU_STREAM_PRIVATE = a non-blocking stream owned by the job
                                        (what concurrent jobs on one device should use) */

  /* --- bloom filter of the output (BlockBasedTableOptions::filter_policy, table.h:118-125) ---
   * YBGPU_FILTER_DOCKEY_V3 = docdb::DocDbAwareV3FilterPolicy (docdb_rocksdb_util.cc:761-763): fixed-size
   * filter blocks of filter_block_size bytes (db_filter_block_size_bytes, 64 KB), 1 % error rate, keyed
   * by the DocKey up to its hashed components / first range component; written into the metadata file
   * with a filter index (block_based_table_builder.cc:514-528,594-620,795-830). */
  int32_t filter_policy;             /* YBGPU_FILTER_* ; default none */
  uint32_t filter_block_size;        /* bytes; 65536 */

  /* --- yield points (PriorityThreadPoolSuspender::PauseIfNecessary, which the reference honours at its
   * file-write points: util/file_reader_writer.cc:343, compaction_job.cc:156-169) --- called on the job's
   * host thread between kernel phases of ybgpu_job_run and, by ybgpu_compact_files, before every range is
   * started; it may block for as long as the scheduler wants the compaction paused. NULL = none. */
  void (*yield_fn)(void* ctx);
  void* yield_ctx;

  /* --- FileMetaData user boundary values (docdb_compaction_context.cc:684-689,754-773) --- non-zero: the engine
   * reduces, over the first surviving entry of every DocKey, the bytewise smallest / largest encoded value of each
   * range-group component (DocBoundaryValuesExtractor, doc_boundary_values_extractor.cc:40-64); read them with
   * ybgpu_job_output_user_values. The caller sets it when DocDBCompactionFeed's could_change_key_range_ holds
   * (input_min has no other data before it, docdb_compaction_context.cc:668): only then does UpdateMeta replace
   * the union of the inputs' values. */
  int32_t compute_user_boundary_values;

  /* --- compression of the output (rocksdb::Options::compression; DocDB sets kSnappyCompression unless
   * enable_ondisk_compression is off, docdb_rocksdb_util.cc:176-202) --- YBGPU_COMPRESSION_SNAPPY: every data block
   * is run through a Snappy-format encoder on the GPU after it was assembled and is stored compressed (trailer type 1,
   * checksum over the compressed bytes) when that saves at least 12.5 % — BlockBasedTableBuilder::WriteBlock /
   * CompressBlock / GoodCompressionRatio (block_based_table_builder.cc:109-131,630-655); index blocks and the filter
   * index of the metadata file likewise (host). The compressed BYTES are this engine's encoder's, not the snappy
   * library's: any Snappy reader decodes them (tests: pyarrow's libsnappy), the block CONTENTS are the reference's.
   * YBGPU_COMPRESSION_LZ4: the same with an LZ4 encoder on the GPU (kLZ4Compression, trailer type 4, varint32 length +
   * one raw LZ4 block: compress_format_version 2, util/compression.h LZ4_Compress); any LZ4 block decoder reads them
   * (tests: liblz4, pyarrow's lz4_raw). Any other value is NotSupported at job creation (ybgpu_job_create,
   * ybgpu_compact_files*, ybgpu_compact_range_sharded, ybgpu_table_builder_create) before the device is touched. */
  int32_t output_compression;        /* YBGPU_COMPRESSION_* ; default none */

  /* --- device memory (INTEGRATION.md section 3 "Device memory") --- bytes of HBM the job may hold at once; 0 = unlimited
   * (the default). Every device allocation of a job (inputs, decode and merge arrays, the output table, the output check's
   * temporaries) is counted at its requested size, the engine's 32-byte pads included; the stream-ordered pool's own
   * rounding is not. add_input* and run first check on the host what is already known — the inputs' device copies plus,
   * when any input block is stored compressed, the uncompressed image (sum of the blocks' varint32 preambles) — and
   * refuse with YBGPU_NOT_SUPPORTED ("device memory budget exceeded ...", need and budget) before anything is uploaded.
   * An allocation during run that would pass the budget fails the job with YBGPU_RUNTIME_ERROR and the message
   * "device memory budget exceeded: need N, in use U, budget B"; the job's stream is drained first, so no kernel of it
   * is left running, and destroy returns every byte to the pool. Pipelined calls (ybgpu_compact_files*) take it as the
   * budget of the whole compaction. ybgpu_job_stats::device_bytes_peak reports the high-water mark either way. */
  uint64_t device_memory_budget;
} ybgpu_job_options;

void ybgpu_job_options_init(ybgpu_job_options* o);   /* reference defaults */

/* rocksdb::BlockHandle (table/format.cc:59-74): offset/size of a data block inside the input's
 * data file (<n>.sst.sblock.0), excluding the 5-byte trailer. */
typedef struct ybgpu_block_handle {
  uint64_t offset;
  uint64_t size;
} ybgpu_block_handle;

/* CompactionJobStats / CompactionIteratorStats fields filled by the loop
 * (compaction_job.cc:851-861,897-920; compaction_iterator.h). */
typedef struct ybgpu_job_stats {
  uint64_t num_input_records;
  uint64_t num_output_records;
  uint64_t num_record_drop_hidden;     /* rule A, compaction_iterator.cc:388-400 */
  uint64_t num_record_drop_obsolete;   /* kTypeDeletion at bottommost, :401-420 */
  uint64_t num_record_drop_feed;       /* dropped by the fused DocDB retention predicate */
  uint64_t total_input_raw_key_bytes;
  uint64_t total_input_raw_value_bytes;
  uint64_t total_output_raw_key_bytes;
  uint64_t total_output_raw_value_bytes;
  uint64_t num_output_data_blocks;
  uint64_t output_data_file_size;      /* bytes of <n>.sst.sblock.0 */
  uint64_t output_meta_file_size;      /* bytes of <n>.sst */
  uint64_t smallest_seqno, largest_seqno;   /* FileMetaData seqno bounds of the output */
  double gpu_seconds;                  /* device time of all kernels (CUDA events) */
  uint32_t gpu_kernel_launches;        /* kernels launched by run() */
  uint64_t h2d_bytes, d2h_bytes;       /* bytes copied by add_input / fetch calls */
  /* device time per phase (CUDA events on the job's stream), seconds:
   * 0 checksum verify + block scan (K1), 1 decode (K1'), 2 partition (K2), 3 merge+filter (K3),
   * 4 survivor scan + block encode + CRC + bloom filter blocks (K4/K5/K6),
   * 5 the block-assembler kernel alone (k_encode_smem, one launch; part of phase 4),
   * 6 / 7 the output block compressor (Snappy or LZ4) / the move of the stored blocks (output_compression; one launch
   * each; part of phase 4) */
  double phase_seconds[8];
  uint32_t phase_launches[8];
  /* which kernels ran (diagnostics, tests): YBGPU_PATH_* bits; summed over the ranges of a pipelined compaction */
  uint32_t path_flags;
  uint32_t tiles_inside_rows;          /* merge tiles that started inside a row group larger than a tile */
  /* high-water mark of the job's device bytes in use (requested sizes, 32-byte pads included, the pool's rounding not:
   * cudaMemPoolAttrUsedMemHigh of a job alone on its device is at least this, larger by the pool's granularity); for a
   * pipelined compaction, the high-water mark of the bytes all its ranges hold at once (every allocation and free of
   * every range updates one shared count), not the sum of the ranges' own peaks */
  uint64_t device_bytes_peak;
} ybgpu_job_stats;
enum {
  YBGPU_PATH_FUSED_INGEST = 1,         /* k_ingest: TMA-staged verify + value CRCs + decode in one pass */
  YBGPU_PATH_GENERAL_DECODE = 2,       /* k_prepass / k_decode_* / k_value_crc (other encodings, long keys, huge blocks) */
  YBGPU_PATH_SNAPPY = 4,               /* Snappy input blocks were uncompressed on the GPU */
  YBGPU_PATH_PARTITION_RETRY = 8,      /* the partition was repeated with a smaller sample stride */
  YBGPU_PATH_ENCODER_V4 = 16,          /* block assembler with checksums by CRC linearity */
  YBGPU_PATH_ENCODER_V5 = 32,          /* ... warp per block, no block image (k_encode_v5) */
  YBGPU_PATH_KV_INPUT = 64,            /* the inputs were KV streams (ybgpu_job_add_input_kv), not table files */
  YBGPU_PATH_SNAPPY_OUTPUT = 128,      /* output data blocks went through the GPU Snappy encoder (k_snappy_compress) */
  YBGPU_PATH_LZ4 = 256,                /* LZ4 (or LZ4HC) input blocks were uncompressed on the GPU */
  YBGPU_PATH_LZ4_OUTPUT = 512,         /* output data blocks went through the GPU LZ4 encoder (k_lz4_compress) */
  YBGPU_PATH_INGEST_RETRY = 1024,      /* k_ingest ran a second time at its widest record stride (a key longer than the probe's sample) */
  YBGPU_PATH_FAST_DECODE = 2048,       /* the general path decoded with k_decode_fast<...> rather than k_decode_all<...> */
  YBGPU_PATH_ENCODER_FUSED = 4096,     /* k_encode_fused wrote the output blocks larger than k_encode_v4's shared-memory image */
  YBGPU_PATH_OUTPUT_VERIFIED = 8192    /* ybgpu_job_verify_output re-read the finished table on the GPU and found it good */
};

typedef struct ybgpu_job ybgpu_job;

/* Replaces: CompactionJob ctor + Prepare() parameter capture (db/compaction_job.h:77-104). */
ybgpu_status ybgpu_job_create(const ybgpu_job_options* options, ybgpu_job** job);
void ybgpu_job_destroy(ybgpu_job* job);
const char* ybgpu_job_error(const ybgpu_job* job);       /* message of the last failure */
const char* ybgpu_last_error(void);                      /* for failures of create itself */

/* Replaces: VersionSet::MakeInputIterator's per-file TableCache::NewIterator
 * (db/version_set.cc:3788-3849). `data_file` is the whole data file in HOST memory; the copy to HBM is QUEUED
 * here on the job's stream (asynchronous DMA when the memory is pinned), so `data_file` must stay valid and
 * unchanged until ybgpu_job_run has returned or the job is destroyed (destroy synchronises the stream);
 * `handles` are the data-block handles in key order as read from the file's index (copied before returning).
 * `hybrid_time_filter` is the file's global HybridTime filter (docdb_rocksdb_util.cc:494-571) or
 * YBGPU_HT_INVALID.  Inputs may be added in any order; order does not affect the output. */
ybgpu_status ybgpu_job_add_input(ybgpu_job* job, const uint8_t* data_file, uint64_t data_file_len,
                                 const ybgpu_block_handle* handles, uint64_t num_handles,
                                 int32_t key_encoding, uint64_t hybrid_time_filter);

/* A sorted run the caller holds in MEMORY instead of a table file — the flush path's input: BuildTable
 * (rocksdb/db/builder.cc:119-318) walks the memtable iterator through the same CompactionIterator / TableBuilder chain a
 * compaction uses, so a job fed with the memtable's entries (and retention_enabled = 0, or the DocDB rules if the
 * caller wants them applied at flush time) writes the L0 table the reference would. `keys` = n internal keys (user key +
 * 8-byte suffix) back to back, key i at [key_offsets[i], key_offsets[i+1]); values likewise; entries in internal-key
 * order (checked: YBGPU_CORRUPTION otherwise). Host memory, copied (queued like ybgpu_job_add_input). KV-stream inputs
 * and table-file inputs cannot be mixed in one job. */
ybgpu_status ybgpu_job_add_input_kv(ybgpu_job* job, const uint8_t* keys, const uint64_t* key_offsets,
                                    const uint8_t* values, const uint64_t* value_offsets, uint64_t n);

/* Per-database cotable HybridTime filters of the input added LAST — the tail of FdWithBoundaries::user_filter_data
 * behind the 8-byte global filter (docdb/docdb_rocksdb_util.cc:503-509; written for the master's sys catalog by a
 * restore): `n` strictly increasing database oids with a hybrid time each. An entry of a cotable ('y' + uuid, the
 * uuid's last four bytes = the database oid) whose DocHybridTime is above its database's filter is invisible to the
 * compaction, like an entry above the global filter (HybridTimeFilteringIterator::Satisfied, :525-565). Copied. */
ybgpu_status ybgpu_job_set_cotable_filters(ybgpu_job* job, const uint32_t* db_oids, const uint64_t* hybrid_times, uint32_t n);

/* Blocks until every host->device copy queued by ybgpu_job_add_input has completed (the input buffers may then be
 * reused). Optional: ybgpu_job_run orders itself behind the copies anyway. The subcompaction pipeline uses it to keep
 * the copy engine on ONE range's inputs at a time instead of interleaving the chunks of all ranges in flight. */
ybgpu_status ybgpu_job_wait_inputs(ybgpu_job* job);

/* Same, but `data_file_dev` already lives in device memory of the job's device (used by the
 * bench's HBM-resident measurement and by callers that stage files themselves). Not copied, not
 * owned; must stay valid until destroy. The kernels fetch 16-byte vectors around entry boundaries:
 * 16 readable bytes before data_file_dev and 48 after data_file_dev + data_file_len are required
 * (ybgpu_job_add_input pads its own device copy the same way). */
ybgpu_status ybgpu_job_add_input_device(ybgpu_job* job, const uint8_t* data_file_dev, uint64_t data_file_len,
                                        const ybgpu_block_handle* handles, uint64_t num_handles,
                                        int32_t key_encoding, uint64_t hybrid_time_filter);

/* Convenience: parse a split SST's metadata file (<n>.sst: footer, metaindex, properties,
 * multi-level index; table/format.cc:118-153, table/index_reader.h:215-256) on the host and call
 * add_input with the handles / encoding found there. */
ybgpu_status ybgpu_job_add_input_sst(ybgpu_job* job, const uint8_t* meta_file, uint64_t meta_file_len,
                                     const uint8_t* data_file, uint64_t data_file_len,
                                     uint64_t hybrid_time_filter);

/* Replaces: CompactionJob::Run() -> ProcessKeyValueCompaction. Runs decode, merge, the fused
 * CompactionIterator + DocDB retention predicate and output encoding on the GPU. `shutting_down`
 * (may be NULL) is polled between kernel phases like compaction_job.cc:771. */
ybgpu_status ybgpu_job_run(ybgpu_job* job, const volatile int32_t* shutting_down);

ybgpu_status ybgpu_job_get_stats(const ybgpu_job* job, ybgpu_job_stats* stats);

/* --- results ---------------------------------------------------------------------------------
 * (a) The surviving KV stream in output order, the form CompactionFeed::Feed /
 *     TableBuilder::Add (table/table_builder.h:93-136) consume.  Sizes first, then one copy. */
ybgpu_status ybgpu_job_kv_stream_sizes(const ybgpu_job* job, uint64_t* num_entries,
                                       uint64_t* key_bytes, uint64_t* value_bytes);
/* key_offsets / value_offsets have num_entries + 1 elements. */
ybgpu_status ybgpu_job_fetch_kv_stream(ybgpu_job* job, uint8_t* keys, uint64_t* key_offsets,
                                       uint8_t* values, uint64_t* value_offsets);
/* Calls emit(ctx, key, klen, value, vlen) for every surviving entry in order; a non-zero return
 * aborts with that status (the reference aborts its loop on the first non-OK Feed,
 * compaction_job.cc:797-800). */
typedef int (*ybgpu_emit_fn)(void* ctx, const uint8_t* key, uint64_t key_len, const uint8_t* value,
                             uint64_t value_len);
ybgpu_status ybgpu_job_emit_kv_stream(ybgpu_job* job, ybgpu_emit_fn emit, void* ctx);

/* (b) The finished output SST, split the way the reference writes it
 *     (block_based_table_builder.cc:762-903, db/filename.cc:44-45): data blocks + trailers for
 *     <n>.sst.sblock.0 and index/properties/metaindex/footer for <n>.sst. */
ybgpu_status ybgpu_job_output_sizes(const ybgpu_job* job, uint64_t* data_file_len, uint64_t* meta_file_len);
ybgpu_status ybgpu_job_fetch_output(ybgpu_job* job, uint8_t* data_file, uint64_t data_cap,
                                    uint8_t* meta_file, uint64_t meta_cap);

/* FileMetaData boundaries of the output (db/version_edit.h:101-165): smallest / largest internal
 * key. Buffers must hold the longest key (use 4096). */
ybgpu_status ybgpu_job_output_boundaries(const ybgpu_job* job, uint8_t* smallest, uint64_t* smallest_len,
                                         uint8_t* largest, uint64_t* largest_len);

/* FileMetaData::smallest.user_values / largest.user_values of the output: one entry per range-group component that
 * occurs in a surviving DocKey, tag = 10 + component index (TagForRangeComponent, doc_boundary_values_extractor.cc:
 * 108-110), value = the encoded key component. Needs options.compute_user_boundary_values. Up to 16 components of up
 * to 255 bytes are reported; more => YBGPU_NOT_SUPPORTED (the caller then keeps the union of the inputs' values,
 * which is a superset range). *n = number of tags; smallest[i].tag == largest[i].tag. */
typedef struct ybgpu_user_value { uint32_t tag; uint32_t len; uint8_t value[256]; } ybgpu_user_value;
ybgpu_status ybgpu_job_output_user_values(ybgpu_job* job, ybgpu_user_value* smallest, ybgpu_user_value* largest,
                                          uint32_t cap, uint32_t* n);

/* --- subcompactions ------------------------------------------------------------------------------
 * Replaces: CompactionJob::GenSubcompactionBoundaries + the per-subcompaction threads of
 * CompactionJob::Run (rocksdb/db/compaction_job.cc:409-519,532-552; DBOptions::max_subcompactions,
 * rocksdb/options.h). One compaction is cut into key ranges on row boundaries; every range is an
 * ordinary job over the data blocks of each input that can hold its keys, bounded by
 * range_lower/range_upper like SubcompactionState::start/end (compaction_job.cc:721-729,779-783), and writes
 * its own output SST — the reference installs every sub-output in range order too
 * (compaction_job.cc:1128-1131). Note: with a single-level universal layout (DocDB's) the reference
 * never forms subcompactions (db/compaction.cc:593-604); see DESIGN.md "End-to-end modes". Ranges run on `max_in_flight` host threads with a private stream
 * each, so that the host->device copy of one range, the kernels of another and the device->host copy
 * of a third overlap (PCIe is full duplex); device memory in use is bounded by max_in_flight ranges
 * instead of the whole compaction. */
typedef struct ybgpu_input_file {
  const uint8_t* meta_file; uint64_t meta_file_len;     /* <n>.sst */
  const uint8_t* data_file; uint64_t data_file_len;     /* <n>.sst.sblock.0 (host memory; pinned = async DMA) */
  uint64_t hybrid_time_filter;                          /* YBGPU_HT_INVALID = none */
  const uint32_t* cotable_db_oids;                      /* per-database cotable filters (ybgpu_job_set_cotable_filters), or NULL */
  const uint64_t* cotable_hybrid_times;
  uint64_t num_cotable_filters;
} ybgpu_input_file;

#define YBGPU_MAX_SPLITTER_LEN 255
typedef struct ybgpu_sub_output {
  uint64_t data_offset, data_len;    /* <n>.sst.sblock.0 of this range inside the caller's data arena; len 0 = no output file */
  uint64_t meta_offset, meta_len;    /* <n>.sst inside the caller's metadata arena */
  ybgpu_job_stats stats;
  uint32_t range_lower_len, range_upper_len;            /* [lower, upper) user keys; len 0 = unbounded */
  uint8_t range_lower[256], range_upper[256];
  uint32_t smallest_key_len, largest_key_len;           /* FileMetaData::smallest / largest (internal keys) */
  uint8_t smallest_key[1032], largest_key[1032];
} ybgpu_sub_output;

/* Splitter user keys for at most `max_subcompactions` ranges, chosen from the inputs' index
 * separators weighted by block size and cut back to the row prefix (the DocKey when
 * docdb_keys != 0, the whole user key otherwise), so that no row — the unit of DocDB's retention
 * state — straddles two ranges. splitters: (max_subcompactions - 1) slots of 256 bytes. */
ybgpu_status ybgpu_plan_subcompactions(const ybgpu_input_file* files, uint32_t num_files, uint32_t max_subcompactions,
                                       int32_t docdb_keys, uint8_t* splitters, uint32_t* splitter_lens,
                                       uint32_t* num_splitters);

/* The row-aligned splitter that cuts the key range [lower, upper) (len 0 = unbounded) of the inputs in two halves of about
 * equal block bytes: the planner of ybgpu_plan_subcompactions on the range's slice. It lies strictly inside the range.
 * YBGPU_NOT_FOUND: no row boundary lies inside (the range holds one row, or no index separator falls inside it).
 * splitter: 256 bytes. */
ybgpu_status ybgpu_split_range(const ybgpu_input_file* files, uint32_t num_files, int32_t docdb_keys, const uint8_t* lower,
                               uint32_t lower_len, const uint8_t* upper, uint32_t upper_len, uint8_t* splitter, uint32_t* splitter_len);

/* Runs the whole compaction as pipelined subcompactions. options->range_* must be empty and
 * options->cuda_stream is ignored (every range gets a private stream). If
 * options->has_largest_user_key == 0 the key (Compaction::GetLargestUserKey) is read from the last
 * data block of every input on the host. outputs: max_subcompactions slots, filled in range order;
 * *num_outputs = number of ranges. err (optional) receives the message of the first failure.
 *
 * options->device_memory_budget != 0 is the budget of the whole compaction (ranges in flight together):
 *   * every range runs as a job with the budget B / max_in_flight and holds that reservation until it has run; it then
 *     holds its measured device_bytes_peak until it is destroyed. A range starts only while the reservations of the
 *     ranges on the device leave room for it, so the ranges' peaks at any moment sum to at most B;
 *   * max_subcompactions == 0: as many ranges as the budget needs; the first plan gives every range about
 *     (B / max_in_flight) / 3 bytes of input (inputs + uncompressed image), through ybgpu_plan_subcompactions;
 *   * a range whose job fails with "device memory budget exceeded" is cut in two at a row boundary (ybgpu_split_range)
 *     and both halves run in its place, one after the other; nothing of the failed attempt reached the caller's buffers.
 *     A range that cannot be cut (one row needs more than the budget) fails the compaction with that message;
 *   * outputs: *num_outputs on entry is the number of slots of `outputs` (ranges can outnumber max_subcompactions);
 *     YBGPU_INVALID_ARGUMENT if more ranges were needed. Ranges stay in key order; ybgpu_sub_output is as without a budget.
 *   * total->device_bytes_peak: the high-water mark of the bytes the ranges hold at once (as without a budget). */
ybgpu_status ybgpu_compact_files(const ybgpu_job_options* options, const ybgpu_input_file* files, uint32_t num_files,
                                 uint32_t max_subcompactions, uint32_t max_in_flight,
                                 uint8_t* data_arena, uint64_t data_arena_cap, uint8_t* meta_arena, uint64_t meta_arena_cap,
                                 const volatile int32_t* shutting_down, ybgpu_sub_output* outputs, uint32_t* num_outputs,
                                 ybgpu_job_stats* total, char* err, uint64_t err_cap);

/* The same pipelined compaction with ONE output table (device_memory_budget as for ybgpu_compact_files; every range that
 * was cut adds a block cut at its join, like any range boundary) — the shape DocDB's single-level universal compaction needs
 * (one sorted run per compaction; db/compaction.cc:593-604 never forms subcompactions there) and the shape
 * CompactionJob::Run writes without subcompactions. The key ranges still run pipelined on private streams, but
 *   * every range's data blocks are copied device->host straight to their final position in data_out (a range's
 *     offset is the sum of the sizes of all earlier ranges, known as soon as those have run), so the data file
 *     <n>.sst.sblock.0 is contiguous without any host copy;
 *   * the metadata file <n>.sst is assembled incrementally, in key order, while later ranges are still running:
 *     one multi-level index over all data blocks (index_builder.cc:143-289), every fixed-size bloom filter block
 *     under one filter index, summed properties — exactly what ybgpu_sst_concat_meta writes for the same pieces.
 * Key/value bytes equal the single-job output; block cuts differ only at the range boundaries.
 * result->smallest_key / largest_key: FileMetaData::smallest / largest of the table (internal keys). */
typedef struct ybgpu_one_table_result {
  uint64_t data_len, meta_len;
  uint32_t num_ranges, num_pieces;                      /* ranges planned / ranges that produced output */
  uint32_t smallest_key_len, largest_key_len;
  uint8_t smallest_key[1032], largest_key[1032];
} ybgpu_one_table_result;
ybgpu_status ybgpu_compact_files_one_table(const ybgpu_job_options* options, const ybgpu_input_file* files, uint32_t num_files,
                                           uint32_t max_subcompactions, uint32_t max_in_flight,
                                           uint8_t* data_out, uint64_t data_cap, uint8_t* meta_out, uint64_t meta_cap,
                                           const volatile int32_t* shutting_down, ybgpu_one_table_result* result,
                                           ybgpu_job_stats* total, char* err, uint64_t err_cap);

/* ybgpu_compact_files / ybgpu_compact_files_one_table with DBOptions::paranoid_file_checks: verify_outputs != 0 runs
 * ybgpu_job_verify_output on every range, on the range's own stream, right after it ran and before its device->host copy
 * starts, so a bad range fails the compaction before a byte of it reaches the caller's buffers (err: the first failing
 * range's message). Every verified range carries YBGPU_PATH_OUTPUT_VERIFIED in its stats. verify_outputs == 0: exactly
 * the unchecked calls. */
ybgpu_status ybgpu_compact_files_checked(const ybgpu_job_options* options, const ybgpu_input_file* files, uint32_t num_files,
                                         uint32_t max_subcompactions, uint32_t max_in_flight,
                                         uint8_t* data_arena, uint64_t data_arena_cap, uint8_t* meta_arena, uint64_t meta_arena_cap,
                                         const volatile int32_t* shutting_down, ybgpu_sub_output* outputs, uint32_t* num_outputs,
                                         ybgpu_job_stats* total, char* err, uint64_t err_cap, int32_t verify_outputs);
ybgpu_status ybgpu_compact_files_one_table_checked(const ybgpu_job_options* options, const ybgpu_input_file* files, uint32_t num_files,
                                                   uint32_t max_subcompactions, uint32_t max_in_flight,
                                                   uint8_t* data_out, uint64_t data_cap, uint8_t* meta_out, uint64_t meta_cap,
                                                   const volatile int32_t* shutting_down, ybgpu_one_table_result* result,
                                                   ybgpu_job_stats* total, char* err, uint64_t err_cap, int32_t verify_outputs);

/* --- one oversized compaction, key-range sharded across the GPUs of a box (SURVEY.md 8e; BASELINE config 5) ----------
 * Replaces, across devices, what CompactionJob::GenSubcompactionBoundaries + the subcompaction threads do inside one
 * process (rocksdb/db/compaction_job.cc:409-519,532-552). One process per GPU; every rank holds some of the tablet's
 * input files in host memory (any distribution). The ranks agree on world * rounds - 1 row-aligned splitter keys
 * (sampled index separators, all-gathered), rank d owns the `rounds` consecutive key ranges starting at d * rounds, and
 * per round every (file, destination) block slice travels once: host -> device staging in chunks of `chunk_bytes` ->
 * grouped ncclSend / ncclRecv over NVLink -> the destination's HBM ("one NCCL all-to-all", counts first). Each rank
 * then compacts its range on its GPU and returns ONE table (its rounds' outputs concatenated); the ranks' tables are
 * key-disjoint and ascending by rank — the order the reference installs sub-outputs in (compaction_job.cc:1128-1131).
 * rounds > 1 bounds HBM use to 1 / (world * rounds) of the compaction per GPU (inputs larger than the GPUs' memory).
 * The communicator is created from an ncclUniqueId the caller distributes (ybgpu_range_comm_unique_id on one rank). */
typedef struct ybgpu_range_comm ybgpu_range_comm;
ybgpu_status ybgpu_range_comm_unique_id(uint8_t id[128]);
ybgpu_status ybgpu_range_comm_create(const uint8_t id[128], int32_t rank, int32_t world, int32_t device, ybgpu_range_comm** comm);
void ybgpu_range_comm_destroy(ybgpu_range_comm* comm);
typedef struct ybgpu_range_shard_result {
  uint64_t data_len, meta_len;                          /* this rank's table */
  uint32_t num_ranges, num_pieces;                      /* key ranges of the whole compaction / outputs of this rank */
  uint64_t sent_bytes, received_bytes;                  /* through the exchange, this rank (incl. its own slices) */
  uint64_t sent_to_peers_bytes;                         /* the part that crossed NVLink */
  double plan_seconds, exchange_seconds, total_seconds; /* exchange: CUDA events around the grouped send / recv rounds */
  uint32_t range_lower_len, range_upper_len;            /* [lower, upper) user keys owned by this rank; len 0 = unbounded */
  uint8_t range_lower[256], range_upper[256];
  uint32_t smallest_key_len, largest_key_len;           /* FileMetaData::smallest / largest of this rank's table */
  uint8_t smallest_key[1032], largest_key[1032];
} ybgpu_range_shard_result;
ybgpu_status ybgpu_compact_range_sharded(ybgpu_range_comm* comm, const ybgpu_job_options* options, const ybgpu_input_file* local_files,
                                         uint32_t num_local_files, uint32_t rounds, uint64_t chunk_bytes,
                                         uint8_t* data_out, uint64_t data_cap, uint8_t* meta_out, uint64_t meta_cap,
                                         ybgpu_range_shard_result* result, ybgpu_job_stats* total, char* err, uint64_t err_cap);

/* One table out of the range outputs. For layouts where a compaction must produce a single sorted run
 * (DocDB's single-level universal compaction, db/compaction.cc:593-604), the per-range SSTs of
 * ybgpu_compact_files — ascending, key-disjoint — concatenate into one split SST without re-encoding
 * anything: the data file is the pieces' data files back to back (the caller appends them in order) and
 * this call writes its metadata file: one multi-level index over all data blocks with offsets rebased
 * (index_builder.cc:143-289), every fixed-size bloom filter block with one filter index, summed
 * properties, footer. Key/value bytes equal the single-pass output; block cuts differ only at the piece
 * boundaries. table_options: the options the pieces were written with. Call with meta_out = NULL to get
 * an upper bound of the size in *meta_len (the call with a buffer returns the exact length). */
typedef struct ybgpu_sst_piece {
  const uint8_t* meta_file; uint64_t meta_file_len;     /* <n>.sst of the piece */
  uint64_t data_file_len;                               /* length of its <n>.sst.sblock.0 */
  const uint8_t* smallest_key; uint32_t smallest_key_len;   /* first / last internal key of the piece */
  const uint8_t* largest_key; uint32_t largest_key_len;     /* (ybgpu_sub_output carries both) */
} ybgpu_sst_piece;
ybgpu_status ybgpu_sst_concat_meta(const ybgpu_job_options* table_options, const ybgpu_sst_piece* pieces,
                                   uint32_t num_pieces, uint8_t* meta_out, uint64_t meta_cap, uint64_t* meta_len);

/* Host-side integrity check of a split SST: walks the index of `meta_file` and verifies the trailer of every
 * `stride`-th data block (type byte kNoCompression, kSnappyCompression, kLZ4Compression or kLZ4HCCompression + masked
 * CRC32C over the stored bytes and the type, format.cc:352-395) in
 * `data_file`; stride 1 = every block. Used by bench.py on the full-size outputs it cannot compare with the
 * oracle. *bad_blocks > 0 => YBGPU_CORRUPTION. */
ybgpu_status ybgpu_sst_verify_blocks(const uint8_t* meta_file, uint64_t meta_file_len, const uint8_t* data_file,
                                     uint64_t data_file_len, uint32_t stride, uint64_t* blocks_checked, uint64_t* bad_blocks);

/* --- output check on the GPU ---------------------------------------------------------------------
 * Replaces: CompactionJob::CheckOutputFile under DBOptions::paranoid_file_checks (compaction_job.cc:932-971), which
 * re-opens the new table and iterates all of it. Here the finished data file is re-read while it is still in device
 * memory, before any byte of it is copied to the host: the block assembler derives the trailers from checksums of the
 * INPUT values and never reads a block back, so a trailer protects the reader but does not check the writer.
 *   1. every block's masked CRC32C is recomputed from the stored bytes and compared with its trailer;
 *   2. blocks stored compressed (Snappy, LZ4) are uncompressed into a scratch image; the stream must be well formed
 *      and as long as its preamble says;
 *   3. every entry is parsed the way BlockIter does (either key encoding): restart array inside the block, restart
 *      offsets ascending and at entries that share nothing, every header and every entry inside the block;
 *   4. internal keys strictly ascend inside every block and from block to block;
 *   5. (jobs only) the table holds the merge result: per-block and total entry counts, the first / last key against
 *      the boundary records of ybgpu_job_output_boundaries, and entry i of the table against survivor i — key bytes,
 *      value length and value bytes, the latter read from where the merge left them (the input file, the re-encoded
 *      control-field prefix, or "X" for a value that expired into a tombstone), not from the output.
 * The first failure is the one with the lowest (block, entry), whatever the kernels' scheduling. */
enum {
  YBGPU_CHECK_OK = 0,
  YBGPU_CHECK_CHECKSUM = 1,            /* stored bytes disagree with the block trailer */
  YBGPU_CHECK_COMPRESSED_STREAM = 2,   /* a compressed block does not decode to the length it announces */
  YBGPU_CHECK_ENTRY_PARSE = 3,         /* restart array or an entry header / body outside its block */
  YBGPU_CHECK_KEY_ORDER = 4,           /* a key is not above its predecessor */
  YBGPU_CHECK_ENTRY_COUNT = 5,         /* a block or the table holds another number of entries than the merge kept */
  YBGPU_CHECK_CONTENTS = 6,            /* an entry's key or value differs from the survivor that belongs there */
  YBGPU_CHECK_KEY_TOO_LONG = 7         /* ybgpu_sst_verify_device only: an internal key above 1016 bytes (NotSupported) */
};
typedef struct ybgpu_output_check {
  uint64_t blocks_checked;             /* data blocks of the table */
  uint64_t blocks_compressed;          /* ... of which stored compressed (trailer type != kNoCompression) */
  uint64_t entries_parsed;
  uint64_t bytes_read;                 /* stored table bytes + uncompressed bytes parsed (+ the values compared with, for a job) */
  double gpu_seconds;                  /* device time of the check (CUDA events on the job's stream) */
  uint32_t failure_kind;               /* YBGPU_CHECK_* of the first failure */
  uint32_t failure_block;              /* its data block (index order) */
  uint32_t failure_entry;              /* its entry inside that block (0 for failures of the block as a whole) */
  uint32_t reserved;
} ybgpu_output_check;

/* Checks 1-5 on the output of a job. Legal after a successful ybgpu_job_run (YBGPU_ILLEGAL_STATE otherwise), any number
 * of times, before or after the fetch calls. An empty output is YBGPU_OK with zero counts (compaction_job.cc:950-952).
 * A failure returns YBGPU_CORRUPTION, fills *result and ybgpu_job_error; success sets YBGPU_PATH_OUTPUT_VERIFIED in the
 * job's path_flags. The only large temporary is the uncompressed image of a compressed output; it is freed on return. */
ybgpu_status ybgpu_job_verify_output(ybgpu_job* job, ybgpu_output_check* result);

/* Checks 1-4 on ANY split SST held in host memory — the device counterpart of ybgpu_sst_verify_blocks, for a caller
 * that wants to scrub an input or re-check a file it wrote. The data file is uploaded (32 MB chunks), checked and
 * dropped. YBGPU_CORRUPTION with *result filled and the message in ybgpu_last_error on a failure. */
ybgpu_status ybgpu_sst_verify_device(int32_t device, const uint8_t* meta_file, uint64_t meta_file_len,
                                     const uint8_t* data_file, uint64_t data_file_len, ybgpu_output_check* result);

/* Last internal key of a split SST (its last data block is decoded on the host): what
 * FileMetaData::largest holds for the file. key must hold 1032 bytes. */
ybgpu_status ybgpu_sst_last_key(const uint8_t* meta_file, uint64_t meta_file_len, const uint8_t* data_file,
                                uint64_t data_file_len, uint8_t* key, uint32_t* key_len);

/* Routing pre-check for one input table, on the host, before any byte is copied to the GPU: walks the index of
 * `meta_file` and reads the trailer type byte of every data block of `data_file` (one byte per block). YBGPU_OK: the engine
 * takes the table (data blocks stored raw, Snappy-, LZ4- or LZ4HC-compressed, a key-value encoding it decodes, handles
 * inside the file). YBGPU_NOT_SUPPORTED: it would refuse it at run time (zlib / bzip2 / xpress / ZSTD blocks, blocks
 * labelled LZ4 / LZ4HC whose first bytes are no LZ4 length preamble it decodes, an unknown encoding) — the caller keeps the
 * stock CPU CompactionJob for this compaction (routing by job type, INTEGRATION.md section 2) without paying the upload;
 * YBGPU_CORRUPTION: the metadata file does not parse or a handle points outside the data file. Packed-row VALUES are not
 * visible from the trailers: the engine still reports those at run time. counts (may be NULL) = blocks stored with
 * CompressionType 0..7 (rocksdb/options.h:92-101). */
ybgpu_status ybgpu_sst_check_supported(const uint8_t* meta_file, uint64_t meta_file_len, const uint8_t* data_file,
                                       uint64_t data_file_len, uint64_t counts[8]);

/* What a job will need for the uncompressed image of this table (device_memory_budget's check before upload): every data
 * block's contents + 5-byte trailer, the contents' size read from the varint32 preamble of a Snappy / LZ4 / LZ4HC block and
 * the stored size of a raw one. A job allocates the image only when some input block is stored compressed:
 * *compressed_blocks counts those. Host only. YBGPU_CORRUPTION: the metadata file does not parse or a handle is outside. */
ybgpu_status ybgpu_sst_uncompressed_bytes(const uint8_t* meta_file, uint64_t meta_file_len, const uint8_t* data_file,
                                          uint64_t data_file_len, uint64_t* image_bytes, uint64_t* compressed_blocks);

/* Device-side checksum of the surviving KV stream: order-sensitive 64-bit hash over
 * (key_len, key, value_len, value) per entry, combined per entry position. Used by the parity
 * tests at sizes where copying the stream back is pointless. */
ybgpu_status ybgpu_job_kv_stream_digest(ybgpu_job* job, uint64_t* digest);

/* --- host-side table builder --------------------------------------------------------------------
 * rocksdb::TableBuilder shape (table/table_builder.h:93-136) over the product's split-SST writer:
 * what TableFactory::NewTableBuilder (rocksdb/table.h:394-397) returns when the engine's KV
 * stream is consumed entry by entry (e.g. after a host-only CompactionFeed such as the packed-row
 * repacker). Keys are internal keys in InternalKeyComparator order. */
typedef struct ybgpu_table_builder ybgpu_table_builder;
ybgpu_status ybgpu_table_builder_create(const ybgpu_job_options* table_options, ybgpu_table_builder** b);
ybgpu_status ybgpu_table_builder_add(ybgpu_table_builder* b, const uint8_t* key, uint64_t key_len,
                                     const uint8_t* value, uint64_t value_len);          /* Add() */
ybgpu_status ybgpu_table_builder_finish(ybgpu_table_builder* b);                         /* Finish() */
uint64_t ybgpu_table_builder_num_entries(const ybgpu_table_builder* b);                  /* NumEntries() */
uint64_t ybgpu_table_builder_total_file_size(const ybgpu_table_builder* b);              /* TotalFileSize() */
uint64_t ybgpu_table_builder_base_file_size(const ybgpu_table_builder* b);               /* BaseFileSize() */
ybgpu_status ybgpu_table_builder_files(const ybgpu_table_builder* b, const uint8_t** data_file, uint64_t* data_len,
                                       const uint8_t** meta_file, uint64_t* meta_len);
void ybgpu_table_builder_destroy(ybgpu_table_builder* b);                                /* Abandon() / dtor */

/* --- synthetic workload generator (benchmark tooling; SURVEY.md 8d "Synthetic inputs") ---------
 * Writes the BASELINE.json config shapes as split SSTs through the product's own table builder.
 * Row i has DocKey 'G' hash16 'S' <24 non-zero bytes> 00 00 '!' '!' (32 B), `cols` columns
 * ('K' + column id) and `versions` versions per column at base_micros + v*1000; version (i,c,v)
 * lives in file mix(seed,i,c,v) % num_files. Values: 'S' + value_len-1 pseudo-random bytes, or
 * the tombstone "X" with probability tombstone_per_1024/1024. */
typedef struct ybgpu_gen_config {
  uint64_t seed, num_rows;
  uint32_t cols, versions, num_files, value_len;
  uint64_t base_micros;
  uint32_t tombstone_per_1024, tombstone_newest;
  uint64_t row_offset, hash_rows_total;
} ybgpu_gen_config;
typedef struct ybgpu_sst ybgpu_sst;
ybgpu_status ybgpu_gen_sst(const ybgpu_gen_config* cfg, uint32_t file_index, const ybgpu_job_options* table_options, ybgpu_sst** out);
ybgpu_status ybgpu_gen_ssts(const ybgpu_gen_config* cfg, const ybgpu_job_options* table_options, ybgpu_sst** out, int32_t max_threads);
void ybgpu_sst_free(ybgpu_sst* s);
const uint8_t* ybgpu_sst_data(const ybgpu_sst* s, uint64_t* len);
const uint8_t* ybgpu_sst_meta(const ybgpu_sst* s, uint64_t* len);
uint64_t ybgpu_sst_num_entries(const ybgpu_sst* s);
uint64_t ybgpu_sst_raw_bytes(const ybgpu_sst* s);

/* Host-side reader of a split SST's metadata file: data-block handles in key order and the data
 * block key encoding (what the reference's TableReader learns at Open,
 * block_based_table_reader.cc:759-765 + index walk). Call with handles=NULL to get the count. */
ybgpu_status ybgpu_sst_meta_handles(const uint8_t* meta_file, uint64_t meta_file_len, ybgpu_block_handle* handles,
                                    uint64_t cap, uint64_t* num_handles, int32_t* key_encoding);

/* Index keys of the data blocks (the separators BlockBasedTableBuilder stored: >= last key of the
 * block, < first key of the next), concatenated into `keys` with num_handles+1 offsets. Used to
 * slice a file by key range (key-range sharding). Call with keys=NULL to get the sizes. */
ybgpu_status ybgpu_sst_meta_separators(const uint8_t* meta_file, uint64_t meta_file_len, uint8_t* keys, uint64_t keys_cap,
                                       uint64_t* key_offsets, uint64_t* num_keys, uint64_t* keys_bytes);

/* --- host placement ---------------------------------------------------------------------------------
 * Binds the CALLING thread to the CPUs of the NUMA node the device is attached to and makes that node the
 * thread's preferred memory node (threads created afterwards inherit both), so that staging buffers
 * allocated / first touched / pinned by it are one PCIe hop from the GPU instead of across the inter-socket
 * link. The reference's PriorityThreadPool workers are unbound (db_impl.cc:397-403); a device-attached worker
 * wants this in addition. ybgpu_compact_files binds its range worker threads this way (YBGPU_NUMA_BIND=0
 * disables). numa_node / num_cpus (optional) receive what was applied (-1 / 0: nothing to do on this host). */
int32_t ybgpu_device_numa_node(int32_t device);
ybgpu_status ybgpu_bind_thread_to_device(int32_t device, int32_t* numa_node, int32_t* num_cpus);

/* Library / device probe. */
int32_t ybgpu_device_count(void);
const char* ybgpu_version(void);

#ifdef __cplusplus
}
#endif
#endif  /* YBGPU_COMPACTION_H_ */
