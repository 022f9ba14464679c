// host_sst.h — host-side (CPU) pieces of the product around the GPU engine:
//   * reading a split SST's metadata file to find the data-block handles
//     (reference: rocksdb/table/format.cc:118-153, table/block_based_table_reader.cc:759-765,
//      table/index_reader.h:215-256) — small, latency-bound host work the reference also does on
//      the CPU before a compaction starts (VersionSet::MakeInputIterator);
//   * the SST writer that turns the GPU's surviving KV stream (or, later, its finished data
//     blocks) into <n>.sst.sblock.0 + <n>.sst, mirroring rocksdb::BlockBasedTableBuilder
//     (table/block_based_table_builder.cc:498-903) and rocksdb::TableBuilder's interface
//     (table/table_builder.h:93-136).
// None of this is a CPU fallback for the GPU path: the merge / filter / decode never run here.
#pragma once
#include <cstdint>
#include <map>
#include <memory>
#include <string>
#include <vector>

namespace ybgpu {
namespace host {

struct Handle { uint64_t offset = 0, size = 0; };

// Contents of a block stored compressed (table/format.cc:441-500 UncompressBlockContents): `type` is the trailer's
// rocksdb::CompressionType — 1 Snappy, 4 LZ4, 5 LZ4HC (the same stream format). False on a malformed stream or another
// codec.
bool UncompressStoredBlock(uint8_t type, const uint8_t* stored, size_t n, std::string* out);
// The uncompressed image the engine builds when any input block is stored compressed (k_snappy_sizes): every block's
// contents + its 5-byte trailer, the contents' size read from the varint32 preamble of a Snappy / LZ4 / LZ4HC block (the
// stored size for a raw one), the way ybgpu_sst_check_supported reads trailers. `compressed` receives the number of
// blocks stored compressed. Handles (Handle or ybgpu_block_handle) must lie inside the file (checked by the callers).
template <typename H>
uint64_t UncompressedImageBytes(const uint8_t* data, const H* blocks, uint64_t n, uint64_t* compressed) {
  uint64_t total = 0, nc = 0;
  for (uint64_t i = 0; i < n; i++) {
    const uint8_t* p = data + blocks[i].offset;
    const uint64_t size = blocks[i].size;
    const uint8_t type = p[size];
    uint64_t u = size;
    if (type == 1 || type == 4 || type == 5) {          // Snappy, LZ4, LZ4HC: varint32 preamble
      nc++;
      u = 0;
      for (uint64_t j = 0; j < 5 && j < size; j++) {
        u |= static_cast<uint64_t>(p[j] & 127) << (7 * j);
        if (!(p[j] & 128)) break;
      }
    }
    total += u + 5;
  }
  *compressed = nc;
  return total;
}
uint32_t Crc32c(const uint8_t* p, size_t n, uint32_t init = 0);   // rocksdb/util/crc32c.h Extend
inline uint32_t Crc32cMask(uint32_t c) { return ((c >> 15) | (c << 17)) + 0xa282ead8u; }

struct SstMeta {
  std::vector<Handle> data_blocks;   // key order
  std::vector<std::string> separators;   // index key of every data block (>= its last key, < next block's first key)
  int key_encoding = 1;
  int index_levels = 1;
  std::map<std::string, std::string> properties;
  // fixed-size bloom filter blocks (metaindex entry "fixedsizefilter.<policy>"): handles inside the metadata
  // file and the keys of the filter index, in index order
  std::string filter_policy_name;
  std::vector<Handle> filter_blocks;
  std::vector<std::string> filter_index_keys;
};
// Returns empty string on success, else an error message.
std::string ParseSplitSstMeta(const uint8_t* meta, uint64_t len, SstMeta* out);

struct TableOptions {
  uint32_t block_size = 32 * 1024;
  int block_restart_interval = 16;
  int index_block_restart_interval = 1;
  int block_size_deviation = 10;
  uint32_t index_block_size = 32 * 1024;
  uint32_t min_keys_per_index_block = 100;
  int key_encoding = 1;
  int filter_policy = 0;             // 1 = DocKeyV3Filter fixed-size bloom blocks (docdb_filter_policy.h:71-80)
  uint32_t filter_block_size = 64 * 1024;
  int compression = 0;               // rocksdb::CompressionType of the output: 0 = kNoCompression, 1 = kSnappyCompression, 4 = kLZ4Compression
};

// The output codecs the writers (this file's and the GPU encoders) produce. Every entry point that takes an
// output_compression checks it against this before it starts, so that no other value silently yields a raw table.
inline bool OutputCompressionSupported(int compression) { return compression == 0 || compression == 1 || compression == 4; }
inline std::string UnsupportedOutputCompression(int compression) {
  return "output_compression " + std::to_string(compression) + " is not written by the engine (0 none, 1 Snappy, 4 LZ4)";
}

// FixedSizeFilterBitsBuilder geometry (util/bloom.cc:389-422) for filter blocks of `block_bytes`.
struct FilterGeometry { uint32_t num_lines = 0, num_probes = 0, max_keys = 0, filter_bytes = 0; };   // filter_bytes incl. 5 metadata bytes
FilterGeometry ComputeFilterGeometry(uint32_t block_bytes);

// Append-only encoder of one block (rocksdb::BlockBuilder, table/block_builder.cc:347-412).
class BlockEncoder {
 public:
  BlockEncoder(int restart_interval, int key_encoding);
  void Add(const uint8_t* key, size_t klen, const uint8_t* val, size_t vlen);
  const std::string& Finish();
  void Reset();
  bool empty() const { return body_.empty(); }
  size_t SizeEstimate() const { return body_.size() + (finished_ ? 0 : restarts_.size() * 4 + 4); }
  size_t SizeAfter(size_t klen, size_t vlen) const;
  size_t NumKeysForPolicy() const { return restarts_.size() * interval_ + in_interval_; }
 private:
  int interval_, encoding_;
  std::string body_, last_key_;
  std::vector<uint32_t> restarts_;
  int in_interval_ = 0;
  bool finished_ = false;
};

class IndexWriter;   // multi-level index (table/index_builder.cc:143-289)

// Writer of the metadata file (<n>.sst) alone: index blocks as data blocks are reported, then
// properties, metaindex and footer (block_based_table_builder.cc:543-592,762-903). Used directly
// when the data file was encoded on the GPU.
struct MetaProps {
  uint64_t raw_key_size = 0, raw_value_size = 0, data_size = 0, num_entries = 0, num_data_blocks = 0, deleted_keys = 0;
};
class MetaFileWriter {
 public:
  explicit MetaFileWriter(const TableOptions& o);
  ~MetaFileWriter();
  // `last_key` = last internal key of the block (modified in place into the separator),
  // `next_key` = first key of the next block (has_next = false for the last block).
  void AddDataBlock(std::string* last_key, const uint8_t* next_key, size_t next_len, bool has_next, const Handle& h);
  // A finished filter block (bits + 5 metadata bytes): BlockBasedTableBuilder::FlushFilterBlock
  // (block_based_table_builder.cc:594-620). `last_filter_key` = last key added to this block,
  // `next_key` = first key of the next filter block (has_next = false for the final flush).
  void AddFilterBlock(const uint8_t* contents, size_t len, std::string* last_filter_key, const uint8_t* next_key, size_t next_len, bool has_next);
  // Entries whose index keys are already final (re-emitting the blocks of finished files).
  void AddDataBlockRaw(const std::string& index_key, bool has_next, const Handle& h);
  void AddFilterBlockRaw(const uint8_t* contents, size_t len, const std::string& filter_index_key);
  void Finish(const MetaProps& p);
  const std::string& meta_file() const { return meta_; }
  void Reserve(size_t bytes) { meta_.reserve(bytes); }
  void TakeMetaFile(std::string* out) { out->swap(meta_); }
 private:
  void AppendBlock(const std::string& contents, Handle* h, bool compressible = false);
  TableOptions o_;
  std::unique_ptr<BlockEncoder> filter_index_;
  uint64_t filter_size_ = 0, num_filter_blocks_ = 0;
  std::unique_ptr<IndexWriter> index_;
  std::string meta_;
  Handle last_index_;
  bool last_index_set_ = false;
  uint64_t num_index_blocks_ = 0;
};

// One piece of a concatenation (ConcatSplitSstMeta): a finished split SST whose keys all sort after the
// previous piece's. smallest / largest = its first / last internal key.
struct SstPiece {
  const uint8_t* meta = nullptr; uint64_t meta_len = 0;
  uint64_t data_len = 0;
  std::string smallest, largest;
};
// Metadata file of the split SST whose data file is the pieces' data files back to back: one multi-level
// index over all data blocks (offsets rebased), every filter block with one filter index, summed
// properties. Nothing in the data files is re-encoded. Returns "" or an error message.
std::string ConcatSplitSstMeta(const TableOptions& o, const std::vector<SstPiece>& pieces, std::string* meta_out);

// The same assembly, piece by piece: a piece can be added as soon as its successor's smallest key is known (the
// index entry of its last block and the filter index entry of its last filter block are separators against it),
// so a pipelined compaction (ybgpu_compact_files_one_table) assembles the one table while later key ranges still
// run. AddPiece / Finish return "" or an error message.
class ConcatBuilder {
 public:
  explicit ConcatBuilder(const TableOptions& o);
  ~ConcatBuilder();
  void Reserve(size_t bytes);
  // next == nullptr: this is the last piece. parsed (optional): the piece's metadata file already parsed.
  std::string AddPiece(const SstPiece& piece, const SstPiece* next, const SstMeta* parsed = nullptr);
  std::string Finish(std::string* meta_out);
  uint64_t data_bytes() const { return base_; }
 private:
  TableOptions o_;
  MetaFileWriter* w_;
  MetaProps* mp_;
  uint64_t base_ = 0;
  size_t n_pieces_ = 0;
  std::string prev_largest_;
};

// rocksdb::TableBuilder shape: Add / Finish / NumEntries / TotalFileSize / status.
class SplitSstWriter {
 public:
  explicit SplitSstWriter(const TableOptions& o);
  ~SplitSstWriter();
  void Add(const uint8_t* ikey, size_t klen, const uint8_t* val, size_t vlen);
  void Finish();
  uint64_t NumEntries() const { return num_entries_; }
  uint64_t TotalFileSize() const { return data_.size() + metaw_.meta_file().size(); }
  uint64_t NumDataBlocks() const { return num_data_blocks_; }
  const std::string& data_file() const { return data_; }
  const std::string& meta_file() const { return metaw_.meta_file(); }
 private:
  void CutDataBlock(const uint8_t* next_key, size_t next_len, bool has_next);
  TableOptions o_;
  BlockEncoder block_;
  MetaFileWriter metaw_;
  std::string data_, last_key_;
  Handle pending_;
  uint64_t num_entries_ = 0, raw_key_ = 0, raw_val_ = 0, data_size_ = 0, num_data_blocks_ = 0, deleted_keys_ = 0;
  // host-side filter builder (the TableBuilder-shaped path; the compaction job builds filters on the GPU)
  void FlushFilter(const uint8_t* next_key, size_t next_len, bool has_next);
  FilterGeometry fg_;
  std::string filter_bits_, last_filter_key_;
  uint64_t filter_keys_ = 0;
};

}  // namespace host
}  // namespace ybgpu
