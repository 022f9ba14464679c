// range_plan.h — host-side planning shared by the pipelined subcompactions (subcompaction.cc) and the key-range
// sharded compaction across GPUs (range_exchange.cc): parsed input indexes, weighted splitter samples, row-aligned
// splitters (the GPU analogue of CompactionJob::GenSubcompactionBoundaries, rocksdb/db/compaction_job.cc:409-519) and
// the data blocks of an input that can hold the keys of a range.
#pragma once
#include <string>
#include <vector>

#include "../../include/ybgpu_compaction.h"
#include "host_sst.h"

namespace ybgpu {
namespace plan {

struct ParsedInput {
  host::SstMeta meta;
  std::vector<std::string> useps;      // user-key part of every block's index separator
};
struct Sample { std::string key; uint64_t w; };     // an index separator (user key) standing for w bytes of blocks
struct Span { size_t a, b; };                       // data blocks [a, b) of one input

std::string UserPart(const std::string& ikey);
bool ParseInputs(const ybgpu_input_file* files, uint32_t n, std::vector<ParsedInput>* out, std::string* err);
void CollectSamples(const std::vector<ParsedInput>& in, uint32_t n_ranges, std::vector<Sample>* out);
// The row prefix of an index separator a splitter is cut to (the DocKey when docdb_keys, the whole key otherwise); false
// when the separator gives no usable splitter (a key the engine does not take, or longer than YBGPU_MAX_SPLITTER_LEN).
bool RowPrefix(const std::string& key, bool docdb_keys, std::string* cut);
std::vector<std::string> SplittersFromSamples(std::vector<Sample> samples, uint32_t n_ranges, bool docdb_keys);
std::vector<std::string> PlanSplitters(const std::vector<ParsedInput>& in, uint32_t n_ranges, bool docdb_keys);
// A row-aligned splitter strictly inside [lo, hi) (empty = unbounded) halving the range's block bytes: the planner on the
// range's slice. False when no row boundary lies inside (one row, or no separator inside the range).
bool SplitRange(const std::vector<ParsedInput>& in, const std::string& lo, const std::string& hi, bool docdb_keys, std::string* mid);
void BlocksForRange(const std::vector<std::string>& useps, const std::string& lo, const std::string& hi, size_t* a, size_t* b);
// The block spans of one input a job over [lo, hi) must load: the blocks that can hold its keys and — when the range
// starts inside a cotable / colocated table — the blocks that hold that table's tombstones `id ! # HT` (they sort in
// front of the range but shadow its rows; the engine keeps them invisible except for seeding the table state).
// Spans are disjoint and ascending; adjacent ones are merged.
void SpansForRange(const ParsedInput& in, const std::string& lo, const std::string& hi, bool retention_enabled, std::vector<Span>* out);
bool LastKeyOfBlock(const uint8_t* blk, uint64_t size, int key_encoding, std::string* key);
bool LastKeyOfFile(const ybgpu_input_file& f, const host::SstMeta& m, std::string* key, bool verify_checksum = true);

}  // namespace plan
}  // namespace ybgpu
