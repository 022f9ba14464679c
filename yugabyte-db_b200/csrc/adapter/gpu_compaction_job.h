// gpu_compaction_job.h — C++ host adapter above the C ABI (include/ybgpu_compaction.h).
//
// Mirrors the reference's operator surface for this path so that the call sites in
// rocksdb::DBImpl (db/db_impl.cc:2548-2592, 4019-4035) change by one type name:
//
//     CompactionJob job(...);  job.Prepare();  mutex_.Unlock();  job.Run();  mutex_.Lock();  job.Install(...)
//
// Names, argument meaning and error behaviour follow rocksdb/db/compaction_job.h:75-194,
// rocksdb/db/compaction_context.h:25-72 and rocksdb/table/table_builder.h:93-136. The types below
// (Slice, Status, CompactionFeed, ...) are minimal stand-ins with the reference's member names so
// that this header compiles stand-alone (tests/test_adapter_cpp.py); inside the reference tree the
// real yb/rocksdb headers are included instead (see INTEGRATION.md).
#pragma once
#include <cstdint>
#include <cstring>
#include <functional>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../../include/ybgpu_compaction.h"

namespace ybgpu_adapter {

#ifndef YBGPU_ADAPTER_USE_REFERENCE_TYPES
struct Slice {   // yb/util/slice.h
  const uint8_t* data_ = nullptr; size_t size_ = 0;
  Slice() {}
  Slice(const uint8_t* d, size_t n) : data_(d), size_(n) {}
  Slice(const std::string& s) : data_(reinterpret_cast<const uint8_t*>(s.data())), size_(s.size()) {}
  const uint8_t* data() const { return data_; }
  size_t size() const { return size_; }
  bool empty() const { return size_ == 0; }
};

class Status {   // yb/util/status.h (codes used on this path)
 public:
  enum Code { kOk = 0, kNotFound = 1, kCorruption = 2, kNotSupported = 3, kInvalidArgument = 4, kIOError = 5,
              kRuntimeError = 7, kIllegalState = 9, kTryAgain = 25, kShutdownInProgress = 27 };   // util/status_codes.h:14-43
  Status() {}
  Status(Code c, std::string m) : code_(c), msg_(std::move(m)) {}
  static Status OK() { return Status(); }
  bool ok() const { return code_ == kOk; }
  bool IsShutdownInProgress() const { return code_ == kShutdownInProgress; }
  bool IsCorruption() const { return code_ == kCorruption; }
  bool IsTryAgain() const { return code_ == kTryAgain; }
  bool IsNotSupported() const { return code_ == kNotSupported; }
  Code code() const { return code_; }
  const std::string& message() const { return msg_; }
  std::string ToString() const { return ok() ? "OK" : msg_; }
 private:
  Code code_ = kOk; std::string msg_;
};

// rocksdb/db/compaction_context.h:25-35
class CompactionFeed {
 public:
  virtual ~CompactionFeed() = default;
  virtual Status Feed(const Slice& key, const Slice& value) = 0;
  virtual Status Flush() = 0;
};

// rocksdb/table/table_builder.h:93-136 (the members the compaction loop uses)
class TableBuilder {
 public:
  virtual ~TableBuilder() = default;
  virtual void Add(const Slice& key, const Slice& value) = 0;
  virtual Status status() const = 0;
  virtual Status Finish() = 0;
  virtual void Abandon() = 0;
  virtual uint64_t NumEntries() const = 0;
  virtual uint64_t TotalFileSize() const = 0;
  virtual uint64_t BaseFileSize() const = 0;
};
#endif

inline Status ToStatus(ybgpu_status s, const char* msg) {
  return s == YBGPU_OK ? Status::OK() : Status(static_cast<Status::Code>(s), msg ? msg : "");
}

// docdb::HistoryRetentionDirective + CompactionHybridTimeConstraints (docdb/docdb_compaction_context.h:57-111,
// 178-196) flattened the way DocDBCompactionContext consumes them (docdb_compaction_context.cc:655-669).
struct DocDBRetention {
  bool enabled = true;                       // false: no compaction_context_factory on this DB
  uint64_t primary_cutoff_ht = YBGPU_HT_MIN;
  uint64_t cotables_cutoff_ht = YBGPU_HT_INVALID;
  int64_t table_ttl_ns = YBGPU_TTL_MAX_NS;
  bool retain_delete_markers_in_major_compaction = false;
  uint64_t other_min_ht = YBGPU_HT_MAX;
  // CompactionHybridTimeConstraints::input_min (docdb_compaction_context.h:178-196). DocDBCompactionFeed replaces the
  // output's user boundary values only when could_change_key_range_ holds, i.e. when no other data can lie before the
  // oldest input entry: !CanHaveOtherDataBefore(input_min) (docdb_compaction_context.cc:668,775-777). The default
  // (unknown) leaves the union of the inputs' values in place.
  uint64_t input_min_ht = YBGPU_HT_MAX;
  std::string key_bounds_lower, key_bounds_upper;
  bool CouldChangeKeyRange() const {
    const uint64_t min_other = retain_delete_markers_in_major_compaction ? YBGPU_HT_MIN : other_min_ht;
    return enabled && input_min_ht < min_other;
  }
};

// rocksdb::UserBoundaryValue (rocksdb/metadata.h): tag + encoded key component.
struct UserBoundaryValue { uint32_t tag = 0; std::string value; };

// FdWithBoundaries::user_filter_data (db/version_set.cc:3824) -> the engine's per-file HybridTime filters. Empty: no
// filter. First 8 bytes: the global filter (docdb/consensus_frontier.cc:245-253; invisible above it,
// docdb_rocksdb_util.cc:534-537). Behind it, n 4-byte database oids followed by n 8-byte hybrid times: the per-database
// cotable filters of the master's sys catalog after a restore (docdb_rocksdb_util.cc:503-509,541-563).
inline Status ParseUserFilterData(const Slice& user_filter_data, uint64_t* hybrid_time_filter,
                                  std::vector<uint32_t>* cotable_db_oids, std::vector<uint64_t>* cotable_hybrid_times) {
  *hybrid_time_filter = YBGPU_HT_INVALID;
  cotable_db_oids->clear(); cotable_hybrid_times->clear();
  if (user_filter_data.empty()) return Status();
  if (user_filter_data.size() < 8) return Status(Status::kCorruption, "user_filter_data shorter than a HybridTime");
  memcpy(hybrid_time_filter, user_filter_data.data(), 8);
  const size_t rest = user_filter_data.size() - 8;
  if (rest % 12) return Status(Status::kCorruption, "cotable filters are 12 bytes per database");
  const size_t n = rest / 12;
  cotable_db_oids->resize(n); cotable_hybrid_times->resize(n);
  if (n) {
    memcpy(cotable_db_oids->data(), user_filter_data.data() + 8, 4 * n);
    memcpy(cotable_hybrid_times->data(), user_filter_data.data() + 8 + 4 * n, 8 * n);
  }
  return Status();
}

// One L0 input file, as VersionSet::MakeInputIterator sees it (db/version_set.cc:3788-3849).
struct InputFile {
  Slice base_file;            // <n>.sst (metadata file) bytes
  Slice data_file;            // <n>.sst.sblock.0 bytes
  uint64_t hybrid_time_filter = YBGPU_HT_INVALID;   // FdWithBoundaries::user_filter_data (:3824), see ParseUserFilterData
  std::vector<uint32_t> cotable_db_oids;            // per-database cotable filters (sorted oids, a hybrid time each)
  std::vector<uint64_t> cotable_hybrid_times;
  // FileMetaData::smallest.seqno / largest.seqno of the input (db/version_edit.h:101-165). The reference seeds
  // every output file's seqno bounds with the union over the inputs (compaction_job.cc:1188-1195) before the
  // surviving entries extend them; leave the defaults when the caller does not track them.
  uint64_t smallest_seqno = YBGPU_MAX_SEQUENCE, largest_seqno = 0;
  // FileMetaData::delete_after_compaction(): set by the picker for files the CompactionFileFilter discards
  // (db/compaction_picker.cc:476-492); MakeInputIterator leaves such a file out of the merge (db/version_set.cc:3812-3820)
  // while it stays an input of the compaction (it is deleted afterwards; its seqno bounds still seed the outputs').
  bool delete_after_compaction = false;
  // The largest user frontier of the file, as far as whole-file TTL expiration reads it (docdb/compaction_file_filter.cc:
  // 70-85): ConsensusFrontier::hybrid_time and ::max_value_level_ttl_expiration_time (YBGPU_HT_INVALID = not set).
  bool has_largest_frontier = false;
  uint64_t frontier_hybrid_time = YBGPU_HT_MAX;
  uint64_t max_value_level_ttl_expiration_time = YBGPU_HT_INVALID;
};

// ---- whole-file TTL expiration: docdb::DocDBCompactionFileFilter(Factory) (docdb/compaction_file_filter.{h,cc}) ----------
// The reference's picker asks the factory for a filter over the compaction's input files and marks the files it discards;
// the compaction then skips them. Host logic on FileMetaData frontiers, no GPU work: it lives here so that the GPU job
// honours the same marks (Prepare) and a caller without the reference's picker can produce them (MarkExpiredFiles).
enum ExpiryMode { EXP_NORMAL = 0, EXP_TABLE_ONLY = 1, EXP_TRUST_VALUE = 2 };    // compaction_file_filter.h:26-30; flags :34-49
enum class FilterDecision { kKeep, kDiscard };                                   // rocksdb/compaction_filter.h
constexpr uint64_t kNoExpiration = YBGPU_HT_MAX;           // dockv/doc_ttl_util.h:73  HybridTime::kMax
constexpr uint64_t kUseDefaultTTL = YBGPU_HT_MIN + 1;      // :69                      HybridTime::kInitial
struct ExpirationTime {                                    // compaction_file_filter.h:32-43
  uint64_t ttl_expiration_ht = kNoExpiration;
  uint64_t created_ht = YBGPU_HT_MAX;
};
inline ExpirationTime ExtractExpirationTime(const InputFile* file) {             // :70-85
  ExpirationTime e;
  if (!file || !file->has_largest_frontier) return e;
  e.ttl_expiration_ht = file->max_value_level_ttl_expiration_time != YBGPU_HT_INVALID ? file->max_value_level_ttl_expiration_time : kNoExpiration;
  e.created_ht = file->frontier_hybrid_time;
  return e;
}
namespace ttl_detail {
inline bool IsSpecial(uint64_t ht) { return ht == YBGPU_HT_MIN || ht == YBGPU_HT_MAX || ht == YBGPU_HT_INVALID; }   // hybrid_time.h:185-194
// CompareHybridTimesToDelta (common/hybrid_time.cc:172-195): physical parts in nanoseconds against the delta, ties by the
// logical parts
inline int CompareToDelta(uint64_t begin, uint64_t end, int64_t delta_ns) {
  if (end < begin) return -1;
  const uint64_t bn = (begin >> 12) * 1000, en = (end >> 12) * 1000, dn = static_cast<uint64_t>(delta_ns);
  if (en - bn > dn) return 1;
  if (en - bn < dn) return -1;
  const uint64_t bl = begin & 0xfff, el = end & 0xfff;
  return el > bl ? 1 : (el < bl ? -1 : 0);
}
// dockv::ComputeExpiration (doc_ttl_util.cc:81-87): ht + ttl, kNoExpiration when the sum overflowed
inline uint64_t ComputeExpiration(uint64_t ht, int64_t ttl_ns) {
  const uint64_t expiry = IsSpecial(ht) ? ht : ht + (static_cast<uint64_t>(ttl_ns / 1000) << 12);
  return CompareToDelta(ht, expiry, ttl_ns) == 0 ? expiry : kNoExpiration;
}
// dockv::MaxExpirationFromValueAndTableTTL (:107-129)
inline uint64_t MaxExpiration(uint64_t key_ht, int64_t table_ttl_ns, uint64_t value_expiry) {
  if (value_expiry == kNoExpiration || IsSpecial(key_ht)) return kNoExpiration;
  if (table_ttl_ns == YBGPU_TTL_MAX_NS) return value_expiry == kUseDefaultTTL ? kNoExpiration : value_expiry;
  const uint64_t table_expiry = ComputeExpiration(key_ht, table_ttl_ns);
  if (table_expiry == kNoExpiration) return kNoExpiration;
  return value_expiry >= table_expiry ? value_expiry : table_expiry;
}
inline bool HasExpired(uint64_t expiration_ht, uint64_t read_ht) {               // dockv::HasExpiredTTL (:42-47)
  return expiration_ht != kNoExpiration && expiration_ht != kUseDefaultTTL && expiration_ht < read_ht;
}
}  // namespace ttl_detail
inline bool TtlIsExpired(const ExpirationTime expiry, int64_t table_ttl_ns, uint64_t now, ExpiryMode mode = EXP_NORMAL) {   // :126-144
  const uint64_t ttl_expiry_ht = mode == EXP_TABLE_ONLY ? kUseDefaultTTL : expiry.ttl_expiration_ht;
  if (mode == EXP_TRUST_VALUE && ttl_expiry_ht != YBGPU_HT_INVALID && ttl_expiry_ht != kUseDefaultTTL)
    return ttl_detail::HasExpired(ttl_expiry_ht, now);
  return ttl_detail::HasExpired(ttl_detail::MaxExpiration(expiry.created_ht, table_ttl_ns, ttl_expiry_ht), now);
}
inline bool IsLastKeyCreatedBeforeHistoryCutoff(ExpirationTime expiry, uint64_t history_cutoff) { return expiry.created_ht < history_cutoff; }

class DocDBCompactionFileFilter {                          // compaction_file_filter.h:69-97, .cc:150-188
 public:
  DocDBCompactionFileFilter(int64_t table_ttl_ns, uint64_t history_cutoff, uint64_t max_ht_to_expire, uint64_t filter_ht, ExpiryMode mode)
      : table_ttl_ns_(table_ttl_ns), history_cutoff_(history_cutoff), max_ht_to_expire_(max_ht_to_expire), filter_ht_(filter_ht), mode_(mode) {}
  // Files are expired from the oldest on: a file goes only if it was created before every file that stays
  // (max_ht_to_expire_); the two conditions the factory already applied are checked again (the reference logs DFATAL and keeps).
  FilterDecision Filter(const InputFile* file) const {
    const ExpirationTime expiry = ExtractExpirationTime(file);
    if (!(expiry.created_ht < max_ht_to_expire_)) return FilterDecision::kKeep;
    if (!IsLastKeyCreatedBeforeHistoryCutoff(expiry, history_cutoff_)) return FilterDecision::kKeep;
    if (!TtlIsExpired(expiry, table_ttl_ns_, filter_ht_, mode_)) return FilterDecision::kKeep;
    return FilterDecision::kDiscard;
  }
  const char* Name() const { return "DocDBCompactionFileFilter"; }
  uint64_t max_ht_to_expire() const { return max_ht_to_expire_; }
 private:
  const int64_t table_ttl_ns_;
  const uint64_t history_cutoff_, max_ht_to_expire_, filter_ht_;
  const ExpiryMode mode_;
};

// DocDBCompactionFileFilterFactory::CreateCompactionFileFilter (:196-243): `now` = clock_->Now(), the retention directive
// as DocDBRetention carries it. The history cutoff is the smaller of the valid cutoffs; the smallest creation time among
// the files that have NOT expired, or still hold keys inside the history retention window, bounds what may be expired.
inline DocDBCompactionFileFilter CreateCompactionFileFilter(const std::vector<InputFile>& input_files, const DocDBRetention& retention,
                                                            uint64_t now, ExpiryMode mode = EXP_NORMAL) {
  uint64_t history_cutoff = YBGPU_HT_MAX;
  if (retention.cotables_cutoff_ht != YBGPU_HT_INVALID && retention.cotables_cutoff_ht < history_cutoff) history_cutoff = retention.cotables_cutoff_ht;
  if (retention.primary_cutoff_ht != YBGPU_HT_INVALID && retention.primary_cutoff_ht < history_cutoff) history_cutoff = retention.primary_cutoff_ht;
  uint64_t min_kept_ht = YBGPU_HT_MAX;
  for (const InputFile& f : input_files) {
    const ExpirationTime expiry = ExtractExpirationTime(&f);
    if (!TtlIsExpired(expiry, retention.table_ttl_ns, now, mode) || !IsLastKeyCreatedBeforeHistoryCutoff(expiry, history_cutoff))
      if (expiry.created_ht < min_kept_ht) min_kept_ht = expiry.created_ht;
  }
  return DocDBCompactionFileFilter(retention.table_ttl_ns, history_cutoff, min_kept_ht, now, mode);
}

// What the picker does with the filter (db/compaction_picker.cc:476-492): marks the discarded files. Returns how many.
inline size_t MarkExpiredFiles(std::vector<InputFile>* input_files, const DocDBRetention& retention, uint64_t now, ExpiryMode mode = EXP_NORMAL) {
  const DocDBCompactionFileFilter filter = CreateCompactionFileFilter(*input_files, retention, now, mode);
  size_t n = 0;
  for (InputFile& f : *input_files)
    if (filter.Filter(&f) == FilterDecision::kDiscard) { f.delete_after_compaction = true; n++; }
  return n;
}

// Routing (INTEGRATION.md section 2, "ShouldOffload"): whether the engine takes these input tables, decided on the host from
// the metadata files and one trailer byte per data block, before any upload. NotSupported = keep the stock CompactionJob
// for this compaction; files marked delete_after_compaction are not read and so not looked at.
inline Status CheckInputsSupported(const std::vector<InputFile>& inputs) {
  for (const InputFile& f : inputs) {
    if (f.delete_after_compaction) continue;
    ybgpu_status s = ybgpu_sst_check_supported(f.base_file.data(), f.base_file.size(), f.data_file.data(), f.data_file.size(), nullptr);
    if (s != YBGPU_OK) return ToStatus(s, ybgpu_last_error());
  }
  return Status::OK();
}

// TableBuilder over the product's host writer (what TableFactory::NewTableBuilder returns when the
// KV stream is consumed by a host-side CompactionFeed chain).
class GpuSideTableBuilder : public TableBuilder {
 public:
  explicit GpuSideTableBuilder(const ybgpu_job_options& table_options) {
    st_ = ToStatus(ybgpu_table_builder_create(&table_options, &b_), ybgpu_last_error());
  }
  ~GpuSideTableBuilder() override { if (b_) ybgpu_table_builder_destroy(b_); }
  void Add(const Slice& key, const Slice& value) override {
    if (st_.ok()) st_ = ToStatus(ybgpu_table_builder_add(b_, key.data(), key.size(), value.data(), value.size()), "Add");
  }
  Status status() const override { return st_; }
  Status Finish() override { if (st_.ok()) st_ = ToStatus(ybgpu_table_builder_finish(b_), "Finish"); return st_; }
  void Abandon() override {}
  uint64_t NumEntries() const override { return ybgpu_table_builder_num_entries(b_); }
  uint64_t TotalFileSize() const override { return ybgpu_table_builder_total_file_size(b_); }
  uint64_t BaseFileSize() const override { return ybgpu_table_builder_base_file_size(b_); }
  Status Files(Slice* data_file, Slice* base_file) const {
    const uint8_t *d, *m; uint64_t dl, ml;
    Status s = ToStatus(ybgpu_table_builder_files(b_, &d, &dl, &m, &ml), "files");
    if (s.ok()) { *data_file = Slice(d, dl); *base_file = Slice(m, ml); }
    return s;
  }
 private:
  ybgpu_table_builder* b_ = nullptr;
  Status st_;
};

// rocksdb::CompactionJob shape (db/compaction_job.h:75-194).
class GpuCompactionJob {
 public:
  struct Params {                       // what the CompactionJob ctor + Compaction* provide
    int device = 0;
    bool bottommost_level = true;       // Compaction::bottommost_level()
    uint64_t last_sequence = YBGPU_MAX_SEQUENCE;   // versions_->LastSequence()
    std::string largest_user_key;       // Compaction::GetLargestUserKey(); empty + !has => derived
    bool has_largest_user_key = false;
    DocDBRetention retention;
    uint32_t block_size = 32 * 1024;    // BlockBasedTableOptions
    int block_restart_interval = 16;
    int block_size_deviation = 10;
    uint32_t index_block_size = 32 * 1024;
    uint32_t min_keys_per_index_block = 100;
    int output_key_encoding = YBGPU_KEY_ENCODING_SHARED_PREFIX;   // data_block_key_value_encoding_format
    int filter_policy = YBGPU_FILTER_NONE;     // YBGPU_FILTER_DOCKEY_V3 for DocDB tables (docdb_rocksdb_util.cc:761-763)
    uint32_t filter_block_size = 64 * 1024;    // db_filter_block_size_bytes
    int output_compression = YBGPU_COMPRESSION_NONE;   // Options::compression: YBGPU_COMPRESSION_SNAPPY in production (docdb_rocksdb_util.cc:184),
                                                       // YBGPU_COMPRESSION_LZ4 when compression_type is LZ4; anything else is NotSupported
    bool verify_checksums = true;
    const volatile int32_t* shutting_down = nullptr;   // std::atomic<bool>* shutting_down_ in the reference
    // DBOptions::max_subcompactions (rocksdb/options.h:1029; default 1, util/options.cc:258). > 1: the
    // compaction is cut into key ranges on row boundaries (GenSubcompactionBoundaries,
    // compaction_job.cc:409-519) that run pipelined on private streams, one output file per range.
    uint32_t max_subcompactions = 1;
    uint32_t subcompactions_in_flight = 3;
    // Bytes of HBM the job (with max_subcompactions > 1: the whole pipelined compaction) may hold at once; 0 = unlimited.
    // A job that cannot fit is refused before upload (NotSupported) or fails when it would pass it (RuntimeError); the
    // pipelined compaction cuts a range that needs more into two at a row boundary and runs the halves instead.
    uint64_t device_memory_budget = 0;
    // Yield point, e.g. [](void* s) { static_cast<yb::PriorityThreadPoolSuspender*>(s)->PauseIfNecessary(); }
    // (util/file_reader_writer.cc:343): called between kernel phases and between subcompaction ranges.
    void (*yield_fn)(void*) = nullptr;
    void* yield_ctx = nullptr;
    // DBOptions::paranoid_file_checks (compaction_job.cc:932-971): Run() re-reads every finished table on the GPU before
    // it is copied to the host (ybgpu_job_verify_output: checksums, compressed streams, every entry, key order, contents
    // against the merge result) and returns Corruption instead of an output that fails it.
    bool paranoid_file_checks = false;
  };

  explicit GpuCompactionJob(const Params& p) : p_(p) {}
  ~GpuCompactionJob() { if (job_) ybgpu_job_destroy(job_); }
  GpuCompactionJob(const GpuCompactionJob&) = delete;
  GpuCompactionJob& operator=(const GpuCompactionJob&) = delete;

  // REQUIRED: mutex held (same contract as CompactionJob::Prepare). Captures parameters only.
  Status Prepare(const std::vector<InputFile>& inputs) {
    ybgpu_job_options o;
    ybgpu_job_options_init(&o);
    o.device = p_.device;
    o.bottommost_level = p_.bottommost_level;
    o.last_sequence = p_.last_sequence;
    o.largest_user_key = reinterpret_cast<const uint8_t*>(p_.largest_user_key.data());
    o.largest_user_key_len = p_.largest_user_key.size();
    o.has_largest_user_key = p_.has_largest_user_key;
    o.retention_enabled = p_.retention.enabled;
    o.history_cutoff_ht = p_.retention.primary_cutoff_ht;
    o.cotables_cutoff_ht = p_.retention.cotables_cutoff_ht;
    o.table_ttl_ns = p_.retention.table_ttl_ns;
    o.retain_delete_markers_in_major_compaction = p_.retention.retain_delete_markers_in_major_compaction;
    o.other_min_ht = p_.retention.other_min_ht;
    o.key_bounds_lower = reinterpret_cast<const uint8_t*>(p_.retention.key_bounds_lower.data());
    o.key_bounds_lower_len = p_.retention.key_bounds_lower.size();
    o.key_bounds_upper = reinterpret_cast<const uint8_t*>(p_.retention.key_bounds_upper.data());
    o.key_bounds_upper_len = p_.retention.key_bounds_upper.size();
    o.block_size = p_.block_size; o.block_restart_interval = p_.block_restart_interval;
    o.block_size_deviation = p_.block_size_deviation; o.index_block_size = p_.index_block_size;
    o.min_keys_per_index_block = p_.min_keys_per_index_block; o.verify_checksums = p_.verify_checksums;
    o.output_key_encoding = p_.output_key_encoding; o.filter_policy = p_.filter_policy; o.filter_block_size = p_.filter_block_size;
    o.output_compression = p_.output_compression;
    o.device_memory_budget = p_.device_memory_budget;
    o.yield_fn = p_.yield_fn; o.yield_ctx = p_.yield_ctx;
    o.compute_user_boundary_values = p_.retention.CouldChangeKeyRange() && p_.max_subcompactions <= 1;
    options_ = o;
    inputs_ = inputs;
    if (p_.max_subcompactions > 1) return Status::OK();      // every range creates its own job in Run()
    ybgpu_status s = ybgpu_job_create(&o, &job_);
    if (s != YBGPU_OK) return ToStatus(s, ybgpu_last_error());
    return Status::OK();
  }

  // REQUIRED: mutex NOT held. Replaces ProcessKeyValueCompaction; on success the output files are
  // available through output_data_file()/output_base_file() and stats().
  Status Run() {
    if (NumReadInputs() == 0) {   // every input was expired as a whole (or there were none): nothing to merge, no output file
      data_.clear(); base_.clear(); outputs_.clear(); stats_ = ybgpu_job_stats{};
      return Status::OK();
    }
    if (p_.max_subcompactions > 1) return RunSubcompactions();
    for (const InputFile& f : inputs_) {
      if (f.delete_after_compaction) continue;             // db/version_set.cc:3812-3820
      ybgpu_status s = ybgpu_job_add_input_sst(job_, f.base_file.data(), f.base_file.size(), f.data_file.data(),
                                               f.data_file.size(), f.hybrid_time_filter);
      if (s == YBGPU_OK && !f.cotable_db_oids.empty())
        s = ybgpu_job_set_cotable_filters(job_, f.cotable_db_oids.data(), f.cotable_hybrid_times.data(), static_cast<uint32_t>(f.cotable_db_oids.size()));
      if (s != YBGPU_OK) return ToStatus(s, ybgpu_job_error(job_));
    }
    ybgpu_status s = ybgpu_job_run(job_, p_.shutting_down);
    if (s != YBGPU_OK) return ToStatus(s, ybgpu_job_error(job_));
    if (p_.paranoid_file_checks) {
      s = ybgpu_job_verify_output(job_, &output_check_);
      if (s != YBGPU_OK) return ToStatus(s, ybgpu_job_error(job_));
    }
    uint64_t dl = 0, ml = 0;
    s = ybgpu_job_output_sizes(job_, &dl, &ml);
    if (s != YBGPU_OK) return ToStatus(s, ybgpu_job_error(job_));
    data_.resize(dl); base_.resize(ml);
    s = ybgpu_job_fetch_output(job_, reinterpret_cast<uint8_t*>(&data_[0]), dl, reinterpret_cast<uint8_t*>(&base_[0]), ml);
    if (s != YBGPU_OK) return ToStatus(s, ybgpu_job_error(job_));
    ybgpu_job_get_stats(job_, &stats_);
    return Status::OK();
  }

  // CompactionJob::Run with subcompactions (compaction_job.cc:521-589): every key range becomes one
  // output file; outputs() lists them in range order the way Install adds them (:1128-1131).
  struct OutputFile {
    std::string data_file, base_file;        // <n>.sst.sblock.0, <n>.sst
    std::string smallest_key, largest_key;   // FileMetaData::smallest / largest (internal keys)
    // FileMetaData seqno bounds of THIS file: the union over the compaction's inputs (every output is seeded with it,
    // compaction_job.cc:1188-1195) extended by the file's own survivors (:156-169)
    uint64_t smallest_seqno = 0, largest_seqno = 0;
    ybgpu_job_stats stats;
  };
  Status RunSubcompactions() {
    ybgpu_job_options o = options_;
    o.largest_user_key = reinterpret_cast<const uint8_t*>(p_.largest_user_key.data());
    o.key_bounds_lower = reinterpret_cast<const uint8_t*>(p_.retention.key_bounds_lower.data());
    o.key_bounds_upper = reinterpret_cast<const uint8_t*>(p_.retention.key_bounds_upper.data());
    std::vector<ybgpu_input_file> files;
    uint64_t in_bytes = 0;
    for (const InputFile& f : inputs_) {
      if (f.delete_after_compaction) continue;             // db/version_set.cc:3812-3820
      files.push_back({f.base_file.data(), f.base_file.size(), f.data_file.data(), f.data_file.size(), f.hybrid_time_filter,
                       f.cotable_db_oids.data(), f.cotable_hybrid_times.data(), f.cotable_db_oids.size()});
      in_bytes += f.data_file.size();
    }
    // the output of a compaction is never larger than its input plus per-file metadata
    std::string data_arena, meta_arena;
    // under a budget a range may be cut again: room for more outputs than planned ranges
    const uint32_t slots = p_.device_memory_budget ? std::max<uint32_t>(1024, p_.max_subcompactions) : p_.max_subcompactions;
    data_arena.resize(in_bytes + in_bytes / 16 + (1u << 20) + 4096ull * slots);
    meta_arena.resize(in_bytes / 32 + (4u << 20) + 4096ull * slots);
    std::vector<ybgpu_sub_output> outs(slots);
    uint32_t n = slots;
    char err[512] = {0};
    ybgpu_status s = ybgpu_compact_files_checked(&o, files.data(), static_cast<uint32_t>(files.size()), p_.max_subcompactions,
                                                 p_.subcompactions_in_flight, reinterpret_cast<uint8_t*>(&data_arena[0]), data_arena.size(),
                                                 reinterpret_cast<uint8_t*>(&meta_arena[0]), meta_arena.size(), p_.shutting_down,
                                                 outs.data(), &n, &stats_, err, sizeof(err), p_.paranoid_file_checks ? 1 : 0);
    if (s != YBGPU_OK) return ToStatus(s, err);
    outputs_.clear();
    for (uint32_t i = 0; i < n; i++) {
      const ybgpu_sub_output& so = outs[i];
      if (!so.data_len) continue;             // nothing survived in this range: no file (compaction_job.cc:156-160)
      OutputFile f;
      f.data_file.assign(data_arena, so.data_offset, so.data_len);
      f.base_file.assign(meta_arena, so.meta_offset, so.meta_len);
      f.smallest_key.assign(reinterpret_cast<const char*>(so.smallest_key), so.smallest_key_len);
      f.largest_key.assign(reinterpret_cast<const char*>(so.largest_key), so.largest_key_len);
      f.stats = so.stats;
      SeqnoBounds(inputs_, so.stats.smallest_seqno, so.stats.largest_seqno, so.stats.num_output_records, &f.smallest_seqno, &f.largest_seqno);
      outputs_.push_back(std::move(f));
    }
    return Status::OK();
  }
  const std::vector<OutputFile>& outputs() const { return outputs_; }
  // What the device check of Run() read (Params::paranoid_file_checks, single-output jobs); zeroes otherwise.
  const ybgpu_output_check& output_check() const { return output_check_; }
  // Inputs that take part in the merge: all but the files marked delete_after_compaction (COMPACTION_FILES_NOT_FILTERED /
  // COMPACTION_FILES_FILTERED tickers, db/version_set.cc:3817-3820).
  size_t NumReadInputs() const { size_t n = 0; for (const InputFile& f : inputs_) n += !f.delete_after_compaction; return n; }
  size_t NumFilteredInputs() const { return inputs_.size() - NumReadInputs(); }

  // The range outputs as ONE table, for layouts where a compaction must leave a single sorted run (DocDB's
  // single-level universal compaction never forms subcompactions, db/compaction.cc:593-604): the data file
  // is the outputs' data files appended in order (nothing is re-encoded), the metadata file is rebuilt over
  // all blocks by ybgpu_sst_concat_meta. Key/value bytes equal the single-job output.
  Status ConcatenatedOutput(std::string* data_file, std::string* base_file) const {
    return ConcatFiles(options_, outputs_, data_file, base_file);
  }
  static Status ConcatFiles(const ybgpu_job_options& table_options, const std::vector<OutputFile>& files,
                            std::string* data_file, std::string* base_file) {
    const ybgpu_job_options& options_ = table_options;
    const std::vector<OutputFile>& outputs_ = files;
    data_file->clear(); base_file->clear();
    if (outputs_.empty()) return Status::OK();
    std::vector<ybgpu_sst_piece> pieces;
    uint64_t total = 0;
    for (const OutputFile& f : outputs_) {
      pieces.push_back({reinterpret_cast<const uint8_t*>(f.base_file.data()), f.base_file.size(), f.data_file.size(),
                        reinterpret_cast<const uint8_t*>(f.smallest_key.data()), static_cast<uint32_t>(f.smallest_key.size()),
                        reinterpret_cast<const uint8_t*>(f.largest_key.data()), static_cast<uint32_t>(f.largest_key.size())});
      total += f.data_file.size();
    }
    uint64_t cap = 0, len = 0;
    ybgpu_status s = ybgpu_sst_concat_meta(&options_, pieces.data(), static_cast<uint32_t>(pieces.size()), nullptr, 0, &cap);
    if (s != YBGPU_OK) return ToStatus(s, ybgpu_last_error());
    base_file->resize(cap);
    s = ybgpu_sst_concat_meta(&options_, pieces.data(), static_cast<uint32_t>(pieces.size()),
                              reinterpret_cast<uint8_t*>(&(*base_file)[0]), cap, &len);
    if (s != YBGPU_OK) return ToStatus(s, ybgpu_last_error());
    base_file->resize(len);
    data_file->reserve(total);
    for (const OutputFile& f : outputs_) data_file->append(f.data_file);
    return Status::OK();
  }

  // Variant for DBs whose CompactionFeed chain must see every surviving entry on the host (e.g. the
  // packed-row repacker): the GPU still does decode + merge + retention, the host feed gets the
  // stream in order (compaction_job.cc:797-800 semantics: first non-OK aborts).
  Status RunIntoFeed(CompactionFeed* feed) {
    if (p_.max_subcompactions > 1 || !job_)
      return Status(Status::kNotSupported, "RunIntoFeed needs max_subcompactions == 1 (the host feed consumes one ordered stream)");
    for (const InputFile& f : inputs_) {
      if (f.delete_after_compaction) continue;             // db/version_set.cc:3812-3820
      ybgpu_status s = ybgpu_job_add_input_sst(job_, f.base_file.data(), f.base_file.size(), f.data_file.data(),
                                               f.data_file.size(), f.hybrid_time_filter);
      if (s == YBGPU_OK && !f.cotable_db_oids.empty())
        s = ybgpu_job_set_cotable_filters(job_, f.cotable_db_oids.data(), f.cotable_hybrid_times.data(), static_cast<uint32_t>(f.cotable_db_oids.size()));
      if (s != YBGPU_OK) return ToStatus(s, ybgpu_job_error(job_));
    }
    ybgpu_status s = ybgpu_job_run(job_, p_.shutting_down);
    if (s != YBGPU_OK) return ToStatus(s, ybgpu_job_error(job_));
    struct Ctx { CompactionFeed* feed; Status st; } ctx{feed, Status::OK()};
    s = ybgpu_job_emit_kv_stream(job_, [](void* c, const uint8_t* k, uint64_t kl, const uint8_t* v, uint64_t vl) -> int {
      Ctx* x = static_cast<Ctx*>(c);
      x->st = x->feed->Feed(Slice(k, kl), Slice(v, vl));
      return x->st.ok() ? 0 : static_cast<int>(x->st.code());
    }, &ctx);
    if (!ctx.st.ok()) return ctx.st;
    if (s != YBGPU_OK) return ToStatus(s, ybgpu_job_error(job_));
    ybgpu_job_get_stats(job_, &stats_);
    return feed->Flush();
  }

  // REQUIRED: mutex held. In the reference this adds the output FileMetaData to a VersionEdit
  // (compaction_job.cc:1098-1141); here it hands the caller what that edit needs.
  struct OutputMeta {
    std::string smallest_key, largest_key; uint64_t smallest_seqno = 0, largest_seqno = 0, num_entries = 0;
    // DocDBCompactionContext::UpdateMeta (docdb_compaction_context.cc:684-689): when replace_user_values is set the
    // caller assigns these to FileMetaData::smallest.user_values / largest.user_values; otherwise it keeps the union
    // of the inputs' values it seeded the output with (compaction_job.cc:1188-1195). The user FRONTIERS are not
    // derived from the KV stream at all: the caller keeps calling its DocDBCompactionContext::GetLargestUserFrontier
    // (history cutoff, :1387-1391) and the inputs' frontier union exactly as before (INTEGRATION.md).
    bool replace_user_values = false;
    std::vector<UserBoundaryValue> smallest_user_values, largest_user_values;
  };
  // rocksdb::CompactionJobStats (rocksdb/compaction_job_stats.h:35-99) as UpdateCompactionJobStats / RecordDroppedKeys /
  // ProcessKeyValueCompaction fill it (compaction_job.cc:851-861,897-920,1337-1371). Timing members stay with the caller
  // (it measures its own wall clock and file IO); num_input_deletion_records is not reported by the engine (0).
  struct CompactionJobStats {
    uint64_t elapsed_micros = 0;
    uint64_t num_input_records = 0, num_input_files = 0, num_input_files_at_output_level = 0;
    uint64_t num_output_records = 0, num_output_files = 0;
    bool is_manual_compaction = false;
    uint64_t total_input_bytes = 0, total_output_bytes = 0;
    uint64_t num_records_replaced = 0;               // += CompactionIteratorStats::num_record_drop_hidden (:904-911)
    uint64_t total_input_raw_key_bytes = 0, total_input_raw_value_bytes = 0;
    uint64_t num_input_deletion_records = 0;
    uint64_t num_expired_deletion_records = 0;       // += num_record_drop_obsolete (:912-919)
    uint64_t num_corrupt_keys = 0;
    static constexpr size_t kMaxPrefixLength = 8;
    std::string smallest_output_key_prefix, largest_output_key_prefix;   // user keys, cut to kMaxPrefixLength (:1359-1368)
  };
  static void FillCompactionJobStats(const ybgpu_job_stats& st, const std::vector<InputFile>& inputs, uint64_t output_bytes,
                                     uint64_t num_output_files, const std::string& smallest_internal_key,
                                     const std::string& largest_internal_key, CompactionJobStats* out) {
    out->num_input_records = st.num_input_records;
    out->num_input_files = inputs.size();            // marked-for-deletion files are inputs of the compaction too (:1318-1334)
    out->num_input_files_at_output_level = 0;        // universal compactions of level-0 files into level 0 count them all as inputs
    out->total_input_bytes = 0;
    for (const InputFile& f : inputs) out->total_input_bytes += f.base_file.size() + f.data_file.size();   // fd.GetTotalFileSize()
    out->num_output_records = st.num_output_records;
    out->num_output_files = num_output_files;
    out->total_output_bytes = output_bytes;
    out->num_records_replaced = st.num_record_drop_hidden;
    out->num_expired_deletion_records = st.num_record_drop_obsolete;
    out->total_input_raw_key_bytes = st.total_input_raw_key_bytes;
    out->total_input_raw_value_bytes = st.total_input_raw_value_bytes;
    out->num_corrupt_keys = 0;                       // a corrupt key aborts the job with Corruption instead of being counted
    auto prefix = [](const std::string& ikey) {
      const size_t ulen = ikey.size() >= 8 ? ikey.size() - 8 : 0;
      return ikey.substr(0, ulen < CompactionJobStats::kMaxPrefixLength ? ulen : CompactionJobStats::kMaxPrefixLength);
    };
    if (num_output_files > 0) { out->smallest_output_key_prefix = prefix(smallest_internal_key); out->largest_output_key_prefix = prefix(largest_internal_key); }
  }
  // After Install(): the job's CompactionJobStats.
  Status UpdateCompactionJobStats(CompactionJobStats* out) {
    OutputMeta m;
    Status s = Install(&m);
    if (!s.ok()) return s;
    uint64_t bytes = 0, files = 0;
    if (p_.max_subcompactions > 1) { for (const OutputFile& f : outputs_) { bytes += f.data_file.size() + f.base_file.size(); files++; } }
    else if (!data_.empty()) { bytes = data_.size() + base_.size(); files = 1; }
    FillCompactionJobStats(stats_, inputs_, bytes, files, m.smallest_key, m.largest_key, out);
    return Status::OK();
  }

  // Output seqno bounds the way the reference computes them: the union of the inputs' FileMetaData bounds
  // (UpdateBoundariesExceptKey, compaction_job.cc:1188-1195; db/version_edit.cc:133-152) extended by every
  // surviving entry's (possibly zeroed) sequence number (SubcompactionState::Feed, :156-169) — which is what the
  // engine reports. E.g. compaction_job_test.cc:389-436: inputs 3..4 and 1..2, one survivor rewritten to
  // seqno 0 => output bounds 0..4.
  static void SeqnoBounds(const std::vector<InputFile>& inputs, uint64_t kept_smallest, uint64_t kept_largest, uint64_t num_kept,
                          uint64_t* smallest, uint64_t* largest) {
    uint64_t lo = YBGPU_MAX_SEQUENCE, hi = 0;
    for (const InputFile& f : inputs) { lo = f.smallest_seqno < lo ? f.smallest_seqno : lo; hi = f.largest_seqno > hi ? f.largest_seqno : hi; }
    if (num_kept) { lo = kept_smallest < lo ? kept_smallest : lo; hi = kept_largest > hi ? kept_largest : hi; }
    *smallest = lo == YBGPU_MAX_SEQUENCE && !num_kept ? 0 : lo; *largest = hi;
  }
  Status Install(OutputMeta* meta) {
    if (p_.max_subcompactions > 1) {          // per-file metadata is in outputs(); this is the union
      *meta = OutputMeta();
      if (!outputs_.empty()) { meta->smallest_key = outputs_.front().smallest_key; meta->largest_key = outputs_.back().largest_key; }
      SeqnoBounds(inputs_, stats_.smallest_seqno, stats_.largest_seqno, stats_.num_output_records, &meta->smallest_seqno, &meta->largest_seqno);
      meta->num_entries = stats_.num_output_records;
      return Status::OK();
    }
    if (NumReadInputs() == 0) { *meta = OutputMeta(); return Status::OK(); }     // nothing was merged: no output file
    uint8_t a[4096], b[4096]; uint64_t al = 0, bl = 0;
    ybgpu_status s = ybgpu_job_output_boundaries(job_, a, &al, b, &bl);
    if (s != YBGPU_OK) return ToStatus(s, ybgpu_job_error(job_));
    meta->smallest_key.assign(reinterpret_cast<char*>(a), al);
    meta->largest_key.assign(reinterpret_cast<char*>(b), bl);
    SeqnoBounds(inputs_, stats_.smallest_seqno, stats_.largest_seqno, stats_.num_output_records, &meta->smallest_seqno, &meta->largest_seqno);
    meta->num_entries = stats_.num_output_records;
    meta->replace_user_values = false;
    if (options_.compute_user_boundary_values) {
      std::vector<ybgpu_user_value> lo(32), hi(32);
      uint32_t n = 0;
      s = ybgpu_job_output_user_values(job_, lo.data(), hi.data(), 32, &n);
      if (s == YBGPU_OK) {
        meta->replace_user_values = true;
        for (uint32_t i = 0; i < n; i++) {
          meta->smallest_user_values.push_back({lo[i].tag, std::string(reinterpret_cast<const char*>(lo[i].value), lo[i].len)});
          meta->largest_user_values.push_back({hi[i].tag, std::string(reinterpret_cast<const char*>(hi[i].value), hi[i].len)});
        }
      } else if (s != YBGPU_NOT_SUPPORTED) {
        return ToStatus(s, ybgpu_job_error(job_));
      }                                        // NotSupported: the inputs' union stays (a superset range, still correct)
    }
    return Status::OK();
  }

  // CompactionJob::CheckOutputFile (compaction_job.cc:932-971) on bytes instead of file names: the table must open —
  // footer, metaindex, properties, every level of the index (the host reader that also reads input tables, Snappy index
  // blocks included) and its first data block's checksum; with paranoid_file_checks (DBOptions::paranoid_file_checks, the
  // reference then iterates the whole table) every data block's stored bytes are checked against its trailer. A non-zero
  // `check_tail_for_zeros` is FLAGS_rocksdb_check_sst_file_tail_for_zeros: that many trailing bytes of the data file must
  // not all be zero (CheckSstTailForZeros, :940-948). The caller still runs the reference's own check on the files it
  // writes; this one catches a bad table before anything touches the disk.
  static Status CheckOutputFile(const Slice& data_file, const Slice& base_file, uint64_t num_entries, bool paranoid_file_checks,
                                uint64_t check_tail_for_zeros = 0) {
    if (check_tail_for_zeros > 0 && data_file.size() > 0) {
      const uint64_t n = check_tail_for_zeros < data_file.size() ? check_tail_for_zeros : data_file.size();
      bool all_zero = true;
      for (uint64_t i = 0; i < n && all_zero; i++) all_zero = data_file.data()[data_file.size() - 1 - i] == 0;
      if (all_zero) return Status(Status::kCorruption, "the tail of the data file is all zeros");
    }
    if (num_entries == 0) return Status::OK();                     // :950-952
    uint64_t checked = 0, bad = 0;
    const uint32_t stride = paranoid_file_checks ? 1u : 0xffffffffu;   // stride beyond the block count: the first block only
    ybgpu_status s = ybgpu_sst_verify_blocks(base_file.data(), base_file.size(), data_file.data(), data_file.size(), stride, &checked, &bad);
    if (s != YBGPU_OK) return ToStatus(s, ybgpu_last_error());
    if (checked == 0) return Status(Status::kCorruption, "the output table has entries but no data blocks");
    return Status::OK();
  }
  Status CheckOutputFile(bool paranoid_file_checks, uint64_t check_tail_for_zeros = 0) const {
    if (p_.max_subcompactions > 1) {
      for (const OutputFile& f : outputs_) {
        Status s = CheckOutputFile(Slice(f.data_file), Slice(f.base_file), f.stats.num_output_records, paranoid_file_checks, check_tail_for_zeros);
        if (!s.ok()) return s;
      }
      return Status::OK();
    }
    return CheckOutputFile(Slice(data_), Slice(base_), stats_.num_output_records, paranoid_file_checks, check_tail_for_zeros);
  }

  const std::string& output_data_file() const { return data_; }    // <n>.sst.sblock.0
  const std::string& output_base_file() const { return base_; }    // <n>.sst
  const ybgpu_job_stats& stats() const { return stats_; }

 private:
  Params p_;
  ybgpu_job* job_ = nullptr;
  std::vector<InputFile> inputs_;
  std::string data_, base_;
  std::vector<OutputFile> outputs_;
  ybgpu_job_options options_{};
  ybgpu_job_stats stats_{};
  ybgpu_output_check output_check_{};
};

}  // namespace ybgpu_adapter
